"""Base class of the seven network modules: an `nn.Module` that owns parameters under the reference's state_dict
keys and whose forward is one C-ABI call into libtha4_b200.so (no PyTorch-op fallback)."""
import math
import weakref
from typing import Dict, List, Optional, Sequence

import torch
from torch import Tensor
from torch.nn import Module, Parameter

from tha4_b200._lib import Context, Tha4Error


# ---------------------------------------------------------------------- shared by the modules' autograd.Functions
def wants_autograd(*tensors: Tensor) -> bool:
    """Dispatch rule of the differentiable modules: forward goes through the module's autograd.Function when grad mode is
    on and any of `tensors` (its inputs; for the students, its parameters too) requires grad; otherwise it is the plain
    inference call."""
    return torch.is_grad_enabled() and any(t.requires_grad for t in tensors)


def refuse_double_backward(module_name: str):
    if torch.is_grad_enabled():
        raise Tha4Error('%s: double backward (create_graph=True) is not supported' % module_name)


def contiguous_grads(grad_outputs: Sequence[Optional[Tensor]]) -> List[Optional[Tensor]]:
    return [None if g is None else g.contiguous() for g in grad_outputs]


class _Node(Module):
    """Anonymous container so that dotted reference keys ('body.down_blocks.0.conv0.weight') map onto a module tree."""

    def forward(self, *args, **kwargs):
        raise Tha4Error('container node: call the owning network module instead')


def _init_tensor(shape, role: str, fan_in: int = 0, key: str = '') -> Tensor:
    """Reference initialisers by role (see state_dict_spec.py).  `fan_in`: fan-in of the weight this bias belongs to."""
    t = torch.empty(shape, dtype=torch.float32)
    if role in ('conv', 'conv1', 'convT', 'student_last'):
        fan_in = shape[1] * (shape[2] * shape[3] if len(shape) == 4 else 1)
        return t.normal_(0.0, math.sqrt(2.0 / fan_in))                      # kaiming_normal_ (init_function.py:14-16)
    if role in ('zconv', 'grid_head', 'last'):
        return t.zero_()                                                    # unet.py:26-30; poser_args.py:62-68
    if role in ('linear', 'film'):
        bound = 1.0 / math.sqrt(shape[1])
        return t.uniform_(-bound, bound)                                    # torch.nn.Linear default
    if role == 'norm_w':
        return t.fill_(1.0)
    if role in ('norm_b',):
        return t.zero_()
    if role == 'bias':
        if key.endswith('last_linear.bias') and fan_in > 0:
            # the students' last_linear is a plain Conv2d whose WEIGHT is re-initialised (siren.py:76-79, HeInitialization);
            # its bias keeps Conv2d's default uniform(+-1/sqrt(fan_in))
            b = 1.0 / math.sqrt(fan_in)
            return t.uniform_(-b, b)
        return t.zero_()
    if role == 'siren_first':
        return t.uniform_(-1.0 / shape[1], 1.0 / shape[1])                  # siren.py:32
    if role == 'siren':
        b = math.sqrt(6.0 / shape[1]) / 30.0
        return t.uniform_(-b, b)                                            # siren.py:34-36
    if role == 'siren_bias':
        # SineLinearLayer only re-initialises the weight (siren.py:31-36): the bias keeps Conv2d's default
        # uniform(+-1/sqrt(fan_in)), fan_in = in_channels of the 1x1 conv
        b = 1.0 / math.sqrt(fan_in) if fan_in > 0 else 0.0
        return t.uniform_(-b, b)
    raise ValueError(role)


class NativeModule(Module):
    NET_NAME: str = ''

    def __init__(self, spec):
        super().__init__()
        self._spec = spec
        fan_in = 0
        for key, shape, role in spec:
            if len(shape) >= 2:      # a weight: remember its fan-in for the bias that follows it in registration order
                fan_in = shape[1] * (shape[2] * shape[3] if len(shape) == 4 else 1)
            parts = key.split('.')
            node = self
            for p in parts[:-1]:
                if p not in node._modules:
                    node.add_module(p, _Node())
                node = node._modules[p]
            node.register_parameter(parts[-1], Parameter(_init_tensor(shape, role, fan_in, key)))
        self._ctx: Optional[Context] = None
        self._uploaded_key = None
        self._param_cache = None        # flat list of the parameters (walking the module tree costs ~0.3 ms per network per call)
        self._sync_calls = 0

    # ------------------------------------------------------------------ context / weights
    def attach_context(self, ctx: Context):
        self._ctx = ctx
        self._uploaded_key = None

    def _params(self):
        if self._param_cache is None:
            self._param_cache = list(self.parameters())
        return self._param_cache

    def _apply(self, fn, *args, **kwargs):
        # .to() / .cuda() / .float(): parameter storage moves, the packed copy in the library is stale
        out = super()._apply(fn, *args, **kwargs)
        self._param_cache = None
        self._uploaded_key = None
        return out

    def invalidate_weights(self):
        """Forces a re-upload on the next call (for writes the version counters do not see, e.g. `p.data = ...`)."""
        self._param_cache = None
        self._uploaded_key = None

    def _device(self) -> torch.device:
        return self._params()[0].device

    def context(self) -> Context:
        dev = self._device()
        if self._ctx is None or self._ctx.device != torch.device('cuda', dev.index if dev.index is not None else 0):
            if dev.type != 'cuda':
                raise Tha4Error('%s lives on %s: tha4_b200 modules run on CUDA only (no CPU fallback); call .to("cuda")'
                                % (type(self).__name__, dev))
            self._ctx = Context(dev)
            self._uploaded_key = None
        return self._ctx

    def sync_weights(self) -> Context:
        """(Re)packs the parameters into the library when they changed since the last upload."""
        ctx = self.context()
        # Every in-place write (optimizer steps, load_state_dict's copy_) bumps a parameter's version counter; storage moves
        # go through _apply.  Reading ~1 100 counters is ~0.1 ms for the whole teacher, against 1.3 ms for the
        # (data_ptr, version) walk over the module tree this replaced -- host time that is serial in a B=1 frame loop.
        # Every 256th call the parameter list itself is rebuilt (a Parameter object replaced by assignment).
        self._sync_calls += 1
        if (self._sync_calls & 255) == 0:
            self._param_cache = None
        params = self._params()
        key = (id(params[0]), params[0].data_ptr(), [p._version for p in params])
        owner = ctx.owners.get(self.NET_NAME)
        if key != self._uploaded_key or (owner is not None and owner() is not self):
            # (re)upload: weights changed, or another module of this class loaded its own weights into the context since
            ctx.load_net(self.NET_NAME, self.state_dict())
            ctx.modules.add(self)
            ctx.owners[self.NET_NAME] = weakref.ref(self)
            self._uploaded_key = key
        return ctx

    def load_state_dict(self, state_dict: Dict[str, Tensor], strict: bool = True):
        self._uploaded_key = None
        return super().load_state_dict(state_dict, strict=strict)
