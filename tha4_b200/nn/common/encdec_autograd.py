"""torch.autograd for the three encoder-decoder teacher networks (EyebrowDecomposer00, EyebrowMorphingCombiner00,
FaceMorpher08) and the two U-Nets (Morpher00, Upscaler02): their outputs are differentiable w.r.t. images, layers and pose, as
the reference modules are (eyebrow_decomposer_00.py:46-64, eyebrow_morphing_combiner_00.py:47-72, face_morpher_08.py:158-193,
morpher_00.py:42-66, upscaler_02.py:59-96).  This is what pose fitting on an arbitrary character (expression and body parameters), or training an
image -> pose regressor with a teacher as a differentiable renderer, needs.

Dispatch: the autograd path runs when grad mode is on and an input (image, layer or pose) requires grad, or when the module
was made trainable (`module.trainable_(True)`) and any of its parameters requires grad; in every other case the forward is
the plain inference call.  Trainability is an explicit opt-in, not the students' "any parameter requires grad" rule,
because a freshly built teacher's parameters require grad (as every nn.Module's do) and its inference calls must stay plain
calls without a graph.  A trainable module's backward returns the gradients of the parameters that require grad (flat
d_params from the same library call as the input gradients).

Forward: the inference call; the outputs are bit-identical to the no-grad path (each in its own allocation, so in-place ops
on them work).  Inputs and parameters are saved, so an in-place write to either between forward and backward raises torch's
usual error.  Backward: tha4_*_backward recomputes the forward in the context's precision mode and returns only the input
gradients autograd asks for (DESIGN.md section 4).  Double backward is refused."""
from typing import List, Sequence

import torch
from torch import Tensor
from torch.autograd.function import once_differentiable

from tha4_b200.nn.common.native_module import contiguous_grads, refuse_double_backward


class Trainable:
    """Opt-in parameter gradients of the teacher modules (mixed into EyebrowDecomposer00, EyebrowMorphingCombiner00,
    FaceMorpher08, Morpher00, Upscaler02), and the dispatch of their forward.  Each module names its library calls once:
    CTX_FORWARD / CTX_BACKWARD are its Context forward and backward methods, INPUT_GRADS the backward's keyword for the
    gradient of each forward input, in input order."""
    CTX_FORWARD = ''
    CTX_BACKWARD = ''
    INPUT_GRADS = ()
    _trainable = False

    def trainable_(self, mode: bool = True):
        """Makes loss.backward() fill the .grad of this module's parameters that require grad; returns the module."""
        self._trainable = bool(mode)
        return self

    def is_trainable(self) -> bool:
        return self._trainable

    def wants_autograd(self, *inputs: Tensor) -> bool:
        if not torch.is_grad_enabled():
            return False
        return any(t.requires_grad for t in inputs) or (self._trainable and any(p.requires_grad for p in self._params()))

    def run_net(self, *inputs: Tensor) -> List[Tensor]:
        """The network's outputs for its forward inputs: through _TeacherFunction when autograd needs a graph, otherwise the
        plain library call."""
        if self.wants_autograd(*inputs):
            return list(_TeacherFunction.apply(self, *inputs, *self._params()))
        return getattr(self.sync_weights(), self.CTX_FORWARD)(*inputs)


def _param_grads(ctx, first: int, device):
    """(flat d_params buffer or None, per-parameter gradient views or None) for the parameter slots that start at
    needs_input_grad[first]: the views are in _params() order, which is state_dict order."""
    need = ctx.needs_input_grad[first:]
    module = ctx.module
    if not (module.is_trainable() and any(need)):      # a module that is not trainable keeps its parameters' .grad untouched
        return None, (None,) * len(need)
    params = module._params()
    if not getattr(module, '_param_order_checked', False):
        assert [k for k, _ in module.named_parameters()] == list(module.state_dict().keys()), 'parameters are not in state_dict order'
        module._param_order_checked = True
    flat = torch.empty((ctx.lib.param_count(module.NET_NAME),), dtype=torch.float32, device=device)
    views, off = [], 0
    for p, w in zip(params, need):
        n = p.numel()
        views.append(flat[off:off + n].view_as(p) if w else None)
        off += n
    assert off == flat.numel(), (off, flat.numel())
    return flat, tuple(views)


def _own(outs: Sequence[Tensor]):
    # one allocation per output: autograd refuses in-place ops on outputs that are views created inside a Function
    return tuple(o.clone() for o in outs)


def _empty_like(t: Tensor) -> Tensor:
    return torch.empty(t.shape, dtype=torch.float32, device=t.device)


class _TeacherFunction(torch.autograd.Function):
    """apply(module, *inputs, *params): the module's forward inputs (len(module.INPUT_GRADS) of them), then its _params()."""

    @staticmethod
    def forward(ctx, module, *tensors: Tensor):
        inputs = tensors[:len(module.INPUT_GRADS)]
        outs = getattr(module.sync_weights(), module.CTX_FORWARD)(*inputs)
        ctx.set_materialize_grads(False)
        ctx.module = module
        ctx.save_for_backward(*tensors)
        return _own(outs)

    @staticmethod
    def backward(ctx, *grad_outputs):
        refuse_double_backward(type(ctx.module).__name__)
        return _teacher_backward(ctx, *grad_outputs)


@once_differentiable
def _teacher_backward(ctx, *grad_outputs):
    module = ctx.module
    saved = ctx.saved_tensors
    n = len(module.INPUT_GRADS)
    inputs, want = saved[:n], ctx.needs_input_grad[1:1 + n]
    nothing = (None,) * (1 + len(saved))
    if not any(ctx.needs_input_grad[1:]) or all(g is None for g in grad_outputs):
        return nothing
    ctx.lib = module.sync_weights()
    flat, dp = _param_grads(ctx, 1 + n, inputs[0].device)
    if flat is None and not any(want):
        return nothing
    d = [_empty_like(t) if w else None for t, w in zip(inputs, want)]
    grads = dict(zip(module.INPUT_GRADS, d))
    # d_params only from a trainable module: the plain one keeps the input-gradient call it always made
    if module.is_trainable():
        grads['d_params'] = flat
    getattr(ctx.lib, module.CTX_BACKWARD)(*inputs, contiguous_grads(grad_outputs), **grads)
    return (None, *d) + dp
