"""torch.autograd for the two SIREN students: `loss.backward()` through SirenMorpher03 / SirenFaceMorpher00 yields the
parameter gradients, as it does for the reference modules (siren_morpher_protocols_03.py:125-135,178-214;
siren_face_morpher_protocols_00.py:72-105), so a custom loss, optimizer or training loop -- DDP included -- works.

Forward: the inference kernels (fp16 operands, fp32 accumulate); the values are bit-identical to the no-grad path.
Backward: tha4_siren_{morpher,face_morpher}_backward recomputes the forward with TF32 products, as the fused distillation
step does, and runs the distillation step's backward from the upstream gradients.  The gradient is therefore that of the
TF32 forward at the same weights (DESIGN.md section 4).  Gradients w.r.t. image or pose and double backward are refused."""
from typing import List, Sequence, Tuple

import torch
from torch import Tensor
from torch.autograd.function import once_differentiable

from tha4_b200._lib import Tha4Error


def wants_autograd(module) -> bool:
    """The autograd path runs when grad mode is on and any parameter requires grad; otherwise the plain forward."""
    return torch.is_grad_enabled() and any(p.requires_grad for p in module._params())


def _refuse_input_grads(module, **inputs):
    for name, t in inputs.items():
        if t.requires_grad:
            raise Tha4Error('%s: gradients w.r.t. `%s` are not supported (only the parameters are differentiable); '
                            'pass %s.detach()' % (type(module).__name__, name, name))


def _refuse_double_backward(module_name: str):
    if torch.is_grad_enabled():
        raise Tha4Error('%s: double backward (create_graph=True) is not supported' % module_name)


def flat_parameters(params: Sequence[Tensor]) -> Tensor:
    """The parameters as one flat fp32 buffer in state_dict order: the buffer itself when they are already consecutive
    views of one (distill.flatten_parameters), else a concatenated copy."""
    p0 = params[0]
    if all(p.dtype == torch.float32 and p.is_contiguous() for p in params):
        base, off = p0.untyped_storage().data_ptr(), p0.storage_offset()
        for p in params:
            if p.untyped_storage().data_ptr() != base or p.storage_offset() != off:
                break
            off += p.numel()
        else:
            return p0.detach().as_strided((off - p0.storage_offset(),), (1,), p0.storage_offset())
    return torch.cat([p.detach().reshape(-1).float() for p in params])


def _split_like(flat: Tensor, params: Sequence[Tensor]) -> Tuple[Tensor, ...]:
    out, off = [], 0
    for p in params:
        out.append(flat[off:off + p.numel()].view_as(p))
        off += p.numel()
    return tuple(out)


class _SirenMorpherFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, module, image: Tensor, pose: Tensor, *params: Tensor):
        lib = module.sync_weights()
        B = image.shape[0]
        # one allocation per output: autograd refuses in-place ops on outputs that are views created inside a Function
        outs = [torch.empty((B, c, s, s), dtype=torch.float32, device=lib.device) for c, s in lib.SIREN_MORPHER_SPECS]
        lib.siren_morpher_into(image, pose, outs)
        ctx.set_materialize_grads(False)
        ctx.lib = lib
        ctx.save_for_backward(image, pose, *params)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *grad_outputs):
        _refuse_double_backward('SirenMorpher03')
        return _siren_morpher_backward(ctx, *grad_outputs)


@once_differentiable
def _siren_morpher_backward(ctx, *grad_outputs):
    image, pose, *params = ctx.saved_tensors
    flat = flat_parameters(params)
    grads = torch.empty_like(flat)
    ctx.lib.siren_morpher_backward(image, pose, [None if g is None else g.contiguous() for g in grad_outputs], flat, grads)
    return (None, None, None) + _split_like(grads, params)


class _SirenFaceMorpherFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, module, pose: Tensor, *params: Tensor):
        lib = module.sync_weights()
        out = lib.siren_face_morpher(pose)
        ctx.set_materialize_grads(False)
        ctx.lib = lib
        ctx.save_for_backward(pose, *params)
        return out

    @staticmethod
    def backward(ctx, grad_output):
        _refuse_double_backward('SirenFaceMorpher00')
        return _siren_face_morpher_backward(ctx, grad_output)


@once_differentiable
def _siren_face_morpher_backward(ctx, grad_output):
    pose, *params = ctx.saved_tensors
    if grad_output is None:
        return (None, None) + (None,) * len(params)
    flat = flat_parameters(params)
    grads = torch.empty_like(flat)
    ctx.lib.siren_face_morpher_backward(pose, grad_output.contiguous(), flat, grads)
    return (None, None) + _split_like(grads, params)


def siren_morpher(module, image: Tensor, pose: Tensor) -> List[Tensor]:
    _refuse_input_grads(module, image=image, pose=pose)
    return list(_SirenMorpherFunction.apply(module, image, pose, *module.parameters()))


def siren_face_morpher(module, pose: Tensor) -> Tensor:
    _refuse_input_grads(module, pose=pose)
    return _SirenFaceMorpherFunction.apply(module, pose, *module.parameters())
