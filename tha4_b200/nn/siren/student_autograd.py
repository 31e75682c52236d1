"""torch.autograd for the two SIREN students: `loss.backward()` through SirenMorpher03 / SirenFaceMorpher00 yields the
parameter gradients, as it does for the reference modules (siren_morpher_protocols_03.py:125-135,178-214;
siren_face_morpher_protocols_00.py:72-105), so a custom loss, optimizer or training loop -- DDP included -- works.
Frozen students (every parameter with requires_grad False) are differentiable w.r.t. image and pose instead, as the
reference modules are: pose fitting, or training an upstream network through the student with an image loss.

Dispatch: the autograd path runs when grad mode is on and a parameter or an input requires grad; in every other case the
forward is the plain inference call.  Gradients w.r.t. parameters and inputs together, and double backward, are refused.

Forward: the inference kernels (fp16 operands, fp32 accumulate); the values are bit-identical to the no-grad path.
Backward: one tha4_siren_{morpher,face_morpher}_backward call computes only the gradients autograd asks for.  The
parameter gradients and d(pose) recompute the forward with TF32 products, as the fused distillation step does, and run
the distillation step's backward from the upstream gradients; they are therefore those of the TF32 forward at the same
weights (DESIGN.md section 4).  d(image) is the exact adjoint of the warp the forward returned (from its grid_change /
alpha outputs, no recompute)."""
from typing import List, Sequence, Tuple

import torch
from torch import Tensor
from torch.autograd.function import once_differentiable

from tha4_b200._lib import Tha4Error
from tha4_b200.nn.common.native_module import contiguous_grads, refuse_double_backward


def _refuse_input_grads(module, **inputs):
    for name, t in inputs.items():
        if t.requires_grad:
            raise Tha4Error('%s: gradients w.r.t. `%s` are not supported while parameters require grad (freeze the module '
                            'with requires_grad_(False) for input gradients); pass %s.detach()' % (type(module).__name__, name, name))


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
        # d(image) is the adjoint of the returned warp: with an input requiring grad the returned alpha and grid_change are
        # saved (version-checked); with parameters requiring grad the outputs stay free for in-place ops
        ctx.saves_warp = ctx.needs_input_grad[1] or ctx.needs_input_grad[2]
        ctx.save_for_backward(image, pose, *params, *((outs[1], outs[4]) if ctx.saves_warp else ()))
        return tuple(outs)

    @staticmethod
    def backward(ctx, *grad_outputs):
        refuse_double_backward('SirenMorpher03')
        return _siren_morpher_backward(ctx, *grad_outputs)


@once_differentiable
def _siren_morpher_backward(ctx, *grad_outputs):
    image, pose, *params = ctx.saved_tensors
    alpha = grid_change = None
    if ctx.saves_warp:
        *params, alpha, grid_change = params
    want_params, want_image, want_pose = any(ctx.needs_input_grad[3:]), ctx.needs_input_grad[1], ctx.needs_input_grad[2]
    if not (want_params or want_image or want_pose):
        return (None, None, None) + (None,) * len(params)
    flat = flat_parameters(params) if want_params or want_pose else None
    grads = torch.empty_like(flat) if want_params else None
    B, dev = image.shape[0], ctx.lib.device
    d_image = torch.empty((B, 4, 512, 512), dtype=torch.float32, device=dev) if want_image else None
    d_pose = torch.empty((B, 45), dtype=torch.float32, device=dev) if want_pose else None
    ctx.lib.siren_morpher_backward(image, pose, contiguous_grads(grad_outputs), grid_change=grid_change, alpha=alpha,
                                   params=flat, grads=grads, d_image=d_image, d_pose=d_pose)
    return (None, d_image, d_pose) + (_split_like(grads, params) if grads is not None else (None,) * len(params))


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
        refuse_double_backward('SirenFaceMorpher00')
        return _siren_face_morpher_backward(ctx, grad_output)


@once_differentiable
def _siren_face_morpher_backward(ctx, grad_output):
    pose, *params = ctx.saved_tensors
    want_params, want_pose = any(ctx.needs_input_grad[2:]), ctx.needs_input_grad[1]
    if grad_output is None or not (want_params or want_pose):
        return (None, None) + (None,) * len(params)
    flat = flat_parameters(params)
    grads = torch.empty_like(flat) if want_params else None
    d_pose = torch.empty((pose.shape[0], 39), dtype=torch.float32, device=ctx.lib.device) if want_pose else None
    ctx.lib.siren_face_morpher_backward(pose, grad_output.contiguous(), flat, grads=grads, d_pose=d_pose)
    return (None, d_pose) + (_split_like(grads, params) if grads is not None else (None,) * len(params))


def siren_morpher(module, image: Tensor, pose: Tensor) -> List[Tensor]:
    if any(p.requires_grad for p in module._params()):
        _refuse_input_grads(module, image=image, pose=pose)
    return list(_SirenMorpherFunction.apply(module, image, pose, *module.parameters()))


def siren_face_morpher(module, pose: Tensor) -> Tensor:
    if any(p.requires_grad for p in module._params()):
        _refuse_input_grads(module, pose=pose)
    return _SirenFaceMorpherFunction.apply(module, pose, *module.parameters())
