"""torch.autograd for the three encoder-decoder teacher networks (EyebrowDecomposer00, EyebrowMorphingCombiner00,
FaceMorpher08) and the body morpher U-Net (Morpher00): their outputs are differentiable w.r.t. image, layers and pose, as the
reference modules are (eyebrow_decomposer_00.py:46-64, eyebrow_morphing_combiner_00.py:47-72, face_morpher_08.py:158-193,
morpher_00.py:42-66).  This is what pose fitting on an arbitrary character (expression and body parameters), or training an
image -> pose regressor with a teacher as a differentiable renderer, needs.

Dispatch: the autograd path runs when grad mode is on and an input (image, layer or pose) requires grad; in every other
case the forward is the plain inference call.  Teacher parameters never receive gradients (there is no teacher training
here), and unlike the SIREN students the module does not have to be frozen first.

Forward: the inference call; the outputs are bit-identical to the no-grad path (each in its own allocation, so in-place ops
on them work).  Inputs and parameters are saved, so an in-place write to either between forward and backward raises torch's
usual error.  Backward: tha4_*_backward recomputes the forward in the context's precision mode and returns only the input
gradients autograd asks for (DESIGN.md section 4).  Double backward is refused."""
from typing import List, Sequence

import torch
from torch import Tensor
from torch.autograd.function import once_differentiable

from tha4_b200.nn.common.native_module import contiguous_grads, refuse_double_backward


def _own(outs: Sequence[Tensor]):
    # one allocation per output: autograd refuses in-place ops on outputs that are views created inside a Function
    return tuple(o.clone() for o in outs)


def _empty_like(t: Tensor) -> Tensor:
    return torch.empty(t.shape, dtype=torch.float32, device=t.device)


class _DecomposerFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, module, image: Tensor, *params: Tensor):
        outs = module.sync_weights().eyebrow_decomposer(image)
        ctx.set_materialize_grads(False)
        ctx.module = module
        ctx.save_for_backward(image, *params)
        return _own(outs)

    @staticmethod
    def backward(ctx, *grad_outputs):
        refuse_double_backward('EyebrowDecomposer00')
        return _decomposer_backward(ctx, *grad_outputs)


@once_differentiable
def _decomposer_backward(ctx, *grad_outputs):
    image, *params = ctx.saved_tensors
    none = (None,) * len(params)
    if not ctx.needs_input_grad[1] or all(g is None for g in grad_outputs):
        return (None, None) + none
    d_image = _empty_like(image)
    ctx.module.sync_weights().eyebrow_decomposer_backward(image, contiguous_grads(grad_outputs), d_image)
    return (None, d_image) + none


class _CombinerFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, module, background_layer: Tensor, eyebrow_layer: Tensor, pose: Tensor, *params: Tensor):
        outs = module.sync_weights().eyebrow_morphing_combiner(background_layer, eyebrow_layer, pose)
        ctx.set_materialize_grads(False)
        ctx.module = module
        ctx.save_for_backward(background_layer, eyebrow_layer, pose, *params)
        return _own(outs)

    @staticmethod
    def backward(ctx, *grad_outputs):
        refuse_double_backward('EyebrowMorphingCombiner00')
        return _combiner_backward(ctx, *grad_outputs)


@once_differentiable
def _combiner_backward(ctx, *grad_outputs):
    background_layer, eyebrow_layer, pose, *params = ctx.saved_tensors
    none = (None,) * len(params)
    want = ctx.needs_input_grad[1:4]
    if not any(want) or all(g is None for g in grad_outputs):
        return (None, None, None, None) + none
    d_bg = _empty_like(background_layer) if want[0] else None
    d_eb = _empty_like(eyebrow_layer) if want[1] else None
    d_pose = _empty_like(pose) if want[2] else None
    ctx.module.sync_weights().eyebrow_morphing_combiner_backward(background_layer, eyebrow_layer, pose, contiguous_grads(grad_outputs),
                                                                d_background_layer=d_bg, d_eyebrow_layer=d_eb, d_pose=d_pose)
    return (None, d_bg, d_eb, d_pose) + none


class _FaceMorpherFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, module, image: Tensor, pose: Tensor, *params: Tensor):
        outs = module.sync_weights().face_morpher(image, pose)
        ctx.set_materialize_grads(False)
        ctx.module = module
        ctx.save_for_backward(image, pose, *params)
        return _own(outs)

    @staticmethod
    def backward(ctx, *grad_outputs):
        refuse_double_backward('FaceMorpher08')
        return _face_morpher_backward(ctx, *grad_outputs)


@once_differentiable
def _face_morpher_backward(ctx, *grad_outputs):
    image, pose, *params = ctx.saved_tensors
    none = (None,) * len(params)
    want_image, want_pose = ctx.needs_input_grad[1], ctx.needs_input_grad[2]
    if not (want_image or want_pose) or all(g is None for g in grad_outputs):
        return (None, None, None) + none
    d_image = _empty_like(image) if want_image else None
    d_pose = _empty_like(pose) if want_pose else None
    ctx.module.sync_weights().face_morpher_backward(image, pose, contiguous_grads(grad_outputs), d_image=d_image, d_pose=d_pose)
    return (None, d_image, d_pose) + none


class _MorpherFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, module, image: Tensor, pose: Tensor, *params: Tensor):
        outs = module.sync_weights().morpher(image, pose)
        ctx.set_materialize_grads(False)
        ctx.module = module
        ctx.save_for_backward(image, pose, *params)
        return _own(outs)

    @staticmethod
    def backward(ctx, *grad_outputs):
        refuse_double_backward('Morpher00')
        return _morpher_backward(ctx, *grad_outputs)


@once_differentiable
def _morpher_backward(ctx, *grad_outputs):
    image, pose, *params = ctx.saved_tensors
    none = (None,) * len(params)
    want_image, want_pose = ctx.needs_input_grad[1], ctx.needs_input_grad[2]
    if not (want_image or want_pose) or all(g is None for g in grad_outputs):
        return (None, None, None) + none
    d_image = _empty_like(image) if want_image else None
    d_pose = _empty_like(pose) if want_pose else None
    ctx.module.sync_weights().morpher_backward(image, pose, contiguous_grads(grad_outputs), d_image=d_image, d_pose=d_pose)
    return (None, d_image, d_pose) + none


def eyebrow_decomposer(module, image: Tensor) -> List[Tensor]:
    return list(_DecomposerFunction.apply(module, image, *module._params()))


def eyebrow_morphing_combiner(module, background_layer: Tensor, eyebrow_layer: Tensor, pose: Tensor) -> List[Tensor]:
    return list(_CombinerFunction.apply(module, background_layer, eyebrow_layer, pose, *module._params()))


def face_morpher(module, image: Tensor, pose: Tensor) -> List[Tensor]:
    return list(_FaceMorpherFunction.apply(module, image, pose, *module._params()))


def morpher(module, image: Tensor, pose: Tensor) -> List[Tensor]:
    return list(_MorpherFunction.apply(module, image, pose, *module._params()))
