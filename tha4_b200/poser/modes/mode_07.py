"""The full five-network THA4 poser -- mirror of src/tha4/poser/modes/mode_07.py (the reference's `create_poser`,
`Network`/`Branch` enums and `FiveStepPoserComputationProtocol`, incl. the eyebrow-decomposer cache of :56-68).

The reference evaluates a memoised Python DAG that dispatches ~1 600 PyTorch ops per frame; here the whole DAG of
mode_07.py:72-132 (crops, pastes, bilinear resizes and the five networks) is one C call,
`tha4_teacher_forward(mode=7)`, which returns the same 33 tensors in the same order.  When grad mode is on and the image or
the pose requires grad, the five modules are composed instead, each differentiable (all 45 pose parameters can be fitted).
"""
from enum import Enum
from typing import Dict, List, Optional

import torch
from torch import Tensor

from tha4_b200.nn.eyebrow_decomposer.eyebrow_decomposer_00 import EyebrowDecomposer00
from tha4_b200.nn.eyebrow_morphing_combiner.eyebrow_morphing_combiner_00 import EyebrowMorphingCombiner00
from tha4_b200.nn.face_morpher.face_morpher_08 import FaceMorpher08
from tha4_b200.nn.morpher.morpher_00 import Morpher00
from tha4_b200.nn.upscaler.upscaler_02 import Upscaler02
from tha4_b200.poser.general_poser_02 import GeneralPoser02
from tha4_b200.poser.modes.pose_parameters import get_pose_parameters
from tha4_b200.shion.core.cached_computation import CachedComputationProtocol, ComputationState
from tha4_b200.shion.core.load_save import torch_load


class Network(Enum):   # mode_07.py:20-29
    eyebrow_decomposer = 1
    eyebrow_morphing_combiner = 2
    face_morpher = 3
    body_morpher = 4
    upscaler = 5

    @property
    def outputs_key(self):
        return f"{self.name}_outputs"


class Branch(Enum):   # mode_07.py:32-35
    face_morphed_half = 1
    face_morphed_full = 2
    all_outputs = 3


NUM_EYEBROW_PARAMS = 12
NUM_FACE_PARAMS = 27
NUM_ROTATION_PARAMS = 6

# slices of the 33-tensor output list (mode_07.py:126-131)
_SLICES = {
    Network.upscaler.outputs_key: slice(0, 5),
    Branch.face_morphed_full.name: slice(5, 6),
    Network.body_morpher.outputs_key: slice(6, 11),
    Network.face_morpher.outputs_key: slice(11, 19),
    Network.eyebrow_morphing_combiner.outputs_key: slice(19, 27),
    Network.eyebrow_decomposer.outputs_key: slice(27, 33),
}


class FiveStepPoserComputationProtocol(CachedComputationProtocol):
    TEACHER_MODE = 7
    SLICES = _SLICES

    def __init__(self, eyebrow_morphed_image_index: int):
        super().__init__()
        self.eyebrow_morphed_image_index = eyebrow_morphed_image_index
        self.cached_batch_0 = None
        self.cached_eyebrow_decomposer_output = None
        self.cached_epoch = None
        self.cached_batch_size = None
        # The reference compares the image with the cached one on every call (mode_07.py:56-61, a reduction + host sync).
        # trust_image_identity = True skips that comparison when the caller passes the very same tensor object with an
        # unchanged version counter; writes that bypass the counter (`.data`, raw CUDA writes) are then NOT seen, so it is
        # opt-in for callers that own the image tensor (the puppeteer apps and bench.py's device-resident loop do).
        self.trust_image_identity = False

    def compute_func(self):
        def func(state: ComputationState) -> List[Tensor]:
            image, pose = state.batch[0], state.batch[1]
            if torch.is_grad_enabled() and (image.requires_grad or pose.requires_grad):
                return self._differentiable(state)
            return self._single_call(state)

        return func

    def _single_call(self, state: ComputationState) -> List[Tensor]:
        ctx = state.context
        image = state.batch[0]
        # eyebrow cache (mode_07.py:56-68): recompute the decomposer iff there is no cache, the batch size changed
        # or the image differs anywhere.  The comparison is skipped when the caller passes the very same, unmodified
        # tensor object; otherwise it is one reduction kernel + the same host sync the reference pays for .item().
        for net in Network:
            if net.name in state.modules:
                state.modules[net.name].sync_weights()
        new_batch_0, key_image = self.eyebrow_cache_miss(ctx, image)
        cached = None if new_batch_0 else self.cached_eyebrow_decomposer_output
        output = ctx.teacher_forward(self.TEACHER_MODE, image, state.batch[1], self.eyebrow_morphed_image_index, cached)
        self._store(state, output)
        if new_batch_0:
            self.eyebrow_cache_store(ctx, image, key_image, output[self.SLICES[Network.eyebrow_decomposer.outputs_key]])
        return output

    def _store(self, state: ComputationState, output: List[Tensor]):
        for key, sl in self.SLICES.items():
            state.outputs[key] = output[sl]
        state.outputs[Branch.all_outputs.name] = output

    def _differentiable(self, state: ComputationState) -> List[Tensor]:
        """The modules composed as in the reference (mode_07.py:72-132; mode_12.py:66-94 for the face part), each through its
        autograd.Function, when the image or the pose requires grad.  The eyebrow cache is used only when the image does not
        require grad: its outputs are then constants."""
        ctx = state.context
        image, pose = state.batch[0], state.batch[1]
        modules = state.modules
        decomposer = modules[Network.eyebrow_decomposer.name]
        if image.requires_grad:
            dec = decomposer(image[:, :, 64:192, 192:320])
        else:
            decomposer.sync_weights()
            miss, key_image = self.eyebrow_cache_miss(ctx, image)
            if miss:
                with torch.no_grad():
                    dec = decomposer(image[:, :, 64:192, 192:320])
                self.eyebrow_cache_store(ctx, image, key_image, dec)
            else:
                dec = self.cached_eyebrow_decomposer_output
        comb = modules[Network.eyebrow_morphing_combiner.name](dec[3], dec[0], pose[:, :NUM_EYEBROW_PARAMS])
        face_in = image[:, :, 32:224, 160:352].clone()
        face_in[:, :, 32:160, 32:160] = comb[self.eyebrow_morphed_image_index]
        n_face = NUM_EYEBROW_PARAMS + NUM_FACE_PARAMS
        face = modules[Network.face_morpher.name](face_in, pose[:, NUM_EYEBROW_PARAMS:n_face])
        output = self._body(state, face[0]) + list(face) + list(comb) + list(dec)
        self._store(state, output)
        return output

    def _body(self, state: ComputationState, face_morphed: Tensor) -> List[Tensor]:
        """upscaler(5) + face_morphed_full + body_morpher(5) of mode_07.py:93-124; the upscaler takes the body morpher's
        256x256 outputs and upsamples them itself, as the single call does."""
        image, pose = state.batch[0], state.batch[1]
        full = image.clone()
        full[:, :, 32:224, 160:352] = face_morphed
        # interpolate(size=256, bilinear, align_corners=False) of a 512x512 image is the mean of each 2x2 block; summed in the
        # order of the library's resize_bilinear, ((a + b) + (c + d)) / 4, it gives the single call's values exactly
        half = ((full[:, :, 0::2, 0::2] + full[:, :, 0::2, 1::2]) + (full[:, :, 1::2, 0::2] + full[:, :, 1::2, 1::2])) * 0.25
        rot = pose[:, NUM_EYEBROW_PARAMS + NUM_FACE_PARAMS:]
        body = state.modules[Network.body_morpher.name](half, rot)
        up = state.modules[Network.upscaler.name](full, body[Morpher00.INDEX_MERGED], body[Morpher00.INDEX_GRID_CHANGE], rot)
        return list(up) + [full] + list(body)

    def eyebrow_cache_miss(self, ctx, image: Tensor):
        """(True iff the cached decomposer outputs cannot be used for `image`, the tensor the cache is keyed by)."""
        # one image posed B times (image.expand(B, ...)) is compared through its single stored frame
        key_image = image[:1] if (image.shape[0] > 1 and image.stride(0) == 0) else image
        if (self.cached_batch_0 is None or image.shape[0] != self.cached_batch_size
                or key_image.shape != self.cached_batch_0.shape
                or self.cached_epoch != ctx.epoch):          # options / weights changed: cached outputs are stale
            return True, key_image
        if self.trust_image_identity and key_image is self.cached_batch_0 and key_image._version == self.cached_version:
            return False, key_image
        return ctx.images_differ(key_image, self.cached_batch_0), key_image

    def eyebrow_cache_store(self, ctx, image: Tensor, key_image: Tensor, decomposer_outputs: List[Tensor]):
        self.cached_batch_0 = key_image
        self.cached_batch_size = image.shape[0]
        self.cached_version = key_image._version
        self.cached_epoch = ctx.epoch
        self.cached_eyebrow_decomposer_output = decomposer_outputs

    def compute_output(self, key: str, state: ComputationState) -> List[Tensor]:
        if key in self.SLICES or key == Branch.all_outputs.name:
            self.compute_func()(state)
            return state.outputs[key]
        raise RuntimeError("Unsupported key: " + key)


def _loader(cls, file_name: Optional[str], state_dict):
    def load():
        module = cls()
        module.load_state_dict(state_dict if state_dict is not None else torch_load(file_name))
        return module

    return load


def load_eyebrow_decomposer(file_name: str):
    return _loader(EyebrowDecomposer00, file_name, None)()


def load_eyebrow_morphing_combiner(file_name: str):
    return _loader(EyebrowMorphingCombiner00, file_name, None)()


def load_face_morpher(file_name: str):
    return _loader(FaceMorpher08, file_name, None)()


def load_morpher_00(file_name: str):
    return _loader(Morpher00, file_name, None)()


def load_upscaler_02(file_name: str):
    return _loader(Upscaler02, file_name, None)()


_CLASSES = {
    Network.eyebrow_decomposer.name: EyebrowDecomposer00,
    Network.eyebrow_morphing_combiner.name: EyebrowMorphingCombiner00,
    Network.face_morpher.name: FaceMorpher08,
    Network.body_morpher.name: Morpher00,
    Network.upscaler.name: Upscaler02,
}


def create_poser(
        device: torch.device,
        module_file_names: Optional[Dict[str, str]] = None,
        eyebrow_morphed_image_index: int = EyebrowMorphingCombiner00.EYEBROW_IMAGE_NO_COMBINE_ALPHA_INDEX,
        default_output_index: int = 0,
        state_dicts: Optional[Dict[str, Dict[str, Tensor]]] = None) -> GeneralPoser02:
    """Same signature and defaults as the reference (mode_07.py:272-315); `state_dicts` additionally accepts
    in-memory reference-format state_dicts instead of files (the teacher weights are a separate download)."""
    if module_file_names is None:
        module_file_names = {}
    for net in Network:
        if net.name not in module_file_names:
            module_file_names[net.name] = "data/tha4/%s.pt" % net.name      # mode_07.py:279-293
    loaders = {
        name: _loader(cls, module_file_names[name], None if state_dicts is None else state_dicts[name])
        for name, cls in _CLASSES.items()
    }
    protocol = FiveStepPoserComputationProtocol(eyebrow_morphed_image_index)
    poser = GeneralPoser02(
        image_size=512,
        module_loaders=loaders,
        pose_parameters=get_pose_parameters().get_pose_parameter_groups(),
        output_list_func=protocol.compute_func(),
        subrect=None,
        device=device,
        output_length=5 + 1 + 5 + 8 + 8 + 6,
        default_output_index=default_output_index)
    poser.protocol = protocol          # not in the reference: gives callers access to `trust_image_identity`
    return poser
