"""The face-only teacher (eyebrow decomposer -> eyebrow morphing combiner -> face morpher) -- mirror of
src/tha4/poser/modes/mode_12.py:41-96,169-202.  Used as the face-distillation teacher
(siren_face_morpher_00_trainer.py:23-26).

Quirk kept from the reference: `get_output_length()` reports 18 (mode_12.py:201) while the returned list has
8 + 8 + 6 = 22 tensors (mode_12.py:88-94)."""
from enum import Enum
from typing import Dict, List, Optional

import torch
from torch import Tensor

from tha4_b200.nn.eyebrow_decomposer.eyebrow_decomposer_00 import EyebrowDecomposer00
from tha4_b200.nn.eyebrow_morphing_combiner.eyebrow_morphing_combiner_00 import EyebrowMorphingCombiner00
from tha4_b200.nn.face_morpher.face_morpher_08 import FaceMorpher08
from tha4_b200.poser.general_poser_02 import GeneralPoser02
from tha4_b200.poser.modes import mode_07
from tha4_b200.poser.modes.pose_parameters import get_pose_parameters
from tha4_b200.shion.core.cached_computation import ComputationState


class Network(Enum):
    eyebrow_decomposer = 1
    eyebrow_morphing_combiner = 2
    face_morpher = 3

    @property
    def outputs_key(self):
        return f"{self.name}_outputs"


class Branch(Enum):
    all_outputs = 3


class FiveStepPoserComputationProtocol(mode_07.FiveStepPoserComputationProtocol):   # (sic) same class name as mode_12.py:41
    TEACHER_MODE = 12
    SLICES = {
        Network.face_morpher.outputs_key: slice(0, 8),
        Network.eyebrow_morphing_combiner.outputs_key: slice(8, 16),
        Network.eyebrow_decomposer.outputs_key: slice(16, 22),
    }

    def compute_func(self):
        single_call = super().compute_func()

        def func(state: ComputationState) -> List[Tensor]:
            image, pose = state.batch[0], state.batch[1]
            if torch.is_grad_enabled() and (image.requires_grad or pose.requires_grad):
                return self._differentiable(state)
            return single_call(state)          # one tha4_teacher_forward call

        return func

    def _differentiable(self, state: ComputationState) -> List[Tensor]:
        """The three modules composed as in the reference (mode_12.py:66-94), each through its autograd.Function.  The eyebrow
        cache is used only when the image does not require grad: its outputs are then constants."""
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
        comb = modules[Network.eyebrow_morphing_combiner.name](dec[3], dec[0], pose[:, :mode_07.NUM_EYEBROW_PARAMS])
        face_in = image[:, :, 32:224, 160:352].clone()
        face_in[:, :, 32:160, 32:160] = comb[self.eyebrow_morphed_image_index]
        n_face = mode_07.NUM_EYEBROW_PARAMS + mode_07.NUM_FACE_PARAMS
        face = modules[Network.face_morpher.name](face_in, pose[:, mode_07.NUM_EYEBROW_PARAMS:n_face])
        output = list(face) + list(comb) + list(dec)
        for key, sl in self.SLICES.items():
            state.outputs[key] = output[sl]
        state.outputs[Branch.all_outputs.name] = output
        return output


_CLASSES = {
    Network.eyebrow_decomposer.name: EyebrowDecomposer00,
    Network.eyebrow_morphing_combiner.name: EyebrowMorphingCombiner00,
    Network.face_morpher.name: FaceMorpher08,
}


def create_poser(
        device: torch.device,
        module_file_names: Optional[Dict[str, str]] = None,
        eyebrow_morphed_image_index: int = EyebrowMorphingCombiner00.EYEBROW_IMAGE_NO_COMBINE_ALPHA_INDEX,
        default_output_index: int = 0,
        state_dicts: Optional[Dict[str, Dict[str, Tensor]]] = None) -> GeneralPoser02:
    if module_file_names is None:
        module_file_names = {}
    for net in Network:
        if net.name not in module_file_names:
            module_file_names[net.name] = "data/tha4/%s.pt" % net.name
    loaders = {
        name: mode_07._loader(cls, module_file_names[name], None if state_dicts is None else state_dicts[name])
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
        output_length=5 + 5 + 8,
        default_output_index=default_output_index)
    poser.protocol = protocol          # not in the reference: gives callers access to `trust_image_identity`
    return poser
