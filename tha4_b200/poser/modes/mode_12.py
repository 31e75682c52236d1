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

    def _body(self, state: ComputationState, face_morphed: Tensor) -> List[Tensor]:
        return []          # the face-only teacher stops after the face morpher (mode_12.py:88-94)


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
