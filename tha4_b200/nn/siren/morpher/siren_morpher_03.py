"""SirenMorpher03 -- mirror of src/tha4/nn/siren/morpher/siren_morpher_03.py:42-145 (hyper-parameters of
mode_14.py:108-131: 3 levels 128/256/512 with 360/180/90 channels)."""
from typing import List

from torch import Tensor

from tha4_b200.nn.common.native_module import NativeModule, wants_autograd
from tha4_b200.nn.siren import student_autograd
from tha4_b200.nn.state_dict_spec import siren_morpher_03_spec


class SirenMorpher03(NativeModule):
    NET_NAME = 'siren_body_morpher'

    def __init__(self, args=None):
        super().__init__(siren_morpher_03_spec())
        self.args = args

    def forward(self, image: Tensor, pose: Tensor) -> List[Tensor]:
        if wants_autograd(image, pose, *self._params()):     # loss.backward() reaches the parameters, or image / pose
            return student_autograd.siren_morpher(self, image, pose)
        return self.sync_weights().siren_morpher(image, pose)

    INDEX_BLENDED_IMAGE = 0
    INDEX_ALPHA = 1
    INDEX_COLOR_CHANGE = 2
    INDEX_WARPED_IMAGE = 3
    INDEX_GRID_CHANGE = 4
