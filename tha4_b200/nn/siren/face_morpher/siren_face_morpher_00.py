"""SirenFaceMorpher00 -- mirror of src/tha4/nn/siren/face_morpher/siren_face_morpher_00.py:28-51 (hyper-parameters of
mode_14.py:93-105: pose 39 + xy -> 8 sine layers of 128 -> 4 channels at 128x128)."""
from typing import Optional

from torch import Tensor

from tha4_b200.nn.common.native_module import NativeModule, wants_autograd
from tha4_b200.nn.siren import student_autograd
from tha4_b200.nn.state_dict_spec import siren_face_morpher_spec


class SirenFaceMorpher00(NativeModule):
    NET_NAME = 'siren_face_morpher'

    def __init__(self, args=None):
        super().__init__(siren_face_morpher_spec())
        self.args = args

    def forward(self, pose: Tensor, position: Optional[Tensor] = None) -> Tensor:
        assert position is None, 'only the default affine_grid position image (siren_face_morpher_00.py:38-44) is supported'
        if wants_autograd(pose, *self._params()):            # loss.backward() reaches the parameters, or the pose
            return student_autograd.siren_face_morpher(self, pose)
        return self.sync_weights().siren_face_morpher(pose)
