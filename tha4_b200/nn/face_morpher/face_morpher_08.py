"""FaceMorpher08 -- mirror of src/tha4/nn/face_morpher/face_morpher_08.py:48-202 (hyper-parameters of
mode_07.py:180-207: 192x192, 27 expression parameters, 24x24 bottleneck, output_iris_mouth_grid_change=True)."""
from typing import List

from torch import Tensor

from tha4_b200.nn.common import encdec_autograd
from tha4_b200.nn.common.native_module import NativeModule
from tha4_b200.nn.state_dict_spec import face_morpher_spec


class FaceMorpher08(encdec_autograd.Trainable, NativeModule):
    NET_NAME = 'face_morpher'
    CTX_FORWARD, CTX_BACKWARD = 'face_morpher', 'face_morpher_backward'
    INPUT_GRADS = ('d_image', 'd_pose')

    def __init__(self, args=None):
        super().__init__(face_morpher_spec())
        self.args = args

    def forward(self, image: Tensor, pose: Tensor, *args) -> List[Tensor]:
        return self.run_net(image, pose)

    OUTPUT_IMAGE_INDEX = 0
    EYE_ALPHA_INDEX = 1
    EYE_COLOR_CHANGE_INDEX = 2
    IRIS_MOUTH_IMAGE_1_INDEX = 3
    IRIS_MOUTH_ALPHA_INDEX = 4
    IRIS_MOUTH_COLOR_CHANGE_INDEX = 5
    IRIS_MOUTH_IMAGE_0_INDEX = 6
    IRIS_MOUTH_GRID_CHANGE_INDEX = 7
