"""EyebrowDecomposer00 -- mirror of src/tha4/nn/eyebrow_decomposer/eyebrow_decomposer_00.py:36-72 (hyper-parameters of
mode_07.py:137-155: 128x128, 64 start channels, 16x16 bottleneck, 6 bottleneck blocks, InstanceNorm + ReLU)."""
from typing import List

from torch import Tensor

from tha4_b200.nn.common import encdec_autograd
from tha4_b200.nn.common.native_module import NativeModule
from tha4_b200.nn.state_dict_spec import eyebrow_decomposer_spec


class EyebrowDecomposer00(encdec_autograd.Trainable, NativeModule):
    NET_NAME = 'eyebrow_decomposer'
    CTX_FORWARD, CTX_BACKWARD = 'eyebrow_decomposer', 'eyebrow_decomposer_backward'
    INPUT_GRADS = ('d_image',)

    def __init__(self, args=None):
        super().__init__(eyebrow_decomposer_spec())
        self.args = args

    def forward(self, image: Tensor, *args) -> List[Tensor]:
        return self.run_net(image)

    EYEBROW_LAYER_INDEX = 0
    EYEBROW_LAYER_ALPHA_INDEX = 1
    EYEBROW_LAYER_COLOR_CHANGE_INDEX = 2
    BACKGROUND_LAYER_INDEX = 3
    BACKGROUND_LAYER_ALPHA_INDEX = 4
    BACKGROUND_LAYER_COLOR_CHANGE_INDEX = 5
    OUTPUT_LENGTH = 6
