"""EyebrowMorphingCombiner00 -- mirror of src/tha4/nn/eyebrow_morphing_combiner/eyebrow_morphing_combiner_00.py:37-82
(hyper-parameters of mode_07.py:158-177)."""
from typing import List

from torch import Tensor

from tha4_b200.nn.common import encdec_autograd
from tha4_b200.nn.common.native_module import NativeModule
from tha4_b200.nn.state_dict_spec import eyebrow_morphing_combiner_spec


class EyebrowMorphingCombiner00(encdec_autograd.Trainable, NativeModule):
    NET_NAME = 'eyebrow_morphing_combiner'
    CTX_FORWARD, CTX_BACKWARD = 'eyebrow_morphing_combiner', 'eyebrow_morphing_combiner_backward'
    INPUT_GRADS = ('d_background_layer', 'd_eyebrow_layer', 'd_pose')

    def __init__(self, args=None):
        super().__init__(eyebrow_morphing_combiner_spec())
        self.args = args

    def forward(self, background_layer: Tensor, eyebrow_layer: Tensor, pose: Tensor, *args) -> List[Tensor]:
        return self.run_net(background_layer, eyebrow_layer, pose)

    EYEBROW_IMAGE_INDEX = 0
    COMBINE_ALPHA_INDEX = 1
    EYEBROW_IMAGE_NO_COMBINE_ALPHA_INDEX = 2
    MORPHED_EYEBROW_LAYER_INDEX = 3
    MORPHED_EYEBROW_LAYER_ALPHA_INDEX = 4
    MORPHED_EYEBROW_LAYER_COLOR_CHANGE_INDEX = 5
    WARPED_EYEBROW_LAYER_INDEX = 6
    MORPHED_EYEBROW_LAYER_GRID_CHANGE_INDEX = 7
    OUTPUT_LENGTH = 8
