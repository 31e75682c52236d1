"""Upscaler02 -- mirror of src/tha4/nn/upscaler/upscaler_02.py:37-102 (hyper-parameters of mode_07.py:241-269).

`forward` keeps the reference signature (rest_image, coarse_posed_image, coarse_grid_change, pose).  The coarse
inputs may be given at 512x512 (as the reference's caller does after `interpolate`, mode_07.py:114-115) or directly
at the body morpher's 256x256, in which case that bilinear x2 upsampling is fused into the prologue kernel.  The outputs
are differentiable w.r.t. all four inputs at either size (encdec_autograd.py)."""
from typing import List

import torch
from torch import Tensor

from tha4_b200.nn.common import encdec_autograd
from tha4_b200.nn.common.native_module import NativeModule, wants_autograd
from tha4_b200.nn.state_dict_spec import upscaler_spec


class Upscaler02(NativeModule):
    NET_NAME = 'upscaler'

    def __init__(self, args=None):
        super().__init__(upscaler_spec())
        self.args = args

    def forward(self, rest_image: torch.Tensor, coarse_posed_image: torch.Tensor, coarse_grid_change: torch.Tensor,
                pose: torch.Tensor) -> List[Tensor]:
        assert len(rest_image.shape) == 4 and rest_image.shape[1:] == (4, 512, 512)       # upscaler_02.py:53-74
        assert coarse_posed_image.shape[0] == pose.shape[0] and coarse_grid_change.shape[1] == 2
        assert pose.shape[1] == 6
        if wants_autograd(rest_image, coarse_posed_image, coarse_grid_change, pose):
            return encdec_autograd.upscaler(self, rest_image, coarse_posed_image, coarse_grid_change, pose)
        return self.sync_weights().upscaler(rest_image, coarse_posed_image, coarse_grid_change, pose)

    INDEX_MERGED = 0
    INDEX_ALPHA = 1
    INDEX_WARPED = 2
    INDEX_GRID_CHANGE = 3
    INDEX_DIRECT = 4
