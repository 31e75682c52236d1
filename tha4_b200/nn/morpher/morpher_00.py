"""Morpher00 (the body morpher U-Net) -- mirror of src/tha4/nn/morpher/morpher_00.py:35-72 (hyper-parameters of
mode_07.py:210-239)."""
from typing import List

import torch
from torch import Tensor

from tha4_b200.nn.common import encdec_autograd
from tha4_b200.nn.common.native_module import NativeModule
from tha4_b200.nn.state_dict_spec import body_morpher_spec


class Morpher00(encdec_autograd.Trainable, NativeModule):
    NET_NAME = 'body_morpher'
    CTX_FORWARD, CTX_BACKWARD = 'morpher', 'morpher_backward'
    INPUT_GRADS = ('d_image', 'd_pose')

    def __init__(self, args=None):
        super().__init__(body_morpher_spec())
        self.args = args

    def forward(self, image: torch.Tensor, pose: torch.Tensor) -> List[Tensor]:
        assert len(image.shape) == 4 and image.shape[1:] == (4, 256, 256)     # morpher_00.py:43-49
        assert len(pose.shape) == 2 and image.shape[0] == pose.shape[0] and pose.shape[1] == 6
        return self.run_net(image, pose)

    INDEX_MERGED = 0
    INDEX_ALPHA = 1
    INDEX_WARPED = 2
    INDEX_GRID_CHANGE = 3
    INDEX_DIRECT = 4
