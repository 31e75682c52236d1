"""CPU oracle of the SIREN students' parameter gradients for given upstream gradients (autograd on the functional
restatement in oracle/tha4_oracle.py) -- what `loss.backward()` through the reference modules produces, for any loss."""
from typing import Dict, Optional, Sequence

import torch
from torch import Tensor

from oracle import tha4_oracle as O


def _flat_grads(sd: Dict[str, Tensor], keys) -> Tensor:
    return torch.cat([(sd[k].grad if sd[k].grad is not None else torch.zeros_like(sd[k])).reshape(-1) for k in keys])


def body_param_grads(student_sd: Dict[str, Tensor], image: Tensor, pose: Tensor,
                     grad_outputs: Sequence[Optional[Tensor]]) -> Tensor:
    """Flat dL/d params (state_dict order) of SirenMorpher03 for upstream gradients of (blended, alpha, color_change,
    warped, grid_change); None = zero."""
    sd = {k: v.detach().clone().requires_grad_(True) for k, v in student_sd.items()}
    outs = O.siren_morpher_03(sd, image, pose)
    pairs = [(o, g) for o, g in zip(outs, grad_outputs) if g is not None]
    torch.autograd.backward([o for o, _ in pairs], [g for _, g in pairs])
    return _flat_grads(sd, student_sd.keys())


def face_param_grads(student_sd: Dict[str, Tensor], pose: Tensor, grad_output: Tensor) -> Tensor:
    """Flat dL/d params of SirenFaceMorpher00 (input pose[:, 0:39]) for the upstream gradient of its output."""
    sd = {k: v.detach().clone().requires_grad_(True) for k, v in student_sd.items()}
    out = O.siren_face_morpher(sd, pose[:, 0:39])
    out.backward(grad_output)
    return _flat_grads(sd, student_sd.keys())


def body_l1_upstream(outs: Sequence[Tensor], t_posed: Tensor, t_warped: Tensor, t_grid: Tensor, weights: Sequence[float]):
    """Upstream gradients of the distillation loss sum_i w_i mean|term_i| (siren_morpher_03_trainer.py:32-50) w.r.t. the five
    outputs: w sign(o - t) / numel for blended, warped, grid_change and color_change; alpha gets none."""
    blended, _, color, warped, grid = outs
    return [weights[0] * torch.sign(blended - t_posed) / blended.numel(), None,
            weights[3] * torch.sign(color - t_posed) / color.numel(),
            weights[1] * torch.sign(warped - t_warped) / warped.numel(),
            weights[2] * torch.sign(grid - t_grid) / grid.numel()]
