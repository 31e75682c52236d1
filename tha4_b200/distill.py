"""Distillation inner loops of the body and face students on the CUDA path -- replaces, as a unit, what the reference does in
`SirenMorpherTrainingProtocol03.run_training_iteration` (src/tha4/nn/siren/morpher/siren_morpher_protocols_03.py:178-214):

    teacher forward under no_grad (mode_07, :102-108)  ->  student forward (:125-135)  ->  SumLoss of four
    time-weighted L1 terms (siren_morpher_03_trainer.py:32-50,237-247)  ->  backward  ->  DDP gradient averaging
    (shion/core/training/distrib/distributed_training_states.py:184-187)  ->  Adam step (optimizer_factories.py:9-17).

One process per GPU; the only collective is ONE all-reduce per step on the flat fp32 gradient buffer (331 567
elements = 1.33 MB), issued through torch.distributed (NCCL on GPUs, gloo in CPU tests of the host logic)."""
from typing import Dict, List, Optional, Sequence

import torch
import torch.distributed as dist
from torch import Tensor

from tha4_b200._lib import Context
from tha4_b200.nn.siren.morpher.siren_morpher_03 import SirenMorpher03
from tha4_b200.poser.general_poser_02 import GeneralPoser02

LOSS_TERMS = ('full_blended', 'full_warped', 'full_grid_change', 'full_color_change')   # siren_morpher_03_trainer.py:26-30


def flatten_parameters(module: torch.nn.Module) -> Tensor:
    """Moves the module's parameters into ONE contiguous fp32 buffer (state_dict order) and rebinds every parameter as
    a view of it, so the CUDA step, the gradient all-reduce and Adam all work on a single flat tensor."""
    params = list(module.parameters())
    flat = torch.cat([p.detach().reshape(-1).float() for p in params]).contiguous()
    off = 0
    for p in params:
        n = p.numel()
        p.data = flat[off:off + n].view_as(p)
        off += n
    return flat


class BodyMorpherDistiller:
    def __init__(self, teacher: GeneralPoser02, student: SirenMorpher03, betas=(0.9, 0.999), eps: float = 1e-8,
                 process_group=None, distributed: bool = True):
        self.teacher = teacher
        self.student = student
        self.ctx: Context = teacher.get_context()
        teacher.get_modules()
        student.to(self.ctx.device)
        self.flat = flatten_parameters(student)
        assert self.flat.numel() == 331567
        self.grad = torch.zeros_like(self.flat)
        self.exp_avg = torch.zeros_like(self.flat)
        self.exp_avg_sq = torch.zeros_like(self.flat)
        self.betas, self.eps = betas, eps
        self.step_count = 0
        self.group = process_group
        self.world = dist.get_world_size(process_group) if (distributed and dist.is_available() and dist.is_initialized()) else 1

    def train_step(self, image: Tensor, pose: Tensor, loss_weights: Sequence[float], lr: float,
                   want_losses: bool = True) -> Optional[Dict[str, float]]:
        """One iteration on this rank's batch (image [b,4,512,512], pose [b,45]; b <= 8 in total across ranks in the
        reference, distiller_config.py:100-104)."""
        with torch.no_grad():
            t = self.teacher.get_posing_outputs(image, pose)            # 33 tensors; 0 posed, 2 warped, 3 grid_change, 5 input
            losses = self.ctx.siren_morpher_train_step(t[5], pose if pose.dim() == 2 else pose.unsqueeze(0), t[0], t[2], t[3],
                                                       loss_weights, self.flat, self.grad, want_losses)
            if self.world > 1:
                dist.all_reduce(self.grad, group=self.group)            # the path's single collective
            self.step_count += 1
            self.ctx.adam_step(self.flat, self.grad, self.exp_avg, self.exp_avg_sq, lr, self.step_count, self.betas, self.eps,
                               grad_scale=1.0 / self.world)
            self.student._uploaded_key = None                           # inference path must re-pack the new weights
        if not want_losses:
            return None
        out = dict(zip(LOSS_TERMS, losses))
        out['loss'] = sum(w * l for w, l in zip(loss_weights, losses))
        return out

    def reset(self, state_dict: Optional[Dict[str, Tensor]] = None):
        """Zeroes the optimiser state (and optionally reloads the student's weights) -- a fresh run on the same buffers."""
        if state_dict is not None:
            self.flat.copy_(torch.cat([state_dict[k].reshape(-1).float() for k in self.student.state_dict().keys()]).to(self.flat.device))
            self.student._uploaded_key = None
        self.exp_avg.zero_()
        self.exp_avg_sq.zero_()
        self.grad.zero_()
        self.step_count = 0

    def state_dict(self) -> Dict[str, Tensor]:
        return self.student.state_dict()


FACE_LOSS_TERMS = ('full', 'eye_mouth')          # siren_face_morpher_00_trainer.py:168-186 (weights 1.0 / 20.0)
FACE_LOSS_WEIGHTS = (1.0, 20.0)


def face_groundtruth_crop(posed_face: Tensor) -> Tensor:
    """transform_poser_posed_image_to_groundtruth (siren_face_morpher_00_trainer.py:123-126): the 128x128 window centred
    at (96, 112) of the teacher's 192x192 face image."""
    return posed_face[:, :, 112 - 64:112 + 64, 96 - 64:96 + 64].contiguous()


class FaceMorpherDistiller:
    """Inner loop of the face student -- replaces SirenFaceMorpherComputationProtocol00 + SirenMorpherTrainingProtocol03
    for KEY_MODULE = SirenFaceMorpher00 (siren_face_morpher_protocols_00.py:48-105): teacher = the mode_12 poser (face
    networks only, get_poser at siren_face_morpher_00_trainer.py:23-26), student input pose[:, 0:39], losses L1 + 20 x
    eye/mouth-masked L1, one flat-gradient all-reduce, Adam."""

    def __init__(self, teacher: GeneralPoser02, student, betas=(0.9, 0.999), eps: float = 1e-8, process_group=None,
                 distributed: bool = True):
        self.teacher = teacher
        self.student = student
        self.ctx: Context = teacher.get_context()
        teacher.get_modules()
        student.to(self.ctx.device)
        self.flat = flatten_parameters(student)
        assert self.flat.numel() == 121476
        self.grad = torch.zeros_like(self.flat)
        self.exp_avg = torch.zeros_like(self.flat)
        self.exp_avg_sq = torch.zeros_like(self.flat)
        self.betas, self.eps = betas, eps
        self.step_count = 0
        self.group = process_group
        self.world = dist.get_world_size(process_group) if (distributed and dist.is_available() and dist.is_initialized()) else 1

    def train_step(self, image: Tensor, pose: Tensor, eye_mouth_mask: Tensor, lr: float,
                   loss_weights: Sequence[float] = FACE_LOSS_WEIGHTS, want_losses: bool = True) -> Optional[Dict[str, float]]:
        """image [b,4,512,512], pose [b,45], eye_mouth_mask [b,4,128,128] (get_face_mask_image, :84-97)."""
        with torch.no_grad():
            t = self.teacher.get_posing_outputs(image, pose)            # mode_12: output 0 = posed face [b,4,192,192]
            target = face_groundtruth_crop(t[0])
            pose2 = pose if pose.dim() == 2 else pose.unsqueeze(0)
            losses = self.ctx.siren_face_morpher_train_step(pose2, target, eye_mouth_mask, loss_weights, self.flat, self.grad, want_losses)
            if self.world > 1:
                dist.all_reduce(self.grad, group=self.group)
            self.step_count += 1
            self.ctx.adam_step(self.flat, self.grad, self.exp_avg, self.exp_avg_sq, lr, self.step_count, self.betas, self.eps,
                               grad_scale=1.0 / self.world)
            self.student._uploaded_key = None
        if not want_losses:
            return None
        out = dict(zip(FACE_LOSS_TERMS, losses))
        out['loss'] = sum(w * l for w, l in zip(loss_weights, losses))
        return out

    def reset(self, state_dict: Optional[Dict[str, Tensor]] = None):
        """Zeroes the optimiser state (and optionally reloads the student's weights) -- a fresh run on the same buffers."""
        if state_dict is not None:
            self.flat.copy_(torch.cat([state_dict[k].reshape(-1).float() for k in self.student.state_dict().keys()]).to(self.flat.device))
            self.student._uploaded_key = None
        self.exp_avg.zero_()
        self.exp_avg_sq.zero_()
        self.grad.zero_()
        self.step_count = 0

    def state_dict(self) -> Dict[str, Tensor]:
        return self.student.state_dict()
