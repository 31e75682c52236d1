"""CPU check of the upstream-gradient oracle the student autograd tests compare against: fed the L1 upstream gradients of
the distillation loss it must reproduce the distillation oracle's gradient (which tests/test_oracle_pinned.py pins to the
reference's own run_training_iteration)."""
import torch

import student_grad_oracle as SGO
from oracle import distill_oracle, make_golden_distill as M, tha4_oracle as O


def test_upstream_oracle_reproduces_distill_oracle(lambda00_sds):
    body, _ = M.distill_inputs()
    sd = lambda00_sds['body_morpher']
    _, ref = distill_oracle.body_losses_and_grads(sd, body['image'], body['pose'], body['t_posed'], body['t_warped'], body['t_grid'],
                                                  M.BODY_WEIGHTS)
    with torch.no_grad():
        outs = O.siren_morpher_03(sd, body['image'], body['pose'])
    ups = SGO.body_l1_upstream(outs, body['t_posed'], body['t_warped'], body['t_grid'], M.BODY_WEIGHTS)
    g = SGO.body_param_grads(sd, body['image'], body['pose'], ups)
    assert g.shape == ref.shape
    assert ((g - ref).norm() / ref.norm()).item() <= 1e-5
    assert (g - ref).abs().max().item() <= 1e-5 * ref.abs().max().item()


def test_face_upstream_oracle_reproduces_distill_oracle(lambda00_sds):
    from tha4_b200.distill import FACE_LOSS_WEIGHTS, face_groundtruth_crop
    _, face = M.distill_inputs()
    sd = lambda00_sds['face_morpher']
    target = face_groundtruth_crop(face['posed_face'])
    _, ref = distill_oracle.face_losses_and_grads(sd, face['pose'], target, face['mask'], FACE_LOSS_WEIGHTS)
    with torch.no_grad():
        out = O.siren_face_morpher(sd, face['pose'][:, 0:39])
    d = out - target
    n = d.numel()
    up = FACE_LOSS_WEIGHTS[0] * torch.sign(d) / n + FACE_LOSS_WEIGHTS[1] * torch.sign(d * face['mask']) * face['mask'] / n
    g = SGO.face_param_grads(sd, face['pose'], up)
    assert ((g - ref).norm() / ref.norm()).item() <= 1e-5
