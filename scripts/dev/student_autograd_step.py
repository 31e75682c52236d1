"""Developer timing of one training iteration of the SIREN students (not a pytest file), device time between CUDA events:

  fused     *Distiller.train_step: teacher forward, then forward + L1 terms + backward + Adam in the library on flat buffers
  autograd  teacher forward under no_grad, then the student module forward, the same L1 terms in PyTorch, loss.backward()
            (tha4_siren_*_backward with the parameter gradients requested) and torch.optim.Adam over module.parameters()
  teacher   the teacher forward alone (part of both iterations above)

for the body student (mode_07 teacher) and the face student (mode_12 teacher) at B = 1 and 8.  Also prints the kernel launches
of one fused library train step.  Usage: python scripts/dev/student_autograd_step.py [--steps N] [--warmup W]"""
import argparse
import json
import os
import sys

import torch

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, _ROOT)
from tha4_b200 import synthetic  # noqa: E402
from tha4_b200.distill import (BodyMorpherDistiller, FaceMorpherDistiller, FACE_LOSS_WEIGHTS,  # noqa: E402
                               face_groundtruth_crop)
from tha4_b200.poser.modes import mode_07, mode_12, mode_14  # noqa: E402

DEV = torch.device('cuda:0')
BODY_W = [1.0, 0.5, 2.0, 0.25]
LR = 1e-4


def device_ms(fn, warmup, steps):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def body(B, tsds, ssds, warmup, steps):
    teacher = mode_07.create_poser(DEV, state_dicts=tsds)
    image = synthetic.synthetic_image(0, B).to(DEV)
    pose = synthetic.random_poses(B, seed=5).to(DEV)
    d = BodyMorpherDistiller(teacher, mode_14.load_body_morpher(None, ssds['body_morpher']))
    ctx = teacher.get_context()
    with torch.no_grad():
        t = teacher.get_posing_outputs(image, pose)
    l0 = ctx.counter('kernel_launches')
    ctx.siren_morpher_train_step(t[5], pose, t[0], t[2], t[3], BODY_W, d.flat, d.grad, want_losses=False)
    launches = ctx.counter('kernel_launches') - l0
    fused = device_ms(lambda: d.train_step(image, pose, BODY_W, LR, want_losses=False), warmup, steps)

    student = mode_14.load_body_morpher(None, ssds['body_morpher']).to(DEV)
    student.attach_context(ctx)
    opt = torch.optim.Adam(student.parameters(), lr=LR)

    def autograd_iter():
        with torch.no_grad():
            t = teacher.get_posing_outputs(image, pose)
        o = student(t[5], pose)
        terms = [(o[0] - t[0]).abs().mean(), (o[3] - t[2]).abs().mean(), (o[4] - t[3]).abs().mean(), (o[2] - t[0]).abs().mean()]
        loss = sum(w * x for w, x in zip(BODY_W, terms))
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()

    def teacher_only():
        with torch.no_grad():
            teacher.get_posing_outputs(image, pose)

    auto = device_ms(autograd_iter, warmup, steps)
    teach = device_ms(teacher_only, warmup, steps)
    return dict(student='body', B=B, fused_ms=fused, autograd_ms=auto, teacher_ms=teach, train_step_launches=launches)


def face(B, tsds, ssds, warmup, steps):
    teacher = mode_12.create_poser(DEV, state_dicts=tsds)
    image = synthetic.synthetic_image(0, B).to(DEV)
    pose = synthetic.random_poses(B, seed=5).to(DEV)
    mask = torch.zeros(B, 4, 128, 128, device=DEV)
    mask[:, :, 40:90, 30:100] = 1.0
    d = FaceMorpherDistiller(teacher, mode_14.load_face_morpher(None, ssds['face_morpher']))
    ctx = teacher.get_context()
    with torch.no_grad():
        target = face_groundtruth_crop(teacher.get_posing_outputs(image, pose)[0])
    l0 = ctx.counter('kernel_launches')
    ctx.siren_face_morpher_train_step(pose, target, mask, FACE_LOSS_WEIGHTS, d.flat, d.grad, want_losses=False)
    launches = ctx.counter('kernel_launches') - l0
    fused = device_ms(lambda: d.train_step(image, pose, mask, LR, want_losses=False), warmup, steps)

    student = mode_14.load_face_morpher(None, ssds['face_morpher']).to(DEV)
    student.attach_context(ctx)
    opt = torch.optim.Adam(student.parameters(), lr=LR)
    pose39 = pose[:, :39].contiguous()

    def autograd_iter():
        with torch.no_grad():
            target = face_groundtruth_crop(teacher.get_posing_outputs(image, pose)[0])
        o = student(pose39)
        loss = FACE_LOSS_WEIGHTS[0] * (target - o).abs().mean() + FACE_LOSS_WEIGHTS[1] * ((target - o) * mask).abs().mean()
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()

    def teacher_only():
        with torch.no_grad():
            face_groundtruth_crop(teacher.get_posing_outputs(image, pose)[0])

    auto = device_ms(autograd_iter, warmup, steps)
    teach = device_ms(teacher_only, warmup, steps)
    return dict(student='face', B=B, fused_ms=fused, autograd_ms=auto, teacher_ms=teach, train_step_launches=launches)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    tsds, ssds = synthetic.teacher_state_dicts(0), synthetic.student_state_dicts(0)
    print(json.dumps({'gpu': torch.cuda.get_device_name(0)}), flush=True)
    for fn in (body, face):
        for B in (1, 8):
            r = fn(B, tsds, ssds, args.warmup, args.steps)
            r['autograd_overhead_ms'] = r['autograd_ms'] - r['fused_ms']
            print(json.dumps({k: round(v, 3) if isinstance(v, float) else v for k, v in r.items()}), flush=True)
            torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
