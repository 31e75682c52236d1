"""Developer timing of the frozen SIREN students' input gradients (not a pytest file), device time between CUDA events.

One forward + backward of a student module for an MSE loss on its outputs; the backward is one tha4_siren_*_backward
call that computes only what is requested:
  image   the frozen body student's d(image) (scatter from the returned warp, no SIREN recompute)
  pose    the frozen student's d(pose) (TF32 recompute + dgrad chain, no weight gradients)
  both    d(image) and d(pose)
  params  the parameter gradients of the trainable module, for comparison
for the body student at B = 1 and 8 and the face student at B = 1 and 64, with the kernel launches of one backward.

Then a pose-fitting loop: the frozen lambda_00 students composed as in mode_14 (face pasted into the image the body
warps), Adam on the 45 pose parameters toward the blended frame rendered at a known pose; prints ms per step and the loss
and pose error after N steps.  Usage: python scripts/dev/student_input_grad_step.py [--steps N] [--warmup W] [--fit-steps N]"""
import argparse
import json
import os
import sys

import torch

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, _ROOT)
from tha4_b200 import image_util, synthetic  # noqa: E402
from tha4_b200.poser.modes import mode_14  # noqa: E402

DEV = torch.device('cuda:0')
GOLDEN = os.path.join(_ROOT, 'tests', 'golden', 'data')


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


def launches_of(ctx, fn):
    l0 = ctx.counter('kernel_launches')
    fn()
    torch.cuda.synchronize()
    return ctx.counter('kernel_launches') - l0


def body(B, sd, warmup, steps):
    frozen = mode_14.load_body_morpher(None, sd).to(DEV).requires_grad_(False)
    trainable = mode_14.load_body_morpher(None, sd).to(DEV)
    ctx = frozen.sync_weights()
    trainable.attach_context(ctx)
    image, pose = synthetic.synthetic_image(0, B).to(DEV), synthetic.random_poses(B, seed=5).to(DEV)
    target = synthetic.synthetic_image(1, B).to(DEV)
    res = dict(student='body', B=B)
    for name, want_image, want_pose in (('image', True, False), ('pose', False, True), ('both', True, True), ('params', False, False)):
        module = trainable if name == 'params' else frozen

        def step():
            im = image.detach().requires_grad_(want_image)
            po = pose.detach().requires_grad_(want_pose)
            o = module(im, po)
            ((o[0] - target).square().mean() + (o[3] - target).square().mean()).backward()
            module.zero_grad(set_to_none=True)

        res[name + '_ms'] = device_ms(step, warmup, steps)
        res[name + '_launches'] = launches_of(ctx, step)
    return res


def face(B, sd, warmup, steps):
    frozen = mode_14.load_face_morpher(None, sd).to(DEV).requires_grad_(False)
    trainable = mode_14.load_face_morpher(None, sd).to(DEV)
    ctx = frozen.sync_weights()
    trainable.attach_context(ctx)
    pose = synthetic.random_poses(B, seed=5)[:, :39].contiguous().to(DEV)
    target = synthetic.synthetic_image(1, B)[:, :, 100:228, 190:318].contiguous().to(DEV)
    res = dict(student='face', B=B)
    for name, module, want_pose in (('pose', frozen, True), ('params', trainable, False)):
        def step():
            o = module(pose.detach().requires_grad_(want_pose))
            (o - target).square().mean().backward()
            module.zero_grad(set_to_none=True)

        res[name + '_ms'] = device_ms(step, warmup, steps)
        res[name + '_launches'] = launches_of(ctx, step)
    return res


def pose_fit(fit_steps, lr):
    sds = {k: torch.load(os.path.join(GOLDEN, 'lambda_00_%s.pt' % k), map_location='cpu') for k in ('face_morpher', 'body_morpher')}
    body_m = mode_14.load_body_morpher(None, sds['body_morpher']).to(DEV).requires_grad_(False)
    face_m = mode_14.load_face_morpher(None, sds['face_morpher']).to(DEV).requires_grad_(False)
    image = image_util.load_poser_image(os.path.join(GOLDEN, 'lambda_00.png')).unsqueeze(0).to(DEV)

    def render(pose):
        body_in = image.clone()
        body_in[:, :, 80:208, 192:320] = face_m(pose[:, :39])
        return body_m(body_in, pose)[0]

    true_pose = synthetic.random_poses(1, seed=31).to(DEV)
    with torch.no_grad():
        target = render(true_pose)
    pose = torch.zeros_like(true_pose).requires_grad_()
    opt = torch.optim.Adam([pose], lr=lr)
    losses = []

    def step():
        loss = (render(pose) - target).abs().mean()
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        losses.append(loss.detach())

    torch.cuda.synchronize()
    ms = device_ms(step, 0, fit_steps)
    losses = [x.item() for x in losses]
    return dict(pose_fit_steps=fit_steps, lr=lr, ms_per_step=ms, loss_first=losses[0], loss_last=losses[-1],
                pose_l1_start=(true_pose.abs()).mean().item(), pose_l1_end=(pose.detach() - true_pose).abs().mean().item())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--fit-steps', type=int, default=200)
    ap.add_argument('--fit-lr', type=float, default=1e-2)
    args = ap.parse_args()
    sds = synthetic.student_state_dicts(0)
    print(json.dumps({'gpu': torch.cuda.get_device_name(0)}), flush=True)
    for fn, sd, bs in ((body, sds['body_morpher'], (1, 8)), (face, sds['face_morpher'], (1, 64))):
        for B in bs:
            r = fn(B, sd, args.warmup, args.steps)
            print(json.dumps({k: round(v, 3) if isinstance(v, float) else v for k, v in r.items()}), flush=True)
            torch.cuda.empty_cache()
    r = pose_fit(args.fit_steps, args.fit_lr)
    print(json.dumps({k: round(v, 5) if isinstance(v, float) else v for k, v in r.items()}), flush=True)


if __name__ == '__main__':
    main()
