"""Device time of the teachers' input gradients: the encoder-decoder networks, the body morpher, the upscaler and the full
mode_07 poser (developer tool; H100).

First the upscaler backward's workspace per frame: the context's pool size after one backward at B = 1 and at B = 2 on a fresh
context.  Then for each network, and for mode_07 with the image and the pose requiring grad, at B = 1 and 8: the forward alone
(no grad) and forward + backward with every input requiring grad, in ms from CUDA events after a warm-up, and the kernel
launches of the forward and of the backward.  Then one mode_12 and one mode_07 pose-fitting step at B = 1 (forward + L1 loss
+ backward + Adam).  The card name and power limit are read in the same run."""
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle import synth  # noqa: E402
from tha4_b200.nn.eyebrow_decomposer.eyebrow_decomposer_00 import EyebrowDecomposer00  # noqa: E402
from tha4_b200.nn.eyebrow_morphing_combiner.eyebrow_morphing_combiner_00 import EyebrowMorphingCombiner00  # noqa: E402
from tha4_b200.nn.face_morpher.face_morpher_08 import FaceMorpher08  # noqa: E402
from tha4_b200.nn.morpher.morpher_00 import Morpher00  # noqa: E402
from tha4_b200.nn.upscaler.upscaler_02 import Upscaler02  # noqa: E402
from tha4_b200.poser.modes import mode_07, mode_12  # noqa: E402

DEV = torch.device('cuda:0')


def timed(fn, warmup=3, reps=10):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        return q or torch.cuda.get_device_name(0)
    except Exception:
        return torch.cuda.get_device_name(0)


def inputs(name, B):
    img = synth.synthetic_image(0, B).to(DEV)
    pose = synth.random_poses(B, seed=1).to(DEV)
    if name == 'eyebrow_decomposer':
        return [img[:, :, 64:192, 192:320].contiguous()]
    if name == 'eyebrow_morphing_combiner':
        c = img[:, :, 64:192, 192:320].contiguous()
        return [c, c.flip(3).contiguous(), pose[:, :12].contiguous()]
    if name == 'body_morpher':
        return [img[:, :, ::2, ::2].contiguous(), pose[:, 39:45].contiguous()]
    if name == 'upscaler':     # coarse inputs at 256, as mode_07 hands them over
        return [img, img[:, :, ::2, ::2].contiguous(), 0.02 * img[:, :2, ::2, ::2].contiguous(), pose[:, 39:45].contiguous()]
    if name == 'mode_07':
        return [img, pose]
    return [img[:, :, 32:224, 160:352].contiguous(), pose[:, 12:39].contiguous()]


def upscaler_workspace(sds):
    """workspace_bytes after one upscaler forward + backward at B on a fresh context (the pool keeps its peak)."""
    for B in (1, 2):
        m = Upscaler02()
        m.load_state_dict(sds['upscaler'])
        m.to(DEV)                  # a module gets a context of its own on first use
        ins = [x.clone().requires_grad_() for x in inputs('upscaler', B)]
        outs = m(*ins)
        torch.autograd.backward([outs[0]], [torch.ones_like(outs[0])])
        torch.cuda.synchronize()
        print('upscaler backward workspace B=%d: %.1f MiB' % (B, m.context().counter('workspace_bytes') / 2 ** 20))
        del m, ins, outs
        torch.cuda.empty_cache()


def main():
    sds = synth.teacher_state_dicts(0)
    print('card: %s' % card())
    upscaler_workspace(sds)
    poser7 = mode_07.create_poser(DEV, state_dicts=sds)
    nets = [('eyebrow_decomposer', EyebrowDecomposer00), ('eyebrow_morphing_combiner', EyebrowMorphingCombiner00),
            ('face_morpher', FaceMorpher08), ('body_morpher', Morpher00), ('upscaler', Upscaler02), ('mode_07', None)]
    for name, cls in nets:
        if cls is None:
            m = poser7.get_posing_outputs
            ctx = poser7.get_modules()['upscaler'].context()
        else:
            m = cls()
            m.load_state_dict(sds[name])
            m.to(DEV)
            ctx = m.context()
        for B in (1, 8):
            xs = inputs(name, B)

            def fwd():
                with torch.no_grad():
                    m(*xs)

            def fwd_bwd():
                ins = [x.clone().requires_grad_() for x in xs]
                outs = m(*ins)
                torch.autograd.backward([outs[0]], [torch.ones_like(outs[0])])

            t_f, t_fb = timed(fwd), timed(fwd_bwd)
            ins = [x.clone().requires_grad_() for x in xs]
            torch.cuda.synchronize()
            l0 = ctx.counter('kernel_launches')
            outs = m(*ins)
            torch.cuda.synchronize()
            l1 = ctx.counter('kernel_launches')
            torch.autograd.backward([outs[0]], [torch.ones_like(outs[0])])
            torch.cuda.synchronize()
            print('%-26s B=%d  forward %.3f ms  forward+backward %.3f ms  forward launches %d  backward launches %d'
                  % (name, B, t_f, t_fb, l1 - l0, ctx.counter('kernel_launches') - l1))
    poser = mode_12.create_poser(DEV, state_dicts=sds)
    image = synth.synthetic_image(0, 1).to(DEV)
    with torch.no_grad():
        target = poser.get_posing_outputs(image, synth.random_poses(1, seed=5).to(DEV))[0].clone()
    p39 = torch.zeros(1, 39, device=DEV, requires_grad=True)
    opt = torch.optim.Adam([p39], lr=5e-2)

    def step():
        pose = torch.cat([p39, torch.zeros(1, 6, device=DEV)], dim=1)
        loss = (poser.get_posing_outputs(image, pose)[0] - target).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()

    print('mode_12 pose-fitting step B=1: %.3f ms' % timed(step))
    with torch.no_grad():
        target7 = poser7.get_posing_outputs(image, synth.random_poses(1, seed=5).to(DEV))[0].clone()
    p45 = torch.zeros(1, 45, device=DEV, requires_grad=True)
    opt7 = torch.optim.Adam([p45], lr=5e-2)

    def step7():
        loss = (poser7.get_posing_outputs(image, p45)[0] - target7).abs().mean()
        opt7.zero_grad()
        loss.backward()
        opt7.step()

    print('mode_07 pose-fitting step B=1: %.3f ms' % timed(step7))


if __name__ == '__main__':
    main()
