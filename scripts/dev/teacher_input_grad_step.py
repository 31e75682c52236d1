"""Device time of the teachers' input gradients: the encoder-decoder networks and the body morpher (developer tool; H100).

For each network at B = 1 and 8: the forward alone (no grad) and forward + backward with every input requiring grad, in ms
from CUDA events after a warm-up, and the kernel launches of the backward.  Then one mode_12 pose-fitting step at B = 1
(forward + L1 loss + backward + Adam).  The card name and power limit are read in the same run."""
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
from tha4_b200.poser.modes import mode_12  # noqa: E402

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
    return [img[:, :, 32:224, 160:352].contiguous(), pose[:, 12:39].contiguous()]


def main():
    sds = synth.teacher_state_dicts(0)
    print('card: %s' % card())
    for name, cls in (('eyebrow_decomposer', EyebrowDecomposer00), ('eyebrow_morphing_combiner', EyebrowMorphingCombiner00),
                      ('face_morpher', FaceMorpher08), ('body_morpher', Morpher00)):
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
            outs = m(*ins)
            torch.cuda.synchronize()
            l0 = ctx.counter('kernel_launches')
            torch.autograd.backward([outs[0]], [torch.ones_like(outs[0])])
            torch.cuda.synchronize()
            print('%-26s B=%d  forward %.3f ms  forward+backward %.3f ms  backward launches %d'
                  % (name, B, t_f, t_fb, ctx.counter('kernel_launches') - l0))
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


if __name__ == '__main__':
    main()
