"""Device time and workspace of fine-tuning the upscaler (Upscaler02; developer tool; H100).

At B = 1 and 8 (8 frames span two passes of the backward, with or without parameter gradients), in ms from CUDA events
after a warm-up: the forward alone (no grad), forward + input-gradient backward, forward + parameter-and-input backward
(trainable_(True)), and one torch.optim.Adam step (forward, backward, step, and the re-upload of the weights the next call
makes).  Then the weight-gradient launches alone (tha4_test_unet_wgrad, every conv of the network in the operand variant the
default mode runs -- the first conv as its two channel views of the 16-channel prologue output -- CUDA events around many
launches) with their achieved TFLOP/s, FLOPs = 2 x the forward's MACs.  Last, the context's workspace pool after one
backward with d_params at B = 1 and 2 on a fresh context, in both precision modes, and without d_params for comparison.
The card name and power limit are read in the same run."""
import ctypes
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts', 'dev'))
from oracle import synth  # noqa: E402
from body_morpher_finetune_step import layers  # noqa: E402
from teacher_finetune_step import DEV, card, timed  # noqa: E402
from tha4_b200._lib import Context, _ptr  # noqa: E402
from tha4_b200.nn.upscaler.upscaler_02 import Upscaler02  # noqa: E402

K3, K1, KUP2 = 0, 1, 2
S, MC, MULTS = 512, 32, (1, 2, 4, 8, 8, 8)


def inputs(B):
    rest = synth.synthetic_image(0, B).to(DEV)
    posed = F.interpolate(synth.synthetic_image(1, B), size=(256, 256), mode='bilinear', align_corners=False).to(DEV)
    grid = (torch.randn(B, 2, 256, 256, generator=torch.Generator().manual_seed(2)) * 0.02).to(DEV)
    pose = synth.random_poses(B, seed=3)[:, 39:45].contiguous().to(DEV)
    return [rest, posed.contiguous(), grid, pose]


def wgrad_layers(c, B):
    total_t, total_f, n = 0.0, 0.0, 0
    # the fused first conv as the backward runs it: two convs on channel views (ld 16) of the fp32 prologue output
    convs = [('first_conv (view 0-3)', K3, 4, MC, S, 0, 0, 0, 0), ('coarse_image_conv (view 4-13)', K3, 10, MC, S, 0, 0, 0, 4)]
    convs += [l + (None,) for l in layers(S, MC, MULTS) if l[0] != 'first_conv']
    for name, kind, Cx, Cout, H, x16, xf, act, view in convs:
        Ho = 2 * H if kind == KUP2 else H
        k = 1 if kind == K1 else 3
        ld = 16 if view is not None else Cx
        x = torch.randn(B, H, H, ld, device=DEV).to(torch.float16 if x16 else torch.float32)
        xp = x[..., view:] if view is not None else x
        dz = torch.randn(B, Ho, Ho, Cout, device=DEV)
        st = torch.rand(B, Cx, 2, device=DEV, dtype=torch.float64) * H * H + H * H if xf else None
        g, bt = torch.ones(Cx, device=DEV), torch.zeros(Cx, device=DEV)
        dW = torch.empty(Cout * Cx * k * k, device=DEV)
        plan = (ctypes.c_int * 4)()

        def run():
            c._call('tha4_test_unet_wgrad', kind, 0, 0, _ptr(xp), x16, ld, B, H, H, Cx, xf, act, _ptr(st), 1, 32,
                    _ptr(g), _ptr(bt), None, None, 0, 0, _ptr(dz), Cout, Cout, _ptr(dW), None, plan, c._stream())

        t = timed(run, warmup=3, reps=20)
        flops = 2.0 * B * Ho * Ho * Cout * Cx * k * k
        total_t += t
        total_f += flops
        n += 1
        print('  wgrad %-30s B=%d %6.3f ms  %7.2f GF  %6.1f TFLOP/s  plan N%d M%d x N%d x split %d'
              % (name, B, t, flops / 1e9, flops / t / 1e9, *plan))
    print('  wgrad total B=%d: %d launches, %.3f ms, %.1f GF, %.1f TFLOP/s' % (B, n, total_t, total_f / 1e9, total_f / total_t / 1e9))


def workspace(sd):
    """MiB of the workspace pool after one backward on a fresh context, per (strict, with d_params) and B."""
    for strict in (0, 1):
        for with_params in (False, True):
            mib = []
            for B in (1, 2):
                c = Context(DEV)
                c.set_option('strict', strict)
                c.load_net('upscaler', sd)
                x = inputs(B)
                ups = [torch.randn(B, ch, 512, 512, device=DEV) * 1e-3 if k != 2 else None for k, ch in enumerate((4, 1, 4, 2, 4))]
                d_pose = torch.empty(B, 6, device=DEV)
                d_params = torch.empty(c.param_count('upscaler'), device=DEV) if with_params else None
                c.upscaler_backward(*x, ups, d_pose=d_pose, d_params=d_params)
                torch.cuda.synchronize()
                mib.append(c.counter('workspace_bytes') / 2 ** 20)
                del c, d_params
                torch.cuda.empty_cache()
            print('workspace strict=%d %-16s B=1 %.0f MiB  B=2 %.0f MiB  per frame %.0f MiB'
                  % (strict, 'with d_params' if with_params else 'inputs only', mib[0], mib[1], mib[1] - mib[0]))


def main():
    sd = synth.teacher_state_dicts(0)['upscaler']
    print('card: %s' % card())
    workspace(sd)
    m = Upscaler02()
    m.load_state_dict(sd)
    m.to(DEV)
    for B in (1, 8):
        x = inputs(B)

        def fwd():
            with torch.no_grad():
                m(*x)

        def fwd_bwd():
            m.zero_grad(set_to_none=True)
            outs = m(x[0].clone().requires_grad_(), *x[1:])
            torch.autograd.backward([outs[0]], [torch.ones_like(outs[0])])

        m.trainable_(False)
        t_f, t_in = timed(fwd), timed(fwd_bwd, warmup=2, reps=5)
        m.trainable_(True)
        t_par = timed(fwd_bwd, warmup=2, reps=5)
        opt = torch.optim.Adam(m.parameters(), lr=1e-6)

        def step():
            opt.zero_grad(set_to_none=True)
            (m(*x)[0].abs().mean()).backward()
            opt.step()

        t_step = timed(step, warmup=2, reps=5)
        m.trainable_(False)
        print('Upscaler02 B=%d  forward %.3f ms  fwd+input bwd %.3f ms  fwd+param+input bwd %.3f ms  Adam step (incl. re-upload) %.3f ms'
              % (B, t_f, t_in, t_par, t_step))
    kc = Context(DEV)
    for B in (1, 4):
        wgrad_layers(kc, B)
    print('card: %s' % card())


if __name__ == '__main__':
    main()
