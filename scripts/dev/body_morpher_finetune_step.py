"""Device time of fine-tuning the body morpher (Morpher00; developer tool; H100).

At B = 1 and 8, in ms from CUDA events after a warm-up: the forward alone (no grad), forward + input-gradient backward,
forward + parameter-and-input backward (trainable_(True)), and one torch.optim.Adam step (forward, backward, step, and the
re-upload of the weights the next call makes).  Then the weight-gradient launches alone (tha4_test_unet_wgrad, every conv
of the network in the operand variant the default mode runs, CUDA events around many launches) with their achieved
TFLOP/s -- FLOPs = 2 x the forward's MACs.  The card name and power limit are read in the same run."""
import ctypes
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts', 'dev'))
from oracle import synth  # noqa: E402
from teacher_finetune_step import DEV, card, timed  # noqa: E402
from tha4_b200._lib import Context, _ptr  # noqa: E402
from tha4_b200.nn.morpher.morpher_00 import Morpher00  # noqa: E402

K3, K1, KUP2, KHEAD = 0, 1, 2, 3
XF_NONE, XF_HALF, XF_FLOAT16 = 0, 1, 3
ACT_NONE, ACT_SILU_FAST = 0, 3


def layers(S=256, mc=64, mults=(1, 2, 4, 4, 4)):
    """(name, kind, Cx, Cout, H of the operand, x f16, transform, act) of every conv of Morpher00 (unet.py:438-529)"""
    L = len(mults)
    out = [('first_conv', K3, 4, mc, S, 0, XF_NONE, ACT_NONE)]

    def res(name, cin, cout, h, pooled=False, up=False):
        r = [(name + '.conv0', KUP2 if up else K3, cin, cout, h, 1, XF_NONE if pooled else XF_HALF, ACT_NONE if pooled else ACT_SILU_FAST),
             (name + '.conv1', K3, cout, cout, 2 * h if up else h, 1, XF_HALF, ACT_SILU_FAST)]
        if cin != cout:
            r.append((name + '.skip', K1, cin, cout, h, 1, XF_NONE, ACT_NONE))
        return r

    def attn(name, c, h):
        return [(name + '.qkv', K1, c, 3 * c, h, 1, XF_HALF, ACT_NONE), (name + '.conv', K1, c, c, h, 0, XF_NONE, ACT_NONE)]

    cur, chans = mc, [mc]
    for i in range(L):
        h, o = S >> i, mc * mults[i]
        out += res('down%d' % i, cur, o, h)
        if i == L - 1:
            out += attn('down%d.attn' % i, o, h)
        chans.append(o)
        if i < L - 1:
            out += res('down%d.downsample' % i, o, o, h // 2, pooled=True)
            chans.append(o)
        cur = o
    h = S >> (L - 1)
    for j in range(4):
        out += res('mid%d' % j, cur, cur, h)
        if j < 3:
            out += attn('mid%d.attn' % j, cur, h)
    for bi, i in enumerate(reversed(range(L))):
        h, o = S >> i, mc * mults[i]
        for r in range(2):
            out += res('up%d.%d' % (bi, r), (cur if r == 0 else o) + chans.pop(), o, h)
            if i == L - 1:
                out += attn('up%d.attn%d' % (bi, r), o, h)
        if i > 0:
            out += res('up%d.upsample' % bi, o, o, h, up=True)
        cur = o
    out.append(('last.2', KHEAD, mc, 7, S, 1, XF_FLOAT16, ACT_SILU_FAST))
    return out


def wgrad_layers(c, B):
    total_t, total_f = 0.0, 0.0
    for name, kind, Cx, Cout, H, x16, xf, act in layers():
        Ho = 2 * H if kind == KUP2 else H
        k = 1 if kind == K1 else 3
        x = torch.randn(B, H, H, Cx, device=DEV).to(torch.float16 if x16 else torch.float32)
        dz = torch.randn(B, Ho, Ho, Cout, device=DEV)
        st = torch.rand(B, Cx, 2, device=DEV, dtype=torch.float64) * H * H + H * H if xf else None
        g, bt = torch.ones(Cx, device=DEV), torch.zeros(Cx, device=DEV)
        dW = torch.empty(Cout * Cx * k * k, device=DEV)
        plan = (ctypes.c_int * 4)()

        def run():
            c._call('tha4_test_unet_wgrad', kind, 0, 0, _ptr(x), x16, Cx, B, H, H, Cx, xf, act, _ptr(st), 1, 32,
                    _ptr(g), _ptr(bt), None, None, 0, 0, _ptr(dz), Cout, Cout, _ptr(dW), None, plan, c._stream())

        t = timed(run, warmup=3, reps=20)
        flops = 2.0 * B * Ho * Ho * Cout * Cx * k * k
        total_t += t
        total_f += flops
        print('  wgrad %-22s B=%d %6.3f ms  %7.2f GF  %6.1f TFLOP/s  plan N%d M%d x N%d x split %d'
              % (name, B, t, flops / 1e9, flops / t / 1e9, *plan))
    print('  wgrad total B=%d: %d launches, %.3f ms, %.1f GF, %.1f TFLOP/s' % (B, len(layers()), total_t, total_f / 1e9, total_f / total_t / 1e9))


def main():
    sd = synth.teacher_state_dicts(0)['body_morpher']
    print('card: %s' % card())
    m = Morpher00()
    m.load_state_dict(sd)
    m.to(DEV)
    for B in (1, 8):
        img = torch.nn.functional.interpolate(synth.synthetic_image(0, B), size=(256, 256), mode='bilinear', align_corners=False).to(DEV)
        pose = synth.random_poses(B, seed=1)[:, 39:45].contiguous().to(DEV)

        def fwd():
            with torch.no_grad():
                m(img, pose)

        def fwd_bwd():
            m.zero_grad(set_to_none=True)
            outs = m(img.clone().requires_grad_(), pose)
            torch.autograd.backward([outs[0]], [torch.ones_like(outs[0])])

        m.trainable_(False)
        t_f, t_in = timed(fwd), timed(fwd_bwd)
        m.trainable_(True)
        t_par = timed(fwd_bwd)
        opt = torch.optim.Adam(m.parameters(), lr=1e-6)

        def step():
            opt.zero_grad(set_to_none=True)
            (m(img, pose)[0].abs().mean()).backward()
            opt.step()

        t_step = timed(step)
        m.trainable_(False)
        print('Morpher00 B=%d  forward %.3f ms  fwd+input bwd %.3f ms  fwd+param+input bwd %.3f ms  Adam step (incl. re-upload) %.3f ms'
              % (B, t_f, t_in, t_par, t_step))
    kc = Context(DEV)
    for B in (1, 8):
        wgrad_layers(kc, B)


if __name__ == '__main__':
    main()
