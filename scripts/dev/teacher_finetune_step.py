"""Device time of fine-tuning the encoder-decoder teachers (developer tool; H100).

For each network at B = 1 and 8, in ms from CUDA events after a warm-up: the forward alone (no grad), forward + input-gradient
backward, forward + parameter-and-input backward (trainable_(True)), and one torch.optim.Adam step (forward, backward,
step, and the re-upload of the weights the next call makes).  Then the weight-gradient launches alone (tha4_test_conv_wgrad,
every layer shape of the network, CUDA events around many launches) with their achieved TFLOP/s -- FLOPs = 2 x the forward's
MACs -- against the data-sheet dense TF32 figure of the H100 SXM (495 TFLOP/s, a data-sheet number, not a measurement), and
beside them the data gradient of the same layer on the conv kernels (tha4_test_conv_backward_data_ex) per FLOP.  The card
name and power limit are read in the same run."""
import ctypes
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))), 'tests'))
from oracle import synth  # noqa: E402
from tha4_b200._lib import Context, _ptr  # noqa: E402
from tha4_b200.nn.eyebrow_decomposer.eyebrow_decomposer_00 import EyebrowDecomposer00  # noqa: E402
from tha4_b200.nn.eyebrow_morphing_combiner.eyebrow_morphing_combiner_00 import EyebrowMorphingCombiner00  # noqa: E402
from tha4_b200.nn.face_morpher.face_morpher_08 import FaceMorpher08  # noqa: E402

DEV = torch.device('cuda:0')
TF32_DATASHEET = 495.0


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
    return [img[:, :, 32:224, 160:352].contiguous(), pose[:, 12:39].contiguous()]


def layers(S, cin0, P):
    """(name, kind, Cx, Cout, H of the operand, x f16, transform) of every conv of a network (kind as tha4_test_conv_wgrad)"""
    b = S // 8
    pp = (P + 7) // 8 * 8
    out = [('down0', 0, cin0, 64, S, 0, 0), ('down1', 1, 64, 128, S, 1, 1), ('down2', 1, 128, 256, S // 2, 1, 1),
           ('down3', 1, 256, 512, S // 4, 1, 1), ('bott0', 0, 512 + pp, 512, b, 1, 1)]
    out += [('res conv0 x5', 0, 512, 512, b, 1, 0), ('res conv1 x5', 0, 512, 512, b, 1, 1)]
    out += [('up0', 2, 512, 256, b, 1, 0), ('up1', 2, 256, 128, 2 * b, 1, 1), ('up2', 2, 128, 64, 4 * b, 1, 1),
            ('head', 3, 64, 16, S, 1, 3)]
    return out


def wgrad_layers(c, S, cin0, P, B, heads):
    total_t, total_f = 0.0, 0.0
    for name, kind, Cx, Cout, H, x16, xf in layers(S, cin0, P):
        if kind == 3:
            Cout = heads
        Ho = H // 2 if kind == 1 else (2 * H if kind == 2 else H)
        x = torch.randn(B, H, H, Cx, device=DEV).to(torch.float16 if x16 else torch.float32)
        dz = torch.randn(B, Ho, Ho, 16 if kind == 3 else Cout, device=DEV)
        norm_C = 512 if name == 'bott0' else Cx
        st = torch.rand(B, norm_C, 2, device=DEV, dtype=torch.float64) * H * H + H * H if xf else None
        g, bt = torch.ones(norm_C, device=DEV), torch.zeros(norm_C, device=DEV)
        c_real = 512 + P if name == 'bott0' else 0
        cr = c_real or Cx
        dW = torch.empty(Cout * cr * (16 if kind in (1, 2) else 9), device=DEV)
        plan = (ctypes.c_int * 4)()

        def run():
            c._call('tha4_test_conv_wgrad', kind, 0, 0, _ptr(x), x16, Cx, B, H, H, Cx, xf, _ptr(st), 1, _ptr(g), _ptr(bt), norm_C,
                    _ptr(dz), dz.shape[-1], Cout, c_real, _ptr(dW), None, plan, c._stream())

        t = timed(run, warmup=3, reps=20)
        pix = B * (H * H if kind == 2 else Ho * Ho)
        flops = 2.0 * pix * Cout * cr * (16 if kind in (1, 2) else 9)
        mult = 5 if 'x5' in name else 1
        total_t += t * mult
        total_f += flops * mult
        print('  wgrad %-13s B=%d %6.3f ms  %7.2f GF  %6.1f TFLOP/s (%4.1f %% of the %.0f data-sheet TF32)  plan N%d M%d x N%d x split %d'
              % (name, B, t, flops / 1e9, flops / t / 1e9, 100 * flops / t / 1e9 / TF32_DATASHEET, TF32_DATASHEET, *plan))
    print('  wgrad total B=%d: %.3f ms, %.1f GF, %.1f TFLOP/s' % (B, total_t, total_f / 1e9, total_f / total_t / 1e9))


def dgrad_res(c, b, B):
    """the data gradient of a 512 -> 512 3x3 ResnetBlock conv at b x b (the same FLOPs as its weight gradient)"""
    w = torch.randn(512, 512, 3, 3, device=DEV) * 0.02
    dy = torch.randn(B, b, b, 512, device=DEV)
    dx = torch.empty(B, b, b, 512, device=DEV)
    split = ctypes.c_int()

    def run():
        c._call('tha4_test_conv_backward_data_ex', 0, _ptr(w), None, None, 0, _ptr(dy), 512, None, 0, _ptr(dx), 512, B, 512, b, b,
                512, 0, 1, ctypes.byref(split), c._stream())

    t = timed(run, warmup=3, reps=20)
    flops = 2.0 * B * b * b * 512 * 512 * 9
    print('  dgrad res conv  B=%d %6.3f ms  %7.2f GF  %6.1f TFLOP/s (conv kernels, adjoint weights; includes packing the adjoint per call)'
          % (B, t, flops / 1e9, flops / t / 1e9))


def main():
    sds = synth.teacher_state_dicts(0)
    print('card: %s' % card())
    nets = [('eyebrow_decomposer', EyebrowDecomposer00, 128, 4, 0, 10), ('eyebrow_morphing_combiner', EyebrowMorphingCombiner00, 128, 8, 12, 8),
            ('face_morpher', FaceMorpher08, 192, 4, 27, 12)]
    kc = Context(DEV)
    for name, cls, S, cin0, P, heads in nets:
        m = cls()
        m.load_state_dict(sds[name])
        m.to(DEV)
        for B in (1, 8):
            xs = inputs(name, B)

            def fwd():
                with torch.no_grad():
                    m(*xs)

            def fwd_bwd_in():
                ins = [x.clone().requires_grad_() for x in xs]
                outs = m(*ins)
                torch.autograd.backward([outs[0]], [torch.ones_like(outs[0])])

            def fwd_bwd_par():
                m.zero_grad(set_to_none=True)
                ins = [x.clone().requires_grad_() for x in xs]
                outs = m(*ins)
                torch.autograd.backward([outs[0]], [torch.ones_like(outs[0])])

            m.trainable_(False)
            t_f, t_in = timed(fwd), timed(fwd_bwd_in)
            m.trainable_(True)
            t_par = timed(fwd_bwd_par)
            opt = torch.optim.Adam(m.parameters(), lr=1e-6)

            def step():
                opt.zero_grad(set_to_none=True)
                (m(*xs)[0].abs().mean()).backward()
                opt.step()

            t_step = timed(step)
            m.trainable_(False)
            print('%-26s B=%d  forward %.3f ms  fwd+input bwd %.3f ms  fwd+param+input bwd %.3f ms  Adam step (incl. re-upload) %.3f ms'
                  % (name, B, t_f, t_in, t_par, t_step))
        for B in (1, 8):
            wgrad_layers(kc, S, cin0, P, B, heads)
            dgrad_res(kc, S // 8, B)
        del m
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
