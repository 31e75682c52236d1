"""Developer timing: conv1 of every U-Net ResBlock with a 1x1 skip, alone, with the skip folded into its K loop (one halo
launch, skip_fold = 1) and as the pair it replaces (the skip conv, then conv1 adding it as its residual, skip_fold = 0).
CUDA events around `--reps` back-to-back runs (tha4_test_conv_skip_fold).  The compulsory HBM bytes are those of the
tensors each variant must read and write once: h0 and x in f16, the output in fp32 and f16, and for the pair the fp32
skip(x) written and read back.  Prints one line per shape and the frame total (the blocks of Morpher00 and Upscaler02 at
batch 1).

    python scripts/dev/skip_fold.py [--reps 200] [--batch 1]
"""
import argparse
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, '..', '..'))
sys.path.insert(0, os.path.join(HERE, '..', '..', 'tests'))
import gpu_util as G                      # noqa: E402
import test_gpu_skip_fold as T            # noqa: E402

# (H, Cin, Cout): blocks per frame (Morpher00 + Upscaler02), see test_gpu_skip_fold.SHAPES
FRAME = {(16, 512, 256): 4, (32, 512, 256): 4, (64, 512, 256): 2, (64, 384, 256): 2, (64, 128, 256): 2, (128, 384, 128): 2,
         (128, 192, 128): 2, (128, 64, 128): 2, (256, 192, 64): 2, (256, 128, 64): 1, (256, 96, 64): 1, (256, 32, 64): 1,
         (512, 96, 32): 1, (512, 64, 32): 1}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=200)
    ap.add_argument('--batch', type=int, default=1)
    args = ap.parse_args()
    c = G.ctx()
    print('%s, power limit %s' % (torch.cuda.get_device_name(0), os.popen('nvidia-smi --query-gpu=power.limit --format=csv,noheader').read().strip()))
    print('%-16s %5s | %9s %9s %6s | %9s %9s | %7s %7s' % ('H Cin->Cout', 'count', 'pair us', 'fold us', 'ratio', 'pair MB', 'fold MB', 'pair GB/s', 'fold GB/s'))
    tot = [0.0, 0.0, 0.0, 0.0]
    for (H, Cin, Cout), cnt in FRAME.items():
        N = args.batch
        inp = T.make_inputs(7, N, Cin, H, H, Cout)
        us = {}
        for fold in (0, 1):
            c.set_option('skip_fold', fold)
            us[fold] = T.skip_fold(**inp, reps=args.reps)[3]
        c.set_option('skip_fold', 1)
        px = N * H * H
        fold_b = px * (2 * Cout + 2 * Cin + 4 * Cout + 2 * Cout)
        pair_b = fold_b + px * Cout * 4 * 2
        print('%4d %4d->%-4d %5d | %9.1f %9.1f %6.2f | %9.1f %9.1f | %7.0f %7.0f' % (
            H, Cin, Cout, cnt, us[0], us[1], us[0] / us[1], pair_b / 1e6, fold_b / 1e6, pair_b / us[0] / 1e3, fold_b / us[1] / 1e3))
        tot[0] += cnt * us[0]; tot[1] += cnt * us[1]; tot[2] += cnt * pair_b; tot[3] += cnt * fold_b
    print('frame (%d blocks): pair %.1f us, folded %.1f us, saved %.1f us; compulsory bytes %.0f -> %.0f MB' % (
        sum(FRAME.values()), tot[0], tot[1], tot[0] - tot[1], tot[2] / 1e6, tot[3] / 1e6))


if __name__ == '__main__':
    main()
