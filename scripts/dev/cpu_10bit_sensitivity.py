"""How much does rounding conv operands to a 10-bit mantissa (what TF32 / f16 tensor-core operands carry) move the
teacher's outputs on the seeded weights used by tests and bench?  Pure CPU experiment on the oracle: every
conv2d / conv_transpose2d input and weight is rounded through float16, everything else stays fp32.
Context for the default-mode tolerances (DESIGN.md)."""
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import synth, tha4_oracle as O  # noqa: E402

torch.set_num_threads(8)
sds = synth.teacher_state_dicts(0)
img = synth.synthetic_image(0, 1)[0]
conv2d, convt = F.conv2d, F.conv_transpose2d
r10 = lambda x: x.half().float()   # noqa: E731
for seed in (99, 7, 1234):
    pose = synth.random_poses(1, seed=seed)[0]
    F.conv2d, F.conv_transpose2d = conv2d, convt
    with torch.no_grad():
        ref = O.mode_07_outputs(sds, img, pose)
    F.conv2d = lambda x, w, b=None, *a, **k: conv2d(r10(x), r10(w), b, *a, **k)
    F.conv_transpose2d = lambda x, w, b=None, *a, **k: convt(r10(x), r10(w), b, *a, **k)
    with torch.no_grad():
        emu = O.mode_07_outputs(sds, img, pose)
    print('pose seed %d: |10-bit-operand oracle - fp32 oracle| per mode_07 output (and mean |output|)' % seed)
    for i, (a, b) in enumerate(zip(emu, ref)):
        print('  out %2d %-18s max %.3e mean %.3e   amp %.3f' % (i, tuple(b.shape), (a - b).abs().max().item(), (a - b).abs().mean().item(), b.abs().mean().item()))
    print('  worst mean: %.3e  worst max: %.3e' % (max((a - b).abs().mean().item() for a, b in zip(emu, ref)),
                                                  max((a - b).abs().max().item() for a, b in zip(emu, ref))))
