"""Developer diagnostics for the wgmma conv kernel (option "tcgen05") (not a pytest file): structured inputs that expose layout bugs."""
import math
import sys
import os

import torch
import torch.nn.functional as F

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, _ROOT)
sys.path.insert(0, os.path.join(_ROOT, 'tests'))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gpu_util as G  # noqa: E402


def run(kind, N, Cin, H, Cout, bias=False, res_mode=0, ksplit=0, seed=0, structured=None):
    g = torch.Generator().manual_seed(seed)
    k = {0: 3, 1: 4, 2: 4, 3: 1}[kind]
    x = torch.randn(N, Cin, H, H, generator=g)
    wshape = (Cin, Cout, k, k) if kind == 2 else (Cout, Cin, k, k)
    w = torch.randn(wshape, generator=g) / math.sqrt(Cin * k * k)
    if structured == 'identity':       # 1x1 identity: output channel c == input channel c
        w = torch.zeros(wshape)
        for c in range(min(Cin, Cout)):
            w[c, c, k // 2, k // 2] = 1.0
    b = torch.randn(Cout, generator=g) if bias else None
    ref = {0: lambda: F.conv2d(x, w, b, 1, 1), 2: lambda: F.conv_transpose2d(x, w, b, 2, 1), 3: lambda: F.conv2d(x, w, b)}[kind]()
    res = None
    if res_mode:
        res = torch.randn(N, Cout, ref.shape[2], ref.shape[3], generator=g)
        ref = ref + res
    G.ctx().set_option('tcgen05', 1)
    out = G.conv(kind, x, w, b, res, res_mode, 0, strict=0, ksplit=ksplit)
    G.ctx().set_option('tcgen05', 0)
    out_mma = G.conv(kind, x, w, b, res, res_mode, 0, strict=0, ksplit=ksplit)
    G.ctx().set_option('tcgen05', 1)
    e, em = G.err(out, ref), G.err(out_mma, ref)
    print('kind %d N%d Cin%d H%d Cout%d bias%d res%d ks%d %s: tc max %.3e mean %.3e | mma max %.3e mean %.3e | ref absmax %.2f'
          % (kind, N, Cin, H, Cout, bias, res_mode, ksplit, structured or '', e[0], e[1], em[0], em[1], ref.abs().max()))
    if e[0] > 5e-2 * max(1.0, ref.abs().max().item()):
        d = (out - ref).abs()
        print('   per-channel err (first 16):', [round(v, 3) for v in d.amax(dim=(0, 2, 3))[:16].tolist()])
        print('   per-row err (first 16):', [round(v, 3) for v in d.amax(dim=(0, 1, 3))[:16].tolist()])
        print('   per-col err (first 16):', [round(v, 3) for v in d.amax(dim=(0, 1, 2))[:16].tolist()])
        print('   out[0,:4,0,:4]', out[0, :4, 0, :4].tolist())
        print('   ref[0,:4,0,:4]', ref[0, :4, 0, :4].tolist())
    return e


if __name__ == '__main__':
    torch.cuda.init()
    run(3, 1, 32, 16, 32, structured='identity')
    run(3, 1, 32, 16, 32)
    run(3, 1, 64, 16, 64)
    run(3, 2, 256, 16, 768, bias=True)
    run(0, 1, 32, 16, 32)
    run(0, 1, 64, 32, 64, bias=True, res_mode=1)
    run(0, 1, 4, 32, 64)
    run(0, 1, 16, 64, 32, bias=True)
    run(0, 1, 96, 32, 32, bias=True)
    run(0, 1, 524, 16, 512)
    run(0, 1, 540, 24, 512, ksplit=3)
    run(0, 2, 256, 64, 256, bias=True)
    run(0, 1, 128, 128, 128, bias=True)
    run(2, 1, 512, 16, 256)
    run(2, 2, 128, 24, 64)
    print('done')
