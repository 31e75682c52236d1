"""Four-phase layers on the halo kernel (-m gpu): the nearest-x2 upsample + 3x3 conv of the up-sampling ResBlocks (kind 4)
and the transposed 4x4 stride-2 conv of the encoder-decoder nets (kind 2), each 4 output phases x 2x2 taps on the
low-resolution input.  halo_conv = 1 runs conv_halo.cu (one halo box per channel chunk, transformed once); halo_conv = 0
runs conv_tc.cu (one box per phase and tap).  ksplit = 1 asks both for an unsplit launch.

Both kernels form the same f16 operands and the same k16 products.  Per phase, conv_tc.cu adds them tap by tap, each tap
over all channel chunks; conv_halo.cu chunk by chunk, each chunk over the four taps.  With one chunk (Cin <= 64) the two
orders are the same, and outputs must be bit-identical.  Otherwise each order's fp32 sum of K = 4 Cin terms is within
gamma_K * sum |a_k b_k| of the exact sum (unit roundoff taken as 2^-23, allowing truncating accumulation), so the two
differ by at most 2 K 2^-23 sum |a_k b_k|, per output element.  The per-channel statistics are folded from per-warp
partials over differently shaped pixel groups (16 x 8 tiles against 8 x 16), so they are checked against the output."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import tha4_oracle as O
from tha4_b200._lib import _ptr
import gpu_util as G

pytestmark = pytest.mark.gpu


def conv_phase(kind, x, norm_C, groups, gamma, beta, film0, film1, act, w, bias=None, ksplit=1, reps=0):
    """Four-phase conv through tha4_test_conv_norm_ex: returns (fp32 output, f16 copy widened, statistics [N, Cout, 2]
    fp64, mean device microseconds per launch over `reps` launches, or None)."""
    c = G.ctx()
    N, Cin, H, W = x.shape
    Cout = w.shape[1] if kind == 2 else w.shape[0]
    y = torch.empty(N, Cout, 2 * H, 2 * W, device='cuda:0')
    y16 = torch.empty_like(y)
    st = torch.empty(N, Cout, 2, dtype=torch.float64, device='cuda:0')
    us = ctypes.c_float(0.0)
    t = [G.dev(v) if v is not None else None for v in (x, gamma, beta, film0, film1, w, bias)]
    c._call('tha4_test_conv_norm_ex', kind, _ptr(t[0]), N, Cin, H, W, norm_C, groups, _ptr(t[1]), _ptr(t[2]), _ptr(t[3]),
            _ptr(t[4]), act, _ptr(t[5]), _ptr(t[6]), _ptr(None), 0, Cout, ksplit, _ptr(y), _ptr(y16), _ptr(st), reps,
            ctypes.byref(us), c._stream())
    torch.cuda.synchronize()
    return y.cpu(), y16.cpu(), st.cpu(), (us.value if reps > 0 else None)


def make_inputs(seed, kind, N, Cin, H, W, Cout, norm, bias=True):
    """norm: None (raw input), 'gn' (GroupNorm 32 + FiLM + SiLU) or 'in' (InstanceNorm + ReLU)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, Cin, H, W, generator=g) * 1.7 + 0.4
    gamma, beta = 1.0 + 0.3 * torch.randn(Cin, generator=g), 0.3 * torch.randn(Cin, generator=g)
    f0 = f1 = None
    if norm == 'gn':
        f0, f1 = torch.randn(2 * Cin, generator=g) * 0.3, torch.randn(N, 2 * Cin, generator=g) * 0.3
    k = 4 if kind == 2 else 3
    w = torch.randn((Cin, Cout, k, k) if kind == 2 else (Cout, Cin, k, k), generator=g) / math.sqrt(Cin * k * k)
    b = torch.randn(Cout, generator=g) if bias else None
    norm_C, groups, act = {None: (0, 0, 0), 'gn': (Cin, 32, 2), 'in': (Cin, 0, 1)}[norm]
    return dict(kind=kind, x=x, norm_C=norm_C, groups=groups, gamma=gamma, beta=beta, film0=f0, film1=f1, act=act, w=w, bias=b)


def reference(inp):
    """fp64 conv of the normalised input, and the same conv of |input| with |weights| (the magnitude the reorder bound
    scales with), computed on the device in fp64."""
    d = torch.device('cuda:0')
    x, w = inp['x'].to(d, torch.float64), inp['w'].to(d, torch.float64)
    h = x
    if inp['norm_C']:
        gamma, beta = inp['gamma'].to(d, torch.float64), inp['beta'].to(d, torch.float64)
        if inp['groups']:
            h = F.group_norm(x, inp['groups'], gamma, beta, eps=1e-5)
            f0, f1 = inp['film0'].to(d, torch.float64), inp['film1'].to(d, torch.float64)
            h = O._scaleshift(O._scaleshift(h, f0.unsqueeze(0).expand(x.shape[0], -1)), f1)
            h = F.silu(h)
        else:
            h = F.relu(F.instance_norm(x, weight=gamma, bias=beta, eps=1e-5))

    def conv(a, k, b):
        if inp['kind'] == 2:
            return F.conv_transpose2d(a, k, b, 2, 1)
        return F.conv2d(F.interpolate(a, scale_factor=2, mode='nearest'), k, b, 1, 1)

    bias = inp['bias'].to(d, torch.float64) if inp['bias'] is not None else None
    return conv(h, w, bias).cpu(), conv(h.abs(), w.abs(), None).cpu()


CASES = [
    # kind, N, Cin, H, W (low resolution), Cout, norm.  The frame's four-phase shapes:
    (4, 1, 64, 256, 256, 64, 'gn'),      # upscaler, 256^2 -> 512^2 (one chunk)
    (4, 1, 128, 128, 128, 128, 'gn'),    # upscaler / morpher, 128^2 -> 256^2
    (4, 1, 256, 64, 64, 256, 'gn'),      # 64^2 -> 128^2
    (4, 1, 256, 32, 32, 256, 'gn'),
    (4, 1, 256, 16, 16, 256, 'gn'),
    (2, 1, 512, 24, 24, 256, None),      # face morpher up_0: raw input (normalised by a separate pass)
    (2, 1, 256, 48, 48, 128, 'in'),      # face morpher up_1, up_2: InstanceNorm + ReLU
    (2, 1, 128, 96, 96, 64, 'in'),
    (2, 1, 512, 16, 16, 256, None),      # eyebrow combiner up_0 .. up_2
    (2, 1, 256, 32, 32, 128, 'in'),
    (2, 1, 128, 64, 64, 64, 'in'),
    # micro-batch of 32 (pose sweep)
    (4, 32, 256, 16, 16, 256, 'gn'),
    (2, 32, 128, 32, 32, 64, 'in'),
    # partial low-resolution tiles (8 x 16), batch 2, one chunk and several
    (4, 2, 64, 20, 28, 64, 'gn'),
    (2, 2, 64, 24, 12, 96, None),
    (4, 2, 192, 40, 20, 32, 'in'),
    (2, 2, 128, 12, 36, 128, 'gn'),
]


@pytest.mark.parametrize('case', CASES)
def test_four_phase_halo_vs_per_tap_kernel(case):
    kind, N, Cin, H, W, Cout, norm = case
    c = G.ctx()
    c.set_option('tcgen05', 1)
    inp = make_inputs(211 + CASES.index(case), kind, N, Cin, H, W, Cout, norm)
    outs = {}
    try:
        for halo in (0, 1):
            c.set_option('halo_conv', halo)
            outs[halo] = conv_phase(**inp)
    finally:
        c.set_option('halo_conv', 1)
    (y0, h0, s0, _), (y1, h1, s1, _) = outs[0], outs[1]
    assert torch.isfinite(y1).all()
    ref, mag_in = reference(inp)
    scale = max(1.0, ref.abs().max().item())
    assert (y1.double() - ref).abs().max().item() < 6e-3 * scale, ('vs fp32 reference', case)
    assert (h1 - y1).abs().max().item() <= 1e-3 * scale, 'the f16 copy is the fp32 output rounded once'
    if Cin <= 64:
        assert torch.equal(y0, y1), ('fp32 output', case, (y0 - y1).abs().max().item())
        assert torch.equal(h0, h1), ('f16 copy', case, (h0 - h1).abs().max().item())
    else:
        K = 4 * Cin
        bound = 2 * K * 2.0 ** -23 * mag_in * 1.01          # 1 %: the kernels' f16 operands against the fp64 ones
        d = (y1.double() - y0.double()).abs()
        assert (d <= bound).all(), ('fp32 reorder bound', case, (d / bound).max().item())
        # f16 copies: the fp32 difference, plus one f16 rounding step of the value (2^-10 relative, normal range)
        d16 = (h1.double() - h0.double()).abs()
        assert (d16 <= bound + 2.0 ** -10 * h1.double().abs() + 2.0 ** -24).all(), ('f16 copy', case)
    # statistics: those of the kernel's own output (fp32 partial sums), and the two kernels' within their outputs' spread
    mag = torch.stack([y1.double().abs().sum(dim=(2, 3)), y1.double().pow(2).sum(dim=(2, 3))], dim=-1)
    st_ref = torch.stack([y1.double().sum(dim=(2, 3)), y1.double().pow(2).sum(dim=(2, 3))], dim=-1)
    assert ((s1 - st_ref).abs() <= 1e-5 * mag + 1e-6).all(), ('statistics vs output', case)
    if Cin <= 64:
        assert ((s1 - s0).abs() <= 1e-5 * mag + 1e-6).all(), ('statistics vs per-tap kernel', case)
