"""256-pixel tiles of the 3x3 halo convolution (-m gpu): two consumer warpgroups share every weight tile.  Each output
pixel gets the same products summed in the same order as on the 128-pixel kernel, so the fp32 output and its f16 copy
must be bit-identical; only the fp64 fold of the per-channel statistics (one atomic pair per CTA instead of two) may
round differently."""
import ctypes
import math

import pytest
import torch

from tha4_b200._lib import _ptr
import gpu_util as G

pytestmark = pytest.mark.gpu


def conv_norm_ex(x, norm_C, groups, gamma, beta, film0, film1, act, w, bias=None, res=None, res_mode=0, ksplit=1, reps=0):
    """3x3 conv through tha4_test_conv_norm_ex: returns (fp32 output, f16 copy widened, statistics [N, Cout, 2] fp64,
    mean device microseconds per launch over `reps` launches, or None)."""
    c = G.ctx()
    N, Cin, H, W = x.shape
    Cout = w.shape[0]
    y = torch.empty(N, Cout, H, W, device='cuda:0')
    y16 = torch.empty_like(y)
    st = torch.empty(N, Cout, 2, dtype=torch.float64, device='cuda:0')
    us = ctypes.c_float(0.0)
    t = [G.dev(v) if v is not None else None for v in (x, gamma, beta, film0, film1, w, bias, res)]
    c._call('tha4_test_conv_norm_ex', 0, _ptr(t[0]), N, Cin, H, W, norm_C, groups, _ptr(t[1]), _ptr(t[2]), _ptr(t[3]), _ptr(t[4]),
            act, _ptr(t[5]), _ptr(t[6]), _ptr(t[7]), res_mode, Cout, ksplit, _ptr(y), _ptr(y16), _ptr(st), reps, ctypes.byref(us),
            c._stream())
    torch.cuda.synchronize()
    return y.cpu(), y16.cpu(), st.cpu(), (us.value if reps > 0 else None)


def make_inputs(seed, N, Cin, H, W, Cout, norm, res_mode, bias=True):
    """norm: None (raw input), 'gn' (GroupNorm 32 + FiLM + SiLU) or 'in' (InstanceNorm + ReLU)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, Cin, H, W, generator=g) * 1.7 + 0.4
    gamma, beta = 1.0 + 0.3 * torch.randn(Cin, generator=g), 0.3 * torch.randn(Cin, generator=g)
    f0 = f1 = None
    if norm == 'gn':
        f0, f1 = torch.randn(2 * Cin, generator=g) * 0.3, torch.randn(N, 2 * Cin, generator=g) * 0.3
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / math.sqrt(Cin * 9)
    b = torch.randn(Cout, generator=g) if bias else None
    res = None
    if res_mode == 1:
        res = torch.randn(N, Cout, H, W, generator=g)
    elif res_mode == 2:
        res = torch.randn(N, Cout, H // 2, W // 2, generator=g)
    norm_C, groups, act = {None: (0, 0, 0), 'gn': (Cin, 32, 2), 'in': (Cin, 0, 1)}[norm]
    return dict(x=x, norm_C=norm_C, groups=groups, gamma=gamma, beta=beta, film0=f0, film1=f1, act=act, w=w, bias=b, res=res,
                res_mode=res_mode)


CASES = [
    # N, Cin, H, W, Cout, norm, res_mode (1: same-size residual, by TMA when the output leaves by TMA; 2: nearest-up x2,
    # plain loads), tma_store
    (1, 32, 64, 64, 32, 'gn', 1, 1),       # BN 32, 64-byte rows, one channel chunk, residual by TMA
    (1, 64, 48, 44, 32, 'in', 0, 1),       # BN 32, 128-byte rows; H = 48: the second warpgroup of the last tile row is below the image
    (2, 64, 120, 36, 64, 'gn', 1, 1),      # BN 64, batch 2, H = 120, W not a multiple of 8
    (1, 96, 48, 52, 64, None, 2, 1),       # BN 64, 64-byte rows, three chunks, raw input, residual by plain loads
    (1, 128, 64, 64, 128, 'gn', 1, 1),     # a 128-column plan: 256 x 64 tiles
    (2, 192, 40, 40, 64, 'in', 0, 1),      # three 128-byte chunks, InstanceNorm + ReLU
    (1, 96, 120, 30, 32, None, 2, 1),      # BN 32, 64-byte rows, four chunks, raw input
    (1, 32, 64, 64, 32, 'gn', 1, 0),       # plain stores and plain residual loads (option tma_store = 0)
    (1, 128, 48, 24, 128, 'in', 1, 0),     # same with a 128-column plan
]


@pytest.mark.parametrize('case', CASES)
def test_m256_bit_identical_to_m128(case):
    N, Cin, H, W, Cout, norm, res_mode, tma_store = case
    c = G.ctx()
    c.set_option('tcgen05', 1)
    c.set_option('halo_conv', 1)
    c.set_option('tma_store', tma_store)
    inp = make_inputs(101 + CASES.index(case), N, Cin, H, W, Cout, norm, res_mode)
    outs = {}
    try:
        for m in (0, 1):
            c.set_option('halo_m256', m)
            outs[m] = conv_norm_ex(**inp)         # ksplit = 1: an unsplit launch whatever the tile count
    finally:
        c.set_option('halo_m256', -1)
        c.set_option('tma_store', 1)
    (y0, h0, s0, _), (y1, h1, s1, _) = outs[0], outs[1]
    assert torch.isfinite(y0).all()
    assert torch.equal(y0, y1), ('fp32 output', case, (y0 - y1).abs().max().item())
    assert torch.equal(h0, h1), ('f16 copy', case, (h0 - h1).abs().max().item())
    # statistics: the same fp32 per-warp partials, folded in another fp64 order -> relative to the magnitudes summed
    mag = torch.stack([y0.double().abs().sum(dim=(2, 3)), y0.double().pow(2).sum(dim=(2, 3))], dim=-1)
    assert ((s1 - s0).abs() <= 1e-12 * mag).all(), ('statistics', case, ((s1 - s0).abs() / mag).max().item())
    # and they are the statistics of the output (fp32 partial sums: a looser, absolute check)
    ref = torch.stack([y0.double().sum(dim=(2, 3)), y0.double().pow(2).sum(dim=(2, 3))], dim=-1)
    assert ((s0 - ref).abs() <= 1e-5 * mag + 1e-6).all(), ('statistics vs output', case)
