"""Two CTAs per SM for the halo convolution's 256 x 64 and four-phase tiles (-m gpu).  halo_ctas = 2 runs the 256-thread
CTAs without a producer warp (consumer thread 0 issues the TMA loads, shallower rings), halo_ctas = 1 the 288-thread CTAs
with a producer warp.  Tile, tap order, wgmma shapes, K order and epilogue arithmetic are the same, so the fp32 output and
its f16 copy must be bit-identical; only the fp64 atomics of the per-channel statistics may add in another order."""
import pytest
import torch

import gpu_util as G
import test_gpu_halo_m256 as M
import test_gpu_halo_phase as P

pytestmark = pytest.mark.gpu


def _compare(outs, case):
    (y1, h1, s1, _), (y2, h2, s2, _) = outs[1], outs[2]
    assert torch.isfinite(y1).all()
    assert torch.equal(y1, y2), ('fp32 output', case, (y1 - y2).abs().max().item())
    assert torch.equal(h1, h2), ('f16 copy', case, (h1 - h2).abs().max().item())
    mag = torch.stack([y1.double().abs().sum(dim=(2, 3)), y1.double().pow(2).sum(dim=(2, 3))], dim=-1)
    assert ((s2 - s1).abs() <= 1e-12 * mag).all(), ('statistics', case, ((s2 - s1).abs() / mag).max().item())


@pytest.mark.parametrize('case', M.CASES)
def test_3x3_two_ctas_bit_identical(case):
    N, Cin, H, W, Cout, norm, res_mode, tma_store = case
    c = G.ctx()
    c.set_option('tcgen05', 1)
    c.set_option('halo_conv', 1)
    c.set_option('tma_store', tma_store)
    c.set_option('halo_m256', 1)                 # 256-pixel tiles whatever the tile count
    inp = M.make_inputs(101 + M.CASES.index(case), N, Cin, H, W, Cout, norm, res_mode)
    outs = {}
    try:
        for k in (1, 2):
            c.set_option('halo_ctas', k)
            outs[k] = M.conv_norm_ex(**inp)
    finally:
        c.set_option('halo_ctas', -1)
        c.set_option('halo_m256', -1)
        c.set_option('tma_store', 1)
    _compare(outs, case)


# batch 32 and a multi-chunk layer with a same-size residual by TMA
EXTRA_3x3 = [
    (32, 64, 32, 32, 64, 'gn', 1, 1),
    (1, 256, 64, 64, 256, 'gn', 1, 1),
    (1, 512, 32, 32, 512, 'in', 0, 1),
]


@pytest.mark.parametrize('case', EXTRA_3x3)
def test_3x3_two_ctas_bit_identical_frame_shapes(case):
    N, Cin, H, W, Cout, norm, res_mode, tma_store = case
    c = G.ctx()
    c.set_option('tcgen05', 1)
    c.set_option('halo_conv', 1)
    c.set_option('halo_m256', 1)
    inp = M.make_inputs(401 + EXTRA_3x3.index(case), N, Cin, H, W, Cout, norm, res_mode)
    outs = {}
    try:
        for k in (1, 2):
            c.set_option('halo_ctas', k)
            outs[k] = M.conv_norm_ex(**inp)
    finally:
        c.set_option('halo_ctas', -1)
        c.set_option('halo_m256', -1)
    _compare(outs, case)


@pytest.mark.parametrize('case', P.CASES)
def test_four_phase_two_ctas_bit_identical(case):
    kind, N, Cin, H, W, Cout, norm = case
    c = G.ctx()
    c.set_option('tcgen05', 1)
    c.set_option('halo_conv', 1)
    inp = P.make_inputs(211 + P.CASES.index(case), kind, N, Cin, H, W, Cout, norm)
    outs = {}
    try:
        for k in (1, 2):
            c.set_option('halo_ctas', k)
            outs[k] = P.conv_phase(**inp)         # ksplit = 1: an unsplit launch, on the halo kernel
    finally:
        c.set_option('halo_ctas', -1)
    _compare(outs, case)
