"""Row-owning cluster pairs of the halo convolution (-m gpu).  halo_cs = 2 splits a one-CTA-per-SM launch of the 256 x 64
and four-phase tiles over a cluster pair: each rank sums half of the channel chunks, and rank r finishes the rows of
warpgroup r with the peer's partial added.  halo_cs = 1 runs the unsplit launch of the same tile.

Both form the same f16 operands and k16 products; the split adds the two halves of K once more at the end.  Each order's
fp32 sum of K terms is within gamma_K * sum |a_k b_k| of the exact sum (unit roundoff taken as 2^-23), so the two differ by
at most 2 K 2^-23 sum |a_k b_k| per output element, the bound of test_gpu_halo_phase.py.  The per-channel statistics are
sums of the outputs themselves, so they are checked against each output and against each other within what the outputs'
differences can move them."""
import math
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from oracle import tha4_oracle as O
import gpu_util as G
import test_gpu_halo_m256 as M
import test_gpu_halo_phase as P

pytestmark = pytest.mark.gpu


def reference_3x3(inp):
    """fp64 conv (+ residual) of the normalised input, and the same conv of |input| with |weights|, on the device."""
    d = torch.device('cuda:0')
    x, w = inp['x'].to(d, torch.float64), inp['w'].to(d, torch.float64)
    h = x
    if inp['norm_C']:
        gamma, beta = inp['gamma'].to(d, torch.float64), inp['beta'].to(d, torch.float64)
        if inp['groups']:
            h = F.group_norm(x, inp['groups'], gamma, beta, eps=1e-5)
            f0, f1 = inp['film0'].to(d, torch.float64), inp['film1'].to(d, torch.float64)
            h = F.silu(O._scaleshift(O._scaleshift(h, f0.unsqueeze(0).expand(x.shape[0], -1)), f1))
        else:
            h = F.relu(F.instance_norm(x, weight=gamma, bias=beta, eps=1e-5))
    bias = inp['bias'].to(d, torch.float64) if inp['bias'] is not None else None
    y = F.conv2d(h, w, bias, 1, 1)
    if inp['res'] is not None:
        r = inp['res'].to(d, torch.float64)
        y = y + (r if inp['res_mode'] == 1 else F.interpolate(r, scale_factor=2, mode='nearest'))
    return y.cpu(), F.conv2d(h.abs(), w.abs(), None, 1, 1).cpu()


def _check(outs, ref, mag_in, K, case):
    (y1, h1, s1, _), (y2, h2, s2, _) = outs[1], outs[2]
    assert torch.isfinite(y2).all()
    scale = max(1.0, ref.abs().max().item())
    for y, h in ((y1, h1), (y2, h2)):
        assert (y.double() - ref).abs().max().item() < 6e-3 * scale, ('vs fp64 reference', case)
        assert (h - y).abs().max().item() <= 1e-3 * scale, 'the f16 copy is the fp32 output rounded once'
    bound = 2 * K * 2.0 ** -23 * mag_in * 1.01          # 1 %: the kernels' f16 operands against the fp64 ones
    d = (y2.double() - y1.double()).abs()
    assert (d <= bound).all(), ('fp32 reorder bound', case, (d / bound).max().item())
    d16 = (h2.double() - h1.double()).abs()
    assert (d16 <= bound + 2.0 ** -10 * h2.double().abs() + 2.0 ** -24).all(), ('f16 copy', case)
    # statistics: each those of its own output (fp32 per-warp partials), and the two within what the outputs' difference moves
    for y, s in ((y1, s1), (y2, s2)):
        mag = torch.stack([y.double().abs().sum(dim=(2, 3)), y.double().pow(2).sum(dim=(2, 3))], dim=-1)
        st_ref = torch.stack([y.double().sum(dim=(2, 3)), y.double().pow(2).sum(dim=(2, 3))], dim=-1)
        assert ((s - st_ref).abs() <= 1e-5 * mag + 1e-6).all(), ('statistics vs output', case)
    st1 = torch.stack([y1.double().sum(dim=(2, 3)), y1.double().pow(2).sum(dim=(2, 3))], dim=-1)
    st2 = torch.stack([y2.double().sum(dim=(2, 3)), y2.double().pow(2).sum(dim=(2, 3))], dim=-1)
    mag = torch.stack([y1.double().abs().sum(dim=(2, 3)), y1.double().pow(2).sum(dim=(2, 3))], dim=-1)
    assert ((s2 - s1).abs() <= (st2 - st1).abs() + 2e-5 * mag + 1e-6).all(), ('statistics, split vs unsplit', case)


CASES_3x3 = [
    # N, Cin, H, W, Cout, norm, res_mode (1: same-size residual, by TMA; 2: nearest-up x2, plain loads), tma_store.
    # The frame's 64^2 layers with Cout 256 (64 CTAs) and 128 -> 128 (32 CTAs):
    (1, 128, 64, 64, 256, 'gn', 0, 1),
    (1, 256, 64, 64, 256, 'gn', 1, 1),
    (1, 512, 64, 64, 256, 'gn', 0, 1),
    (1, 384, 64, 64, 256, 'gn', 1, 1),
    (1, 128, 64, 64, 128, 'gn', 0, 1),
    (1, 128, 64, 64, 128, None, 0, 1),
    # partial tiles (the second warpgroup's rows below the image, W not a multiple of 8), batch 2, InstanceNorm + ReLU
    (2, 192, 40, 36, 64, 'in', 1, 1),
    (1, 128, 48, 44, 32, 'in', 0, 1),          # BN 32
    (1, 96, 48, 52, 64, None, 2, 1),           # 64-byte rows, three chunks, raw input, up-sampled residual
    (1, 256, 64, 64, 256, 'gn', 1, 0),         # plain stores and plain residual loads
]


@pytest.mark.parametrize('case', CASES_3x3)
def test_3x3_row_split_vs_unsplit(case):
    N, Cin, H, W, Cout, norm, res_mode, tma_store = case
    c = G.ctx()
    c.set_option('tcgen05', 1)
    c.set_option('halo_conv', 1)
    c.set_option('tma_store', tma_store)
    c.set_option('halo_m256', 1)
    c.set_option('halo_ctas', 1)
    inp = M.make_inputs(601 + CASES_3x3.index(case), N, Cin, H, W, Cout, norm, res_mode)
    outs = {}
    try:
        for k in (1, 2):
            c.set_option('halo_cs', k)
            outs[k] = M.conv_norm_ex(**inp)
    finally:
        for o in ('halo_cs', 'halo_ctas', 'halo_m256'):
            c.set_option(o, -1)
        c.set_option('tma_store', 1)
    ref, mag_in = reference_3x3(inp)
    _check(outs, ref, mag_in, 9 * Cin, case)


CASES_PHASE = [
    # kind, N, Cin, H, W (low resolution), Cout, norm
    (4, 1, 256, 32, 32, 256, 'gn'),      # U-Net up-sampling from 32^2 (64 CTAs)
    (2, 1, 128, 64, 64, 64, 'in'),       # combiner transposed conv from 64^2
    (2, 1, 256, 48, 48, 128, 'in'),      # face morpher transposed conv from 48^2 (72 CTAs)
    (2, 1, 512, 24, 24, 256, None),      # raw input
    (4, 2, 192, 40, 20, 32, 'in'),       # partial tiles, batch 2, three chunks
]


@pytest.mark.parametrize('case', CASES_PHASE)
def test_four_phase_row_split_vs_unsplit(case):
    kind, N, Cin, H, W, Cout, norm = case
    c = G.ctx()
    c.set_option('tcgen05', 1)
    c.set_option('halo_conv', 1)
    c.set_option('halo_ctas', 1)
    inp = P.make_inputs(701 + CASES_PHASE.index(case), kind, N, Cin, H, W, Cout, norm)
    outs = {}
    try:
        for k in (1, 2):
            c.set_option('halo_cs', k)
            outs[k] = P.conv_phase(**inp)
    finally:
        c.set_option('halo_cs', -1)
        c.set_option('halo_ctas', -1)
    ref, mag_in = P.reference(inp)
    _check(outs, ref, mag_in, 4 * Cin, case)


_PLAN_CODE = r'''
import sys
sys.path.insert(0, %r)
sys.path.insert(0, %r)
import gpu_util as G, test_gpu_halo_m256 as M, test_gpu_halo_phase as P
c = G.ctx()
c.set_option('tcgen05', 1)
c.set_option('halo_conv', 1)
for N in (1, 4):
    sys.stderr.write('BATCH %%d\n' %% N); sys.stderr.flush()
    M.conv_norm_ex(**M.make_inputs(5, N, 256, 64, 64, 256, 'gn', 1), ksplit=0)
    P.conv_phase(**P.make_inputs(6, 4, N, 256, 32, 32, 256, 'gn'), ksplit=0)
'''


def test_automatic_plan_splits_under_one_wave():
    """The launch log (THA4_HALO_DEBUG=2) of the automatic plan: the 64^2 256 -> 256 conv and the 32^2 four-phase
    up-sampling run as cluster pairs at batch 1 (64 CTAs each) and unsplit at batch 4 (256 CTAs)."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = _PLAN_CODE % (os.path.dirname(here), here)
    r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, env=dict(os.environ, THA4_HALO_DEBUG='2'))
    assert r.returncode == 0, r.stderr[-3000:]
    launches = {}
    for part in r.stderr.split('BATCH ')[1:]:
        n = int(part.split('\n', 1)[0])
        launches[n] = [line for line in part.splitlines() if line.startswith('halo launch:')]
    for n, want in ((1, 2), (4, 1)):
        assert any(' phases 1 ' in line for line in launches[n]) and any(' phases 4 ' in line for line in launches[n]), launches[n]
        for line in launches[n]:
            assert (' cs %d ' % want) in line, (n, line)
