"""Kernel-level parity of the default-mode teacher forward (-m gpu) in the layouts the networks run it: outputs written into
channel slices of a concatenation buffer (f16 only, or fp32 and f16), statistics of two producers accumulated into one slot
with the networks' replica counts, GroupNorm groups that straddle the boundary between the two producers, FiLM rows of the
11008-wide table at a block's offset, slice inputs and slice residuals (through the TMA residual box and without TMA
stores), the folded skip, the four-phase up-sampling conv and the RES_UP2 conv after it, the encoder-decoder bottleneck
(a stride-2 producer on the tensor-core kernel's cluster split-K writing next to the pose planes, a consumer that normalises
512 of its 528 channels), the five fused tail sites with their images read from the network input, and the attention.

Each launch is checked against an fp64 reference built from its own actual inputs (what the previous launch really wrote,
the statistics it really accumulated), with the elementwise bound of tests/teacher_forward_ref.py, so bounds never compound
along a chain.  Every buffer has guard channels around each slice (NaN in fp32 / f16 data, a sentinel in the statistics
columns and replicas outside the slot); after every launch everything outside what the launch owns must be bit-identical.
The conv cases assert the plan they target (halo kernel, cluster size, warpgroups, CTAs per SM, TMA-store bits)."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import gpu_util as G
import teacher_forward_ref as R
from tha4_b200._lib import _ptr, _ptr_array
from test_gpu_teacher_backward_kernels import _film1_layout

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
NAN = float('nan')
SENT = -7777.0
GUARD = 8                 # guard channels on each side of a buffer's data (16 bytes of f16: TMA stores stay legal)

BODY = _film1_layout(64, [1, 2, 4, 4, 4])
SMS = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 0
PLAN_SMS = 132            # the pinned plans below are those of an H100 SXM: halo_plan / tc_plan size grids by the SM count
UPSCALER = _film1_layout(32, [1, 2, 4, 8, 8, 8])


def _bits(t):
    return t.view({torch.float16: torch.int16, torch.float32: torch.int32, torch.float64: torch.int64}[t.dtype])


def _same_bits(name, a, b):
    assert torch.equal(_bits(a), _bits(b)), '%s: a value outside what the launch owns changed' % name


def _nchw(v):
    return v.permute(0, 3, 1, 2).double().cpu()


def _reps(H):
    """Statistics replicas of a tensor of H x H pixels (nets.cu make_view / make_act)."""
    tiles = ((H + 15) // 16) * ((H + 7) // 8)
    rep = 1
    while rep < 16 and rep * 32 <= tiles:
        rep *= 2
    return rep


def _act(N, H, C, dtype):
    return torch.full((N, H, H, GUARD + C + GUARD), NAN, dtype=dtype, device=DEV)


def _slot(rep, N, C):
    """Statistics buffer [rep + 1][N][C + GUARD][2]: the slot's columns of replicas 0..rep-1 zeroed, the rest sentinels."""
    st = torch.full((rep + 1, N, C + GUARD, 2), SENT, dtype=torch.float64, device=DEV)
    st[:rep, :, :C] = 0
    return st


def _stats_arg(st, c0, rep):
    return (st[:, :, c0:], st.shape[2], rep, st.stride(0))


def _check(name, out, ref, bound):
    out = out.double()
    assert torch.isfinite(out).all(), name
    ratio = ((out - ref).abs() / bound).max().item()
    print('\n%s: max |err| / bound %.3e (max |err| %.3e, max |ref| %.3e)' % (name, ratio, (out - ref).abs().max().item(),
                                                                          ref.abs().max().item()))
    assert ratio <= 1.0, (name, ratio)
    return ratio


def _f16_input(x, rep, seed):
    """A fresh f16 operand [N, H, W, C] (contiguous) and its statistics replicas [rep][N][C][2]."""
    x16 = x.half()
    st = R.split_replicas(R.stats_of(x16.double()), rep, seed).contiguous().to(DEV)
    return x16.permute(0, 2, 3, 1).contiguous().to(DEV), st


class Nin:
    def __init__(self, stats, C, groups, act, gamma, beta, film0=None, film1=None, film1_ld=0, film1_off=0):
        self.stats, self.C, self.groups, self.act = stats, C, groups, act
        self.gamma, self.beta, self.film0, self.film1_full, self.film1_ld, self.film1_off = gamma, beta, film0, film1, film1_ld, film1_off

    def sums(self):
        v, _, rep, _ = self.stats
        return v[:rep, :, :self.C].sum(0).cpu()

    def film1_rows(self):
        return None if self.film1_full is None else self.film1_full[:, self.film1_off:self.film1_off + 2 * self.C]


def _launch(kind, w, bias, x, Cin, Cout, out=None, out16=None, stats=None, res=None, res_mode=0, nin=None, skip=None, ksplit=0):
    """tha4_test_conv_forward_ex on device views (NHWC slices); returns the plan record."""
    N, H, W = x.shape[0], x.shape[1], x.shape[2]
    c = G.ctx()
    wd, bd = G.dev(w), G.dev(bias)
    ws = bs = x2 = None
    Cin2 = 0
    if skip is not None:
        ws, bs, x2 = G.dev(skip[0]), G.dev(skip[1]), skip[2]
        Cin2 = skip[0].shape[1]
    st = stats if stats is not None else (None, 0, 0, 0)
    n = nin
    keep = [G.dev(t) if t is not None else None for t in ((n.gamma, n.beta, n.film0, n.film1_full) if n else (None,) * 4)]
    f1 = keep[3][:, n.film1_off:] if n and n.film1_full is not None else None
    ist = n.stats if n else (None, 0, 0, 0)
    plan = (ctypes.c_int * 10)()
    c._call('tha4_test_conv_forward_ex', kind, _ptr(wd), _ptr(bd), Cin, Cout, _ptr(ws), _ptr(bs), Cin2, _ptr(x), x.stride(2), N, H, W,
            _ptr(x2), x2.stride(2) if x2 is not None else 0, _ptr(out), out.stride(2) if out is not None else 0,
            _ptr(out16), out16.stride(2) if out16 is not None else 0, _ptr(st[0]), st[1], st[2], ctypes.c_int64(st[3]),
            _ptr(res), res.stride(2) if res is not None else 0, res_mode, _ptr(ist[0]), ist[1], ist[2], ctypes.c_int64(ist[3]),
            n.C if n else 0, n.groups if n else 0, n.act if n else 0, _ptr(keep[0]), _ptr(keep[1]), _ptr(keep[2]), _ptr(f1),
            n.film1_ld if n else 0, ksplit, plan, c._stream())
    torch.cuda.synchronize()
    return list(plan)


def _windows(H):
    """Output windows the fp64 reference is evaluated on: all of a small map, else two 16 x 16 corners (borders and the
    interior rows and columns next to them).  A wrong stride or offset moves every pixel."""
    if H <= 32:
        return [(0, H, 0, H)]
    return [(0, 16, 0, 16), (H - 16, H, H - 24, H - 8)]


def _conv_reference(kind, w, bias, x_nchw, nin, win, res=None, skip=None, samples=None):
    """fp64 reference and bound of a 3x3 / 1x1 conv on output window win = (y0, y1, x0, x1) of the given samples."""
    s = samples if samples is not None else list(range(x_nchw.shape[0]))
    if win is None:          # the whole map (4x4 stride 2, four phases): the reference's own zero padding
        xin = x_nchw[s]
        if nin is not None:
            f1 = nin.film1_rows()
            a, e = R.normalized_operand(xin, nin.sums()[s], nin.C, nin.groups, nin.gamma, nin.beta, nin.act, nin.film0,
                                        f1[s] if f1 is not None else None)
        else:
            a, e = xin.double(), torch.zeros_like(xin.double())
        return R.conv_ref(kind, a, e, R.kernel_weights(kind, w), bias, res[s] if res is not None else None,
                          1 if res is not None else 0)
    y0, y1, x0, x1 = win
    H, W = x_nchw.shape[2], x_nchw.shape[3]
    p = 1 if kind == 0 else 0
    ya, yb, xa, xb = max(0, y0 - p), min(H, y1 + p), max(0, x0 - p), min(W, x1 + p)
    xin = x_nchw[s][:, :, ya:yb, xa:xb]
    if nin is not None:
        sums = nin.sums()[s]
        f1 = nin.film1_rows()
        a, e = R.normalized_operand(xin, sums, nin.C, nin.groups, nin.gamma, nin.beta, nin.act, nin.film0,
                                    f1[s] if f1 is not None else None, hw=H * W)
    else:
        a, e = xin.double(), torch.zeros_like(xin.double())
    pads = (xa - (x0 - p), (x1 + p) - xb, ya - (y0 - p), (y1 + p) - yb)
    a, e = F.pad(a, pads), F.pad(e, pads)
    wk = R.kernel_weights(kind, w)
    a2 = wk2 = None
    if skip is not None:
        a2 = skip[2][s][:, :, y0:y1, x0:x1]
        wk2 = R.kernel_weights(3, skip[0])
    r = res[s][:, :, y0:y1, x0:x1] if res is not None else None
    return R.conv_ref(0 if kind == 0 else 3, a, e, wk, bias, r, 1 if r is not None else 0, a2, wk2, pad=0)


def _check_launch(name, kind, w, bias, x_nchw, nin, out32, out16, stats, res=None, skip=None, samples=None):
    """Compares a launch's outputs (NHWC device views) with the reference on the windows, the f16 copy with the fp32
    output, and the statistics (all pixels) with the fp64 sums of the kernel's own output."""
    worst = 0.0
    H = x_nchw.shape[2]
    s = samples if samples is not None else list(range(x_nchw.shape[0]))
    y32 = _nchw(out32) if out32 is not None else None
    y16 = _nchw(out16) if out16 is not None else None
    for win in (_windows(H) if kind in (0, 3) else [None]):
        ref, bound = _conv_reference(kind, w, bias, x_nchw, nin, win, res, skip, s)
        y0, y1, x0, x1 = win if win is not None else (0, ref.shape[2], 0, ref.shape[3])
        if y32 is not None:
            worst = max(worst, _check(name + ' fp32', y32[s][:, :, y0:y1, x0:x1], ref, bound))
        else:
            b16 = bound + R.U16 * (ref.abs() + bound) + R.F16_FLOOR
            worst = max(worst, _check(name + ' f16', y16[s][:, :, y0:y1, x0:x1], ref, b16))
    if y32 is not None and y16 is not None:
        assert ((y16 - y32).abs() <= R.f16_copy_bound(y32)).all(), name + ': the f16 copy is not the fp32 output rounded once'
    if stats is not None:
        v, _, rep, _ = stats
        C = (out32 if out32 is not None else out16).shape[-1]
        got = v[:rep, :, :C].sum(0).cpu()
        if y32 is not None:
            ref_s, b = R.stats_of(y32), R.stats_bound(y32)
        else:
            ref_s, b = R.stats_ref_from_f16(y16)
        worst = max(worst, _check(name + ' stats', got, ref_s, b + 1e-300))
    return worst


# ------------------------------------------------------------------------------------------ U-Net concatenation chain
# (label, concat width, slice boundary ch_h, resolution, FiLM table, consumer block (up_res[j])): the concatenations whose
# 32 GroupNorm groups straddle the two producers (Morpher00 j = 5, 7; Upscaler02 j = 9 at 3 channels per group), and the
# other distinct (width, group size, boundary) of both U-Nets at a reduced resolution
CONCAT_CASES = [
    ('morpher_j5', 384, 256, 64, BODY, 'up_blocks.2.resnet_blocks.1'),
    ('morpher_j7', 192, 128, 128, BODY, 'up_blocks.3.resnet_blocks.1'),
    ('upscaler_j9', 96, 64, 256, UPSCALER, 'up_blocks.4.resnet_blocks.1'),
    ('morpher_j9', 128, 64, 64, BODY, 'up_blocks.4.resnet_blocks.1'),
    ('upscaler_j11', 64, 32, 64, UPSCALER, 'up_blocks.5.resnet_blocks.1'),
    ('morpher_j1', 512, 256, 16, BODY, 'up_blocks.0.resnet_blocks.1'),
]
CHAIN_PARAMS = [(c, 1) for c in CONCAT_CASES] + [(c, 3) for c in CONCAT_CASES] + [(CONCAT_CASES[0], 32)]

# The plan each launch of a chain is expected to take at (label, N): (kernel, cluster size, warpgroups, CTAs per SM,
# TMA-store bits) of producer A, producer B and the consumer.  Kernel 1 is the halo kernel.
PLANS = {
    ('morpher_j5', 1): [(1, 2, 2, 1, 2), (1, 2, 2, 1, 3), (1, 2, 2, 1, 3)],        # row-owning cluster pairs
    ('morpher_j7', 1): [(1, 1, 2, 1, 2), (1, 1, 2, 1, 3), (1, 1, 2, 1, 3)],        # unsplit, one CTA per SM
    ('upscaler_j9', 1): [(1, 1, 2, 2, 2), (1, 1, 2, 1, 3), (1, 1, 2, 2, 3)],
    ('morpher_j9', 1): [(1, 1, 2, 1, 2), (1, 1, 2, 1, 3), (1, 2, 2, 1, 3)],
    ('upscaler_j11', 1): [(1, 1, 2, 1, 2), (1, 1, 2, 1, 3), (1, 1, 2, 1, 3)],
    ('morpher_j1', 1): [(1, 4, 1, 1, 0), (1, 4, 1, 1, 0), (1, 8, 1, 1, 0)],        # cluster split-K, plain stores
    ('morpher_j5', 3): [(1, 1, 2, 2, 2), (1, 1, 2, 1, 3), (1, 1, 2, 2, 3)],
    ('morpher_j7', 3): [(1, 1, 2, 2, 2), (1, 1, 2, 2, 3), (1, 1, 2, 2, 3)],        # two CTAs per SM
    ('upscaler_j9', 3): [(1, 1, 2, 2, 2), (1, 1, 2, 1, 3), (1, 1, 2, 2, 3)],
    ('morpher_j9', 3): [(1, 1, 2, 1, 2), (1, 1, 2, 1, 3), (1, 2, 2, 1, 3)],
    ('upscaler_j11', 3): [(1, 1, 2, 1, 2), (1, 1, 2, 1, 3), (1, 1, 2, 1, 3)],
    ('morpher_j1', 3): [(1, 4, 1, 1, 0), (1, 4, 1, 1, 0), (1, 8, 1, 1, 0)],
    ('morpher_j5', 32): [(1, 1, 2, 2, 2), (1, 1, 2, 2, 3), (1, 1, 2, 2, 3)],
}


def _plan_key(plan):
    return (plan[0], plan[2], plan[3], plan[4], plan[6])


def _weights(g, cout, cin, k=3):
    return torch.randn(cout, cin, k, k, generator=g) * (2.0 / (cin * k * k)) ** 0.5, torch.randn(cout, generator=g) * 0.1


@pytest.mark.parametrize('case,N', CHAIN_PARAMS, ids=['%s-N%d' % (c[0], n) for c, n in CHAIN_PARAMS])
def test_unet_concat_chain(case, N):
    label, width, ch_h, S, film, block = case
    cs = width - ch_h
    g = torch.Generator().manual_seed(width + S + N)
    rep = _reps(S)
    samples = [0, N - 1] if N > 1 else [0]
    cat32, cat16 = _act(N, S, width, torch.float32), _act(N, S, width, torch.float16)
    slot = _slot(rep, N, width)
    plans = []
    worst = 0.0
    # producer A: [0, ch_h), f16 only; producer B: [ch_h, width), fp32 and f16 -- both into one statistics slot
    for which, c0, C in (('A', 0, ch_h), ('B', ch_h, cs)):
        x = torch.randn(N, C, S, S, generator=g) * 1.5 + 0.3
        xd, xst = _f16_input(x, 2, seed=C)
        gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.3
        nin = Nin((xst, C, 2, xst.stride(0)), C, 32, 2, gamma, beta)
        w, b = _weights(g, C, C)
        before32, before16, before_st = cat32.clone(), cat16.clone(), slot.clone()
        o32 = cat32[..., GUARD + c0:GUARD + c0 + C] if which == 'B' else None
        o16 = cat16[..., GUARD + c0:GUARD + c0 + C]
        st = _stats_arg(slot, c0, rep)
        plans.append(_launch(0, w, b, xd, C, C, o32, o16, st, nin=nin))
        name = '%s N %d producer %s' % (label, N, which)
        worst = max(worst, _check_launch(name, 0, w, b, _nchw(xd), nin, o32, o16, st, samples=samples))
        keep = torch.ones(width + 2 * GUARD, dtype=torch.bool, device=DEV)
        keep[GUARD + c0:GUARD + c0 + C] = False
        _same_bits(name + ' f16 buffer', cat16[..., keep], before16[..., keep])
        _same_bits(name + ' fp32 buffer', cat32[..., keep] if which == 'B' else cat32, before32[..., keep] if which == 'B' else before32)
        kst = torch.ones(slot.shape, dtype=torch.bool, device=DEV)
        kst[:rep, :, c0:c0 + C] = False
        _same_bits(name + ' statistics', slot[kst], before_st[kst])
    # consumer: conv0 of up_res[j] on the whole concatenation, GroupNorm(32) with groups across the boundary, FiLM rows of
    # the block in the full table
    off, _, total = film
    # The networks' conv0 applies no FiLM; these rows test the row stride of the full table and a per-block column offset
    # (2 x width columns from the block's own offset, moved left where they would run past the table's end)
    off = min(off[block], total - 2 * width)
    gamma, beta = torch.rand(width, generator=g) + 0.5, torch.randn(width, generator=g) * 0.3
    film0 = torch.randn(2 * width, generator=g) * 0.3
    film1 = torch.randn(N, total, generator=g) * 0.3
    nin = Nin(_stats_arg(slot, 0, rep), width, 32, 2, gamma, beta, film0, film1, total, off)
    w, b = _weights(g, ch_h, width)
    y32, y16 = _act(N, S, ch_h, torch.float32), _act(N, S, ch_h, torch.float16)
    yslot = _slot(1, N, ch_h)
    o32, o16 = y32[..., GUARD:GUARD + ch_h], y16[..., GUARD:GUARD + ch_h]
    st = _stats_arg(yslot, 0, 1)
    xin = cat16[..., GUARD:GUARD + width]
    plans.append(_launch(0, w, b, xin, width, ch_h, o32, o16, st, nin=nin))
    name = '%s N %d consumer' % (label, N)
    worst = max(worst, _check_launch(name, 0, w, b, _nchw(xin), nin, o32, o16, st, samples=samples))
    for buf in (y32, y16):
        assert torch.isnan(buf[..., :GUARD]).all() and torch.isnan(buf[..., GUARD + ch_h:]).all(), name + ': guard written'
    assert (yslot[1:] == SENT).all() and (yslot[:, :, ch_h:] == SENT).all(), name + ': statistics guard written'
    got = [_plan_key(p) for p in plans]
    print('plans %s N %d: %s (worst ratio %.3e)' % (label, N, got, worst))
    assert all(p[0] == 1 for p in plans), got                       # every launch of the chain runs on the halo kernel
    _plans_match(got, PLANS[(label, N)])


def _plans_match(got, expected):
    """The values were checked above; the plan assertion needs the SM count the plans were pinned for."""
    if SMS != PLAN_SMS:
        pytest.skip('plans are pinned for %d SMs, this GPU has %d (results were checked)' % (PLAN_SMS, SMS))
    assert got == expected, ('plans', got, expected)


# ------------------------------------------------------------------------------------------ ResBlock convs on slices
@pytest.mark.parametrize('tma_store', [1, 0])
def test_down_resblock_conv1_slice_input_and_residual(tma_store):
    """Morpher00 down_res[1].conv1 (128 -> 128 at 128^2): the block input is hs[2] = cat[7].slice(64, 128) (width 192); conv1
    adds it as its residual, read through the TMA residual box (or plain loads without TMA stores), and writes
    hs[3] = cat[6].slice(128, 128) (width 256) in fp32 and f16.  conv0 reads the block input's f16 slice with its slice of
    the statistics slot."""
    N, S, C, wi, wo = 3, 128, 128, 192, 256
    g = torch.Generator().manual_seed(700 + tma_store)
    rep = _reps(S)
    cin32, cin16 = _act(N, S, wi, torch.float32), _act(N, S, wi, torch.float16)
    slot_in = _slot(rep, N, wi)
    x = torch.randn(N, C, S, S, generator=g) * 1.5 + 0.3
    cin32[..., GUARD + 64:GUARD + wi] = x.permute(0, 2, 3, 1).to(DEV)
    cin16[..., GUARD + 64:GUARD + wi] = x.half().permute(0, 2, 3, 1).to(DEV)
    slot_in[:rep, :, 64:wi] = R.split_replicas(R.stats_of(x), rep, 5).to(DEV)
    xin16, xres = cin16[..., GUARD + 64:GUARD + wi], cin32[..., GUARD + 64:GUARD + wi]
    c = G.ctx()
    c.set_option('tma_store', tma_store)
    try:
        # conv0: GroupNorm + SiLU of the slice -> h0 (f16 only, with statistics)
        gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.3
        nin0 = Nin(_stats_arg(slot_in, 64, rep), C, 32, 2, gamma, beta)
        w0, b0 = _weights(g, C, C)
        h16 = _act(N, S, C, torch.float16)
        hslot = _slot(rep, N, C)
        o16, st = h16[..., GUARD:GUARD + C], _stats_arg(hslot, 0, rep)
        p0 = _launch(0, w0, b0, xin16, C, C, None, o16, st, nin=nin0)
        _check_launch('down conv0 tma %d' % tma_store, 0, w0, b0, _nchw(xin16), nin0, None, o16, st, samples=[0, 2])
        # conv1: norm1 + FiLM + SiLU of h0, + the block input (fp32 slice) -> the output slice of the next concatenation
        off, _, total = BODY
        gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.3
        film0, film1 = torch.randn(2 * C, generator=g) * 0.3, torch.randn(N, total, generator=g) * 0.3
        nin1 = Nin(_stats_arg(hslot, 0, rep), C, 32, 2, gamma, beta, film0, film1, total, off['down_blocks.1.res_blocks.0'])
        w1, b1 = _weights(g, C, C)
        y32, y16 = _act(N, S, wo, torch.float32), _act(N, S, wo, torch.float16)
        yslot = _slot(rep, N, wo)
        o32, o16 = y32[..., GUARD + 128:GUARD + wo], y16[..., GUARD + 128:GUARD + wo]
        st1 = _stats_arg(yslot, 128, rep)
        before = cin32.clone(), cin16.clone()
        p1 = _launch(0, w1, b1, h16[..., GUARD:GUARD + C], C, C, o32, o16, st1, res=xres, res_mode=1, nin=nin1)
        _check_launch('down conv1 tma %d' % tma_store, 0, w1, b1, _nchw(h16[..., GUARD:GUARD + C]), nin1, o32, o16, st1,
                      res=_nchw(xres), samples=[0, 2])
    finally:
        c.set_option('tma_store', 1)
    _same_bits('block input', cin32, before[0])
    _same_bits('block input f16', cin16, before[1])
    for buf in (y32, y16):
        assert torch.isnan(buf[..., :GUARD + 128]).all() and torch.isnan(buf[..., GUARD + wo:]).all(), 'guard written'
    assert (yslot[:rep, :, :128] == 0).all() and (yslot[rep:] == SENT).all() and (yslot[:, :, wo:] == SENT).all(), 'statistics guard written'
    print('plans conv0 %s conv1 %s' % (p0, p1))
    assert p0[0] == 1 and p1[0] == 1
    assert p1[6] == (7 if tma_store else 0), p1          # the residual arrives through the TMA box with its own stride


@pytest.mark.parametrize('N', [1, 3])
def test_up_resblock_folded_skip_into_concat_slice(N):
    """Morpher00 up_res[7] (192 -> 64 at 128^2, folded 1x1 skip): conv1 reads h0 and, for the skip, the whole concatenation
    cat[7] (f16, width 192); it writes cat[8].slice(0, 64) (width 128) in f16 only, with the statistics slot's first 64
    columns."""
    S, Cin2, C, wo = 128, 192, 64, 128
    g = torch.Generator().manual_seed(800 + N)
    rep = _reps(S)
    x2 = torch.randn(N, Cin2, S, S, generator=g)
    cat16 = _act(N, S, Cin2, torch.float16)
    cat16[..., GUARD:GUARD + Cin2] = x2.half().permute(0, 2, 3, 1).to(DEV)
    h = torch.randn(N, C, S, S, generator=g) * 1.5 + 0.3
    hd, hst = _f16_input(h, rep, 9)
    off, _, total = BODY
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.3
    film0, film1 = torch.randn(2 * C, generator=g) * 0.3, torch.randn(N, total, generator=g) * 0.3
    nin = Nin((hst, C, rep, hst.stride(0)), C, 32, 2, gamma, beta, film0, film1, total, off['up_blocks.3.resnet_blocks.1'])
    w, b = _weights(g, C, C)
    wsk, bsk = _weights(g, C, Cin2, 1)
    y16 = _act(N, S, wo, torch.float16)
    yslot = _slot(rep, N, wo)
    o16, st = y16[..., GUARD:GUARD + C], _stats_arg(yslot, 0, rep)
    xin2 = cat16[..., GUARD:GUARD + Cin2]
    before = cat16.clone()
    plan = _launch(0, w, b, hd, C, C, None, o16, st, nin=nin, skip=(wsk, bsk, xin2))
    bias = (b + bsk).float()                                 # conv_make_fold's summed bias (one fp32 addition)
    _check_launch('folded skip N %d' % N, 0, w, bias, _nchw(hd), nin, None, o16, st, skip=(wsk, bsk, x2.half().double()),
                  samples=[0, N - 1])
    _same_bits('skip input', cat16, before)
    assert torch.isnan(y16[..., :GUARD]).all() and torch.isnan(y16[..., GUARD + C:]).all(), 'guard written'
    assert (yslot[:rep, :, C:wo] == 0).all() and (yslot[:, :, wo:] == SENT).all() and (yslot[rep:] == SENT).all(), 'statistics guard written'
    print('plan', plan)
    assert plan[0] == 1 and plan[8] == 1, plan


# ------------------------------------------------------------------------------------------ up-sampling block
@pytest.mark.parametrize('N', [1, 3])
def test_up_sampling_block_into_concat_slice(N):
    """Morpher00 up_us at 32^2 -> 64^2 (256 channels): conv0 is the four-phase nearest-x2 + 3x3 conv (GroupNorm + SiLU of
    its fp32 + f16 input pending), written here f16-only into a slice of a wider buffer (four-phase launches store without
    TMA, so this is the plain-store path with ld > C); conv1 reads that slice with FiLM at the block's offset, adds the
    block input through RES_UP2 (a slice of a wider fp32 buffer), and writes f16_only(cat[j+1].slice(0, 256)) of the
    384-wide concatenation."""
    S, C, wc = 32, 256, 384
    g = torch.Generator().manual_seed(1100 + N)
    x = torch.randn(N, C, S, S, generator=g) * 1.5 + 0.3
    xb32, xb16 = _act(N, S, C + 64, torch.float32), _act(N, S, C + 64, torch.float16)
    xb32[..., GUARD + 64:GUARD + 64 + C] = x.permute(0, 2, 3, 1).to(DEV)
    xb16[..., GUARD + 64:GUARD + 64 + C] = x.half().permute(0, 2, 3, 1).to(DEV)
    rin = _reps(S)
    xslot = _slot(rin, N, C)
    xslot[:rin, :, :C] = R.split_replicas(R.stats_of(x), rin, 11).to(DEV)
    x16v, x32v = xb16[..., GUARD + 64:GUARD + 64 + C], xb32[..., GUARD + 64:GUARD + 64 + C]
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.3
    nin0 = Nin(_stats_arg(xslot, 0, rin), C, 32, 2, gamma, beta)
    w0, b0 = _weights(g, C, C)
    rep = _reps(2 * S)
    hb = _act(N, 2 * S, C + 32, torch.float16)
    hslot = _slot(rep, N, C)
    h16, st0 = hb[..., GUARD + 32:GUARD + 32 + C], _stats_arg(hslot, 0, rep)
    p0 = _launch(4, w0, b0, x16v, C, C, None, h16, st0, nin=nin0)
    _check_launch('up conv0 four-phase N %d' % N, 4, w0, b0, _nchw(x16v), nin0, None, h16, st0)
    assert torch.isnan(hb[..., :GUARD + 32]).all() and torch.isnan(hb[..., GUARD + 32 + C:]).all(), 'four-phase guard written'
    assert (hslot[:, :, C:] == SENT).all() and (hslot[rep:] == SENT).all()
    off, _, total = BODY
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.3
    film0, film1 = torch.randn(2 * C, generator=g) * 0.3, torch.randn(N, total, generator=g) * 0.3
    nin1 = Nin(st0, C, 32, 2, gamma, beta, film0, film1, total, off['up_blocks.2.upsample'])
    w1, b1 = _weights(g, C, C)
    cat16 = _act(N, 2 * S, wc, torch.float16)
    cslot = _slot(rep, N, wc)
    o16, st1 = cat16[..., GUARD:GUARD + C], _stats_arg(cslot, 0, rep)
    before = xb32.clone()
    p1 = _launch(0, w1, b1, h16, C, C, None, o16, st1, res=x32v, res_mode=2, nin=nin1)
    res_up = F.interpolate(_nchw(x32v), scale_factor=2, mode='nearest')
    _check_launch('up conv1 RES_UP2 N %d' % N, 0, w1, b1, _nchw(h16), nin1, None, o16, st1, res=res_up, samples=[0, N - 1])
    _same_bits('block input', xb32, before)
    assert torch.isnan(cat16[..., :GUARD]).all() and torch.isnan(cat16[..., GUARD + C:]).all(), 'concat guard written'
    assert (cslot[:rep, :, C:wc] == 0).all() and (cslot[:, :, wc:] == SENT).all() and (cslot[rep:] == SENT).all()
    print('plans conv0 %s conv1 %s' % (p0, p1))
    assert p0[0] == 1 and p0[5] == 4 and p0[6] == 0, p0          # four-phase halo launch, plain stores
    assert p1[0] == 1 and p1[6] & 4 == 0, p1                     # RES_UP2 never comes through the residual box
    _plans_match([_plan_key(p0), _plan_key(p1)], UP_PLANS[N])


UP_PLANS = {1: [(1, 2, 2, 1, 0), (1, 2, 2, 1, 2)],      # four phases on a row-owning cluster pair; conv1 likewise
            3: [(1, 1, 2, 2, 0), (1, 1, 2, 2, 2)]}      # two CTAs per SM


# ------------------------------------------------------------------------------------------ encoder-decoder bottleneck
@pytest.mark.parametrize('N', [1, 3])
def test_encdec_bottleneck(N):
    """The decomposer's down_[3] (4x4 stride 2, 256 -> 512, 32^2 -> 16^2, InstanceNorm + ReLU of its input pending) on the
    tensor-core kernel's cluster split-K: f16 only into bin16.slice(0, 512) of the 528-wide buffer whose pose planes
    [512, 528) were tiled in before and must survive, statistics into their own 512-column slot.  Then bott0_ reads all 528
    channels with only the first 512 normalised (InstanceNorm + ReLU), the pose planes passed through raw."""
    S, Ci, C, P = 32, 256, 512, 16
    b = S // 2
    g = torch.Generator().manual_seed(1200 + N)
    x = torch.randn(N, Ci, S, S, generator=g) * 1.5 + 0.3
    xd, xst = _f16_input(x, _reps(S), seed=12)
    gamma, beta = torch.rand(Ci, generator=g) + 0.5, torch.randn(Ci, generator=g) * 0.3
    nin = Nin((xst, Ci, _reps(S), xst.stride(0)), Ci, 0, 1, gamma, beta)
    w, bias = _weights(g, C, Ci, 4)
    bin16 = _act(N, b, C + P, torch.float16)
    pose = torch.randn(N, P, generator=g)
    bin16[..., GUARD + C:GUARD + C + P] = pose.half().view(N, 1, 1, P).expand(N, b, b, P).to(DEV)
    rep = _reps(b)
    slot = _slot(rep, N, C)
    o16, st = bin16[..., GUARD:GUARD + C], _stats_arg(slot, 0, rep)
    before = bin16.clone()
    p0 = _launch(1, w, bias, xd, Ci, C, None, o16, st, nin=nin)
    _check_launch('bottleneck producer N %d' % N, 1, w, bias, _nchw(xd), nin, None, o16, st)
    keep = torch.ones(C + P + 2 * GUARD, dtype=torch.bool, device=DEV)
    keep[GUARD:GUARD + C] = False
    _same_bits('pose planes and guards', bin16[..., keep], before[..., keep])
    assert (slot[:, :, C:] == SENT).all() and (slot[rep:] == SENT).all()
    assert p0[0] == 2 and p0[9] == 1, p0                         # tensor-core kernel, K split over a cluster
    # bott0_: 528 -> 512, InstanceNorm + ReLU on the first 512 channels only
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.3
    nin1 = Nin(st, C, 0, 1, gamma, beta)
    w1, b1 = _weights(g, C, C + P)
    y32 = _act(N, b, C, torch.float32)
    yslot = _slot(1, N, C)
    o32, st1 = y32[..., GUARD:GUARD + C], _stats_arg(yslot, 0, 1)
    xin = bin16[..., GUARD:GUARD + C + P]
    p1 = _launch(0, w1, b1, xin, C + P, C, o32, None, st1, nin=nin1)
    _check_launch('bottleneck consumer N %d' % N, 0, w1, b1, _nchw(xin), nin1, o32, None, st1)
    assert torch.isnan(y32[..., :GUARD]).all() and torch.isnan(y32[..., GUARD + C:]).all(), 'guard written'
    print('plans producer %s consumer %s' % (p0, p1))
    _plans_match([_plan_key(p0) + (p0[9],), _plan_key(p1) + (p1[9],)], BOTTLENECK_PLANS[N])


# (kernel, cluster size, warpgroups, CTAs per SM, TMA-store bits, tensor-core split plan): the producer on the tensor-core
# kernel's cluster split-K, bott0_ on a 4-way halo cluster split
BOTTLENECK_PLANS = {1: [(2, 0, 0, 0, 0, 1), (1, 4, 1, 1, 0, 0)], 3: [(2, 0, 0, 0, 0, 1), (1, 4, 1, 1, 0, 0)]}


# ------------------------------------------------------------------------------------------ attention
@pytest.mark.parametrize('N', [1, 3, 32])
@pytest.mark.parametrize('mode', ['peaked', 'uniform'])
@pytest.mark.parametrize('strict', [0, 1])
def test_attention_forward(N, mode, strict):
    """Default mode: mma.sync on f16 q, k, P and v; strict: fp32.  Bound: S carries the f16 rounding of q and k (2 u16 of
    |q| . |k|) and its fp32 sum; P the error of S - max (both terms), of the exponential and of its f16 rounding; the output
    the error of P against |v|, the f16 rounding of v and the fp32 sums over 256 keys."""
    g = torch.Generator().manual_seed(900 + N + len(mode))
    C, heads = 256, 8
    qkv = torch.randn(N, 3 * C, 16, 16, generator=g)
    if mode == 'peaked':
        qkv[:, :2 * C] *= 3.0
    else:
        qkv[:, C:2 * C] = qkv[:, C:2 * C, :1, :1].expand(N, C, 16, 16)
    ref = R.attention_ref(qkv.double(), heads)
    b, L, ch = N, 256, C // heads
    s2 = 1.0 / ch ** 0.5
    q, k, v = [t.reshape(b * heads, ch, L).transpose(1, 2) for t in qkv.double().reshape(b, 3 * C, L).chunk(3, dim=1)]
    P = torch.softmax(s2 * q @ k.transpose(1, 2), -1)
    Sabs = s2 * q.abs() @ k.abs().transpose(1, 2)
    ulo = R.U32 if strict else R.U16
    rel_p = (2 * ulo + 64 * R.U32) * (Sabs + Sabs.amax(-1, keepdim=True)) + 2 * ulo + 300 * R.U32
    e = (P * rel_p) @ v.abs() + (2 * ulo + 256 * R.U32) * (P @ v.abs())
    bound = e.transpose(1, 2).reshape(b, C, 16, 16)
    c = G.ctx()
    c.set_option('strict', strict)
    try:
        out = G.attention(qkv, heads)
    finally:
        c.set_option('strict', 0)
    _check('attention N %d %s strict %d' % (N, mode, strict), out, ref, bound)


# ------------------------------------------------------------------------------------------ fused tail
# The five sites (kind, C, S, groups, act, network input width, image0 offset, image1 offset or None, head couts in tail.cu
# order, which heads have a bias): Morpher00 and Upscaler02 (image0 = x0.slice(0, 4) of their 4- / 16-channel input), the
# decomposer and the face morpher (x0.slice(0, 4) of a 4-channel input), the combiner (image0 = x0.slice(4, 4), image1 =
# x0.slice(0, 4) of its 8-channel input)
TAIL_CASES = [(0, 64, 256, 32, 2, 4, 0, None, [7], [True]), (0, 32, 512, 32, 2, 16, 0, None, [7], [True]),
              (1, 64, 128, 0, 1, 4, 0, None, [1, 4, 1, 4], [True] * 4),
              (2, 64, 128, 0, 1, 8, 4, 0, [2, 1, 4, 1], [False, True, True, True]),
              (3, 64, 192, 0, 1, 4, 0, None, [2, 4, 1, 4, 1], [False, True, True, True, True])]


def _tail_ex(kind, fd, st, rep, gamma, beta, groups, act, ws, bs, img0, sn0, img1, sn1, g0, g1, N, C, S):
    c = G.ctx()
    outs = [torch.full((N, ch, S, S), NAN, device=DEV) for ch in G.TAIL_OUT_SPECS[kind]]
    hw = G.dev(torch.cat([w.reshape(-1) for w in ws]))
    hb = G.dev(torch.cat([(b if b is not None else torch.zeros(w.shape[0])) for w, b in zip(ws, bs)]))
    couts = (ctypes.c_int * len(ws))(*[w.shape[0] for w in ws])
    c._call('tha4_test_tail_ex', kind, _ptr(fd), N, C, S, _ptr(st), C, rep, ctypes.c_int64(st.stride(0)), _ptr(gamma), _ptr(beta),
            groups, act, _ptr(hw), _ptr(hb), couts, len(ws), _ptr(img0), ctypes.c_int64(sn0), _ptr(img1), ctypes.c_int64(sn1),
            _ptr(g0), g0.stride(2) if g0 is not None else 0, _ptr(g1), g1.stride(2) if g1 is not None else 0,
            _ptr_array(outs), c._stream())
    torch.cuda.synchronize()
    for o in outs:
        assert torch.isfinite(o).all()
    return outs


def _tail_weights(g, kind, C, couts, has_b):
    """Trained-like head scales: colour ~0.3, warps of a few pixels (grid heads 0.01 of the colour heads)."""
    ws, bs = [], []
    for co, hb in zip(couts, has_b):
        w = torch.randn(co, C, 3, 3, generator=g) / (9 * C) ** 0.5 * 0.3
        if not hb:
            w = w * 0.03
        ws.append(w)
        bs.append(0.1 * torch.randn(co, generator=g) if hb else None)
    if kind == 0:
        ws[0][4:6] *= 0.03
    return ws, bs


def _smooth_images(g, N, S):
    """N distinct smooth RGBA images in [-1, 1] (low-frequency noise upsampled): the warp's Lipschitz bound stays small."""
    lo = torch.rand(N, 4, S // 16, S // 16, generator=g) * 2 - 1
    return F.interpolate(lo, size=(S, S), mode='bilinear', align_corners=False).contiguous()


@pytest.mark.parametrize('case', TAIL_CASES, ids=['kind%d-%d' % (c[0], c[2]) for c in TAIL_CASES])
def test_tail_site(case):
    """One tail site at N = 3 on 16 statistics replicas, its images read through per-sample distinct slices of the
    interleaved network input, against the fp64 reference ops with their bound.  The reads of the NCHW images are the same
    arithmetic (identical outputs); one stored image at batch stride 0 gives the outputs of that image stored per sample; the
    16 replicas give the outputs of their sum in one."""
    kind, C, S, groups, act, xw, o0, o1, couts, has_b = case
    N = 3
    g = torch.Generator().manual_seed(1000 + kind + S)
    feat = torch.randn(N, C, S, S, generator=g) * 1.5 + 0.3
    fd, st16 = _f16_input(feat, 16, seed=S)
    st1 = st16.sum(0, keepdim=True).contiguous()
    gam, bet = 1.0 + 0.2 * torch.randn(C, generator=g), 0.2 * torch.randn(C, generator=g)
    gamma, beta = G.dev(gam), G.dev(bet)
    ws, bs = _tail_weights(g, kind, C, couts, has_b)
    img0, img1 = _smooth_images(g, N, S), _smooth_images(g, N, S)
    x0 = torch.randn(N, S, S, xw, generator=g)                           # the network input, NHWC; other channels random
    x0[..., o0:o0 + 4] = img0.permute(0, 2, 3, 1)
    if o1 is not None:
        x0[..., o1:o1 + 4] = img1.permute(0, 2, 3, 1)
    x0 = x0.to(DEV)
    i0d, i1d = G.dev(img0), G.dev(img1) if o1 is not None else None
    args = (gamma, beta, groups, act, ws, bs)
    sn = 4 * S * S
    g1 = x0[..., o1:o1 + 4] if o1 is not None else None
    gather = _tail_ex(kind, fd, st16, 16, *args, i0d, sn, i1d, sn, x0[..., o0:o0 + 4], g1, N, C, S)
    fallback = _tail_ex(kind, fd, st16, 16, *args, i0d, sn, i1d, sn, None, None, N, C, S)
    folded1 = _tail_ex(kind, fd, st1, 1, *args, i0d, sn, i1d, sn, x0[..., o0:o0 + 4], g1, N, C, S)
    refs = R.tail_ref(kind, fd.permute(0, 3, 1, 2).double().cpu(), st16.sum(0).cpu(), groups, act, gam, bet, ws, bs, img0,
                      img1 if o1 is not None else None)
    worst = 0.0
    for i, (a, b, d, (ref, bound)) in enumerate(zip(gather, fallback, folded1, refs)):
        _same_bits('tail %d output %d: gather vs NCHW reads' % (kind, i), a, b)
        err = (a - d).abs().max().item() / max(1.0, d.abs().max().item())
        assert err <= 1e-4, ('tail %d output %d: 16 replicas vs their sum' % (kind, i), err)
        worst = max(worst, _check('tail %d S %d output %d' % (kind, S, i), a.cpu(), ref, bound + 1e-30))
    print('tail %d S %d worst ratio %.3e' % (kind, S, worst))
    # batch stride 0: one stored image for every sample
    one0 = G.dev(img0[:1])
    one1 = G.dev(img1[:1]) if o1 is not None else None
    rep0 = G.dev(img0[:1].expand(N, 4, S, S))
    rep1 = G.dev(img1[:1].expand(N, 4, S, S)) if o1 is not None else None
    stride0 = _tail_ex(kind, fd, st16, 16, *args, one0, 0, one1, 0, None, None, N, C, S)
    stored = _tail_ex(kind, fd, st16, 16, *args, rep0, sn, rep1, sn, None, None, N, C, S)
    for i, (a, b) in enumerate(zip(stride0, stored)):
        _same_bits('tail %d output %d: batch stride 0 vs stored per sample' % (kind, i), a, b)
