"""Kernel-level parity of the teachers' parameter-gradient reductions (-m gpu), each through the launcher the network
backwards call: the GroupNorm (+FiLM) fold of the U-Nets (d gamma, d beta and the time FiLM's d(film0)), the InstanceNorm
fold of the encoder-decoders, the conv bias sums (with the copy the skip and coarse_image_conv biases get), the dense
layers' weight gradients at every call site of the pose and time MLPs, the encoder-decoders' head biases through their
offset map, and their d(pose) sum.

These kernels accumulate in fp64 in a fixed order, so the references are tight: fp64 autograd for the norm folds with a
bound on the fp32 terms the backward reduction sums, and elsewhere the exact sum rounded once to fp32.  On dyadic inputs
(few-bit multiples of a power of two) every fp64 partial sum is exact, so the outputs must equal the rounded exact sums
bitwise, which catches a dropped or doubled element that a tolerance would blur.  Inputs sit in the layouts the networks
use (f16 tapes with statistics replicas, strided views with NaN guard columns, FiLM tables at a block's offset) and outputs
inside NaN-guarded flat buffers, which must keep their guards."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import gpu_util as G
import teacher_backward_ref as R
from test_gpu_teacher_backward_kernels import BODY_COUT, BODY_FILM1, BODY_FILM1_OFF, UPSCALER_FILM1, _film1_layout, _place, _stats_dev
from tha4_b200._lib import _ptr

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
NAN = float('nan')
U = R.U32
UPSCALER_FILM1_OFF, UPSCALER_COUT, _ = _film1_layout(32, [1, 2, 4, 8, 8, 8])


def _ratio(name, out, ref, bound):
    out = out.double().cpu()
    assert torch.isfinite(out).all(), name
    r = ((out - ref.double().cpu()).abs() / bound.double().cpu()).max().item()
    print('\n%s: max |err| / bound %.3e' % (name, r))
    assert r <= 1.0, (name, r)
    return r


def _bitwise(name, out, ref32):
    out, ref32 = out.cpu(), ref32.cpu()
    bad = (out != ref32).sum().item()
    assert bad == 0, '%s: %d of %d values differ from the rounded exact sum' % (name, bad, out.numel())


def _slot(n, lead=5, tail=7):
    """A NaN-filled flat buffer with an n-float output slot inside it; returns (buffer, slot view)."""
    buf = torch.full((lead + n + tail,), NAN, device=DEV)
    return buf, buf[lead:lead + n]


def _outside_nan(name, buf, lo, hi):
    assert torch.isnan(torch.cat([buf[:lo], buf[hi:]])).all(), '%s: written outside its slot' % name


def _dyadic(shape, g, bits=10, device='cpu'):
    """Odd multiples of 2^-bits in (-1, 1): never zero, exact in f16 / fp32, and fp64 sums of up to 2^40 of them are exact."""
    k = torch.randint(-(1 << (bits - 1)), 1 << (bits - 1), shape, generator=g) * 2 + 1
    return (k.double() * 2.0 ** -bits).float().to(device)


# ------------------------------------------------------------------------------------------ GroupNorm (+FiLM) fold
def gn_param_ref(x, groups, gamma, beta, dy, act, film0, film1, dy_pool):
    """(d gamma, d beta, d film0 or None) by fp64 autograd of out = pool?(act(FiLM1(FiLM0(GroupNorm(x))))) with gamma, beta,
    film0 and film1 as leaves, and their bounds.  The kernels form S1 = sum dz, S2 = sum dz xhat per (n, c) (fp32 per thread
    over at most 32 pixels, fp64 beyond) from fp32 affine coefficients; the bound on each is that of the d(film1) check in
    tests/teacher_backward_ref.py (64 u of the absolute terms sum |dz| and sum |dz| xa, plus the SiLU' error of the fp32
    affine), and the fold multiplies it by the factors' magnitudes, plus 4 u of the folded absolute terms for the fp64
    products and the final rounding to fp32."""
    x = x.double()
    N, C, H, W = x.shape
    leaves = [t.double().clone().requires_grad_() if t is not None else None for t in (gamma, beta, film0, film1)]
    gl, bl, f0l, f1l = leaves
    h = F.group_norm(x, groups, gl, bl, eps=R.EPS)
    if film0 is not None:
        h = h * (1 + f0l[:C].view(1, C, 1, 1)) + f0l[C:].view(1, C, 1, 1)
    if film1 is not None:
        h = h * (1 + f1l[:, :C].view(N, C, 1, 1)) + f1l[:, C:].view(N, C, 1, 1)
    y = F.silu(h) if act == 2 else h
    (F.avg_pool2d(y, 2) if dy_pool else y).backward(dy.double())

    mean, rstd = R._group_moments(x, groups)
    s0, s1, b0, b1 = R._film_factors(N, C, film0, film1)
    M = s0 * s1
    dyu = 0.25 * F.interpolate(dy.double(), scale_factor=2, mode='nearest') if dy_pool else dy.double()
    hd = h.detach()
    if act == 2:
        sg = torch.sigmoid(hd)
        dz = dyu * sg * (1 + hd * (1 - sg))
    else:
        dz = dyu
    xa = R._bcast(rstd) * (x.abs() + R._bcast(mean.abs()))
    K = rstd * gamma.double().view(1, C) * M
    hs = R._bcast(K.abs()) * (x.abs() + R._bcast(mean.abs())) + R._bcast(beta.double().abs().view(1, C) * M.abs() + b0.abs() * s1.abs() + b1.abs())
    e_dz = dyu.abs() * (0.5 * 16 * U * hs + 8 * U) if act == 2 else torch.zeros_like(dyu)
    T1, T2 = dz.abs().sum((2, 3)), (dz.abs() * xa).sum((2, 3))
    dS1 = 64 * U * T1 + e_dz.sum((2, 3))
    dS2 = 64 * U * T2 + (e_dz * xa).sum((2, 3))
    g_, b_ = gamma.double().abs().view(1, C), beta.double().abs().view(1, C)
    bg = (M.abs() * dS2 + 4 * U * M.abs() * T2).sum(0)
    bb = (M.abs() * dS1 + 4 * U * M.abs() * T1).sum(0)
    out = [gl.grad.detach(), bl.grad.detach(), f0l.grad.detach() if film0 is not None else None]
    bounds = [bg, bb, None]
    if film0 is not None:
        bs0 = (s1.abs() * (g_ * dS2 + b_ * dS1) + 4 * U * s1.abs() * (g_ * T2 + b_ * T1)).sum(0)
        bb0 = (s1.abs() * dS1 + 4 * U * s1.abs() * T1).sum(0)
        bounds[2] = torch.cat([bs0, bb0])
    return out, bounds


# (C, H, N, role, FiLM table): role = the normalisation's call in res_bwd / attn_bwd (unet_backward.cu): 'film' norm1 with
# both FiLMs and SiLU, 'down' a down-sampling block's norm0 (dy pooled), 'norm0' SiLU without FiLM, 'attn' no activation
GN_FOLD_CASES = [(32, 64, 1, 'film', 'upscaler'), (64, 64, 3, 'film', 'body'), (128, 32, 6, 'film', 'upscaler'),
                 (256, 16, 6, 'film', 'body'), (256, 16, 1, 'film', 'upscaler'), (32, 128, 3, 'down', None),
                 (64, 64, 6, 'down', None), (96, 32, 1, 'norm0', None), (192, 32, 3, 'norm0', None), (384, 16, 6, 'norm0', None),
                 (512, 16, 3, 'norm0', None), (256, 16, 1, 'attn', None), (512, 16, 6, 'attn', None), (384, 32, 3, 'attn', None)]


def _film_block(table, C):
    off, cout = (BODY_FILM1_OFF, BODY_COUT) if table == 'body' else (UPSCALER_FILM1_OFF, UPSCALER_COUT)
    name = [k for k in off if cout[k] == C][-1]
    return off[name], (BODY_FILM1 if table == 'body' else UPSCALER_FILM1)


def _gn_fold_call(c, xv, xld, x_f16, N, C, H, st, rep, gd, bd, f0d, f1d, film1_ld, off, act, dyv, dyld, dy_pool, dxv, dxld,
                  dgv, dbv, df0v, df0_ld, accumulate):
    dfb = torch.full((N, film1_ld), -7777.0, device=DEV) if f1d is not None else None
    c._call('tha4_test_group_norm_param_grads', _ptr(xv), x_f16, xld, N, C, H, H, 32, _ptr(st), rep, C, _ptr(gd), _ptr(bd),
            _ptr(f0d), _ptr(f1d), film1_ld, off, act, _ptr(dyv), dyld, int(dy_pool), _ptr(None), 0, 0, _ptr(None), 0,
            _ptr(dxv), dxld, _ptr(dfb), film1_ld, _ptr(dgv), _ptr(dbv), _ptr(df0v), df0_ld, off, accumulate, c._stream())
    torch.cuda.synchronize()


@pytest.mark.parametrize('C,H,N,role,table', GN_FOLD_CASES)
@pytest.mark.parametrize('x_f16', [0, 1])
def test_group_norm_param_fold(C, H, N, role, table, x_f16):
    g = torch.Generator().manual_seed(7 * C + H + N + x_f16 + len(role))
    x = torch.randn(N, C, H, H, generator=g) * 2 + 0.5
    if x_f16:
        x = x.half().float()
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.3
    film = role == 'film'
    act = 0 if role == 'attn' else 2
    dy_pool = role == 'down'
    off, film1_ld = _film_block(table, C) if film else (0, 2 * C)
    film0 = torch.randn(2 * C, generator=g) * 0.3 if film else None          # the block's time FiLM at t = 0 (ResBlockW::film0)
    film1_full = torch.randn(N, film1_ld, generator=g) * 0.3 if film else None
    film1 = film1_full[:, off:off + 2 * C] if film else None
    hd = H // 2 if dy_pool else H
    dy = torch.randn(N, C, hd, hd, generator=g)
    (ref_g, ref_b, ref_f0), (bd_g, bd_b, bd_f0) = gn_param_ref(x, 32, gamma, beta, dy, act, film0, film1, dy_pool)

    c = G.ctx()
    xb, xv = _place(x, C + 8, 4, NAN, torch.float16 if x_f16 else torch.float32)
    dyb, dyv = _place(dy, C + 32, 0, NAN)
    gd, bd = G.dev(gamma), G.dev(beta)
    f0d = G.dev(film0) if film else None
    f1d = G.dev(film1_full) if film else None
    dxb = torch.full((N, H, H, C + 12), NAN, device=DEV)
    dxv = dxb[..., 4:4 + C]
    worst, first = 0.0, None
    for rep in (1, 2, 16):
        st = _stats_dev(x, rep, seed=rep + C)
        gbuf, dgv = _slot(C)
        bbuf, dbv = _slot(C)
        f0buf = torch.full((film1_ld,), NAN, device=DEV) if film else None
        df0v = f0buf if film else None
        args = (c, xv, xb.shape[-1], x_f16, N, C, H, st, rep, gd, bd, f0d, f1d, film1_ld, off, act, dyv, dyb.shape[-1], dy_pool,
                dxv, dxb.shape[-1])
        _gn_fold_call(*args, dgv, dbv, df0v, film1_ld, 0)
        name = 'GN fold C %d %d^2 N %d %s f16 %d rep %d' % (C, H, N, role, x_f16, rep)
        worst = max(worst, _ratio(name + ' d(gamma)', dgv, ref_g, bd_g), _ratio(name + ' d(beta)', dbv, ref_b, bd_b))
        _outside_nan(name + ' d(gamma)', gbuf, 5, 5 + C)
        _outside_nan(name + ' d(beta)', bbuf, 5, 5 + C)
        got = [dgv.clone(), dbv.clone()]
        if film:
            worst = max(worst, _ratio(name + ' d(film0)', f0buf[off:off + 2 * C], ref_f0, bd_f0))
            _outside_nan(name + ' d(film0)', f0buf, off, off + 2 * C)
            got.append(f0buf[off:off + 2 * C].clone())
        if first is None:
            first = got
        # accumulate = 1 onto a finite prefill adds the same gradient; d(film0) is written again, never accumulated, and
        # nothing outside its 2C columns changes
        pre_g, pre_b = torch.randn(C, generator=g).to(DEV), torch.randn(C, generator=g).to(DEV)
        dgv.copy_(pre_g)
        dbv.copy_(pre_b)
        if film:
            f0buf.fill_(-7777.0)
        _gn_fold_call(*args, dgv, dbv, df0v, film1_ld, 1)
        _bitwise(name + ' accumulate d(gamma)', dgv, pre_g + got[0])
        _bitwise(name + ' accumulate d(beta)', dbv, pre_b + got[1])
        if film:
            _bitwise(name + ' d(film0) overwritten', f0buf[off:off + 2 * C], got[2])
            rest = torch.cat([f0buf[:off], f0buf[off + 2 * C:]])
            assert (rest == -7777.0).all(), name + ': d(film0) written outside the block columns'
    # the replicas change only the fp64 statistics' summation; a second run of rep 16 repeats the first bitwise
    gbuf, dgv = _slot(C)
    bbuf, dbv = _slot(C)
    _gn_fold_call(c, xv, xb.shape[-1], x_f16, N, C, H, _stats_dev(x, 16, seed=16 + C), 16, gd, bd, f0d, f1d, film1_ld, off, act,
                  dyv, dyb.shape[-1], dy_pool, dxv, dxb.shape[-1], dgv, dbv, None, film1_ld, 0)
    assert torch.equal(dgv, got[0]) and torch.equal(dbv, got[1]), 'GN fold: two runs differ'
    print('worst ratio %.3e' % worst)


# ------------------------------------------------------------------------------------------ InstanceNorm fold
IN_CASES = [(64, 192, 1, 1), (128, 64, 2, 1), (256, 48, 2, 1), (256, 32, 2, 0), (512, 16, 2, 1), (512, 24, 2, 1), (512, 16, 3, 0)]


def in_param_ref(x, gamma, beta, dy, act, mask):
    """(d gamma, d beta) by fp64 autograd of act(InstanceNorm(x)) (ReLU through the kernel's own mask) and their bounds:
    sum_n of the per-(n, c) bounds on S2 / S1 (64 u of sum |dz| xa / sum |dz|: fp32 per thread, fp64 beyond), plus 4 u of
    the absolute sums for the fold and its rounding."""
    x = x.double()
    N, C = x.shape[:2]
    gl, bl = gamma.double().clone().requires_grad_(), beta.double().clone().requires_grad_()
    h = F.instance_norm(x, weight=gl, bias=bl, eps=R.EPS)
    (h * mask if act else h).backward(dy.double())
    mean, rstd = R._group_moments(x, C)
    xa = R._bcast(rstd) * (x.abs() + R._bcast(mean.abs()))
    dz = dy.double().abs() * (mask if act else 1.0)
    T1, T2 = dz.sum((2, 3)), (dz * xa).sum((2, 3))
    return (gl.grad.detach(), bl.grad.detach()), (68 * U * T2.sum(0), 68 * U * T1.sum(0))


@pytest.mark.parametrize('C,H,N,act', IN_CASES)
@pytest.mark.parametrize('x_f16', [0, 1])
def test_norm_param_fold(C, H, N, act, x_f16):
    g = torch.Generator().manual_seed(11 * C + H + act + x_f16)
    x = torch.randn(N, C, H, H, generator=g) * 2 + 0.5
    if x_f16:
        x = x.half().float()
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.3
    dy = torch.randn(N, C, H, H, generator=g)
    mask = None
    if act:
        mask, amb = R.relu_mask_and_ambiguous(x, gamma, beta)
        dy = torch.where(amb, torch.zeros_like(dy), dy)
    (ref_g, ref_b), (bd_g, bd_b) = in_param_ref(x, gamma, beta, dy, act, mask)
    c = G.ctx()
    xb, xv = _place(x, C + 8, 4, NAN, torch.float16 if x_f16 else torch.float32)
    dyb, dyv = _place(dy, C + 16, 0, NAN)
    gd, bd = G.dev(gamma), G.dev(beta)
    rep = {64: 16, 128: 2, 256: 1, 512: 16}[C]
    st = _stats_dev(x, rep, seed=C)
    dxb = torch.full((N, H, H, C + 8), NAN, device=DEV)
    dxv = dxb[..., 4:4 + C]

    def run(dgv, dbv, accumulate):
        c._call('tha4_test_norm_param_grads', _ptr(xv), x_f16, xb.shape[-1], N, C, H, H, _ptr(st), rep, C, _ptr(gd), _ptr(bd), act,
                _ptr(dyv), dyb.shape[-1], _ptr(dxv), dxb.shape[-1], _ptr(dgv), _ptr(dbv), accumulate, c._stream())
        torch.cuda.synchronize()
    gbuf, dgv = _slot(C)
    bbuf, dbv = _slot(C)
    run(dgv, dbv, 0)
    name = 'IN fold C %d %d^2 N %d act %d f16 %d' % (C, H, N, act, x_f16)
    _ratio(name + ' d(gamma)', dgv, ref_g, bd_g)
    _ratio(name + ' d(beta)', dbv, ref_b, bd_b)
    _outside_nan(name, gbuf, 5, 5 + C)
    _outside_nan(name, bbuf, 5, 5 + C)
    got = [dgv.clone(), dbv.clone()]
    pre_g, pre_b = torch.randn(C, generator=g).to(DEV), torch.randn(C, generator=g).to(DEV)
    dgv.copy_(pre_g)
    dbv.copy_(pre_b)
    run(dgv, dbv, 1)
    _bitwise(name + ' accumulate d(gamma)', dgv, pre_g + got[0])
    _bitwise(name + ' accumulate d(beta)', dbv, pre_b + got[1])
    run(dgv, dbv, 0)
    assert torch.equal(dgv, got[0]) and torch.equal(dbv, got[1]), name + ': two runs differ'


# ------------------------------------------------------------------------------------------ conv bias sums
# pixel counts around the 4096-pixel chunk of the partial sums, and the networks' maps; (C, ld): the last.2 head's 7 channels
# inside the 16-channel dh, contiguous dz, a dcat-like slice, a slice of a wide buffer, the attention qkv
CS_PIXELS = [256, 4095, 4096, 4097, 3 * 64 * 64, 5 * 192 * 192, 2 * 512 * 512]
CS_LAYOUTS = [(7, 16), (64, 64), (96, 100), (512, 528), (768, 768)]
CS_CASES = [(p, c, ld) for p in CS_PIXELS for c, ld in CS_LAYOUTS if c <= 96 or p <= 3 * 64 * 64]


def _channel_sums(x, ld, pixels, C, out, out2, accumulate):
    c = G.ctx()
    c._call('tha4_test_channel_sums', _ptr(x), ld, ctypes.c_int64(pixels), C, _ptr(out), _ptr(out2), accumulate, c._stream())
    torch.cuda.synchronize()


@pytest.mark.parametrize('pixels,C,ld', CS_CASES)
def test_channel_sums(pixels, C, ld):
    g = torch.Generator().manual_seed(pixels % 1000 + C)
    name = 'channel sums %d px C %d ld %d' % (pixels, C, ld)
    # one guard row past the last pixel and NaN columns past C: neither may be read
    xb = torch.full((pixels + 1, ld), NAN, device=DEV)
    ob, out = _slot(C)
    o2b, out2 = _slot(C, 3, 9)
    # dyadic: the output is the exact sum rounded once, bitwise, and out2 is the same value
    xb[:pixels, :C] = _dyadic((pixels, C), g, device=DEV)
    exact = xb[:pixels, :C].double().sum(0)
    _channel_sums(xb, ld, pixels, C, out, out2, 0)
    _bitwise(name + ' dyadic', out, exact.float())
    _bitwise(name + ' dyadic out2', out2, out)
    _outside_nan(name, ob, 5, 5 + C)
    _outside_nan(name + ' out2', o2b, 3, 3 + C)
    first = out.clone()
    pre = torch.randn(C, generator=g).to(DEV)
    out.copy_(pre)
    out2.copy_(pre)
    _channel_sums(xb, ld, pixels, C, out, out2, 1)
    _bitwise(name + ' accumulate', out, pre + first)
    _bitwise(name + ' accumulate out2', out2, out)
    _channel_sums(xb, ld, pixels, C, out, None, 0)
    assert torch.equal(out, first), name + ': two runs differ'
    assert torch.equal(out2, pre + first), name + ': out2 written without being given'
    # random: 1/2 ulp of the result for the final rounding, 2^-40 of the absolute sum for the fp64 partial sums
    xb[:pixels, :C] = torch.randn(pixels, C, generator=g).to(DEV) * 3
    x64 = xb[:pixels, :C].double()
    ref = x64.sum(0)
    _channel_sums(xb, ld, pixels, C, out, out2, 0)
    _ratio(name + ' random', out, ref, 0.5 * R.ulp32(ref.cpu()) + 2.0 ** -40 * x64.abs().sum(0).cpu())
    _bitwise(name + ' random out2', out2, out)


# ------------------------------------------------------------------------------------------ dense layer weight gradients
def _linear_wgrad(dyb, dy_off, dy_ld, N, R_, xb, x_ld, K, silu_x, dW, db, accumulate):
    c = G.ctx()
    c._call('tha4_test_linear_wgrad', _ptr(dyb[:, dy_off:] if dyb.dim() == 2 else dyb[dy_off:]), dy_ld, N, R_, _ptr(xb), x_ld, K,
            silu_x, _ptr(dW), _ptr(db), accumulate, c._stream())
    torch.cuda.synchronize()


def _linear_sites(mc, film_table, N):
    """Every linear_wgrad call of UNetNet::backward (unet_backward.cu) at its real (dy offset, dy_ld, N, R, x_ld, K,
    silu_x): the pose FiLM projections cond1_layers.1 of every ResBlock against SiLU(c2), cond_embed.2 against SiLU(c1),
    cond_embed.0 against the pose (K = 6 inside a wider pose row), the time FiLM projections cond0_layers.1 against SiLU(t2)
    (N = 1: d(film0) is summed over the batch), time_embed.3 against SiLU(t1), time_embed.1 against t0 (K = mc)."""
    off, cout, total = film_table
    sites = [('%s.cond1_layers.1' % b, o, total, N, 2 * cout[b], 256, 256, 1) for b, o in off.items()]
    sites += [('cond_embed.2', 0, 256, N, 256, 256, 256, 1), ('cond_embed.0', 0, 256, N, 256, 45, 6, 0)]
    sites += [('%s.cond0_layers.1' % b, o, total, 1, 2 * cout[b], 256, 256, 1) for b, o in off.items()]
    sites += [('time_embed.3', 0, 256, 1, 256, 256, 256, 1), ('time_embed.1', 0, 256, 1, 256, mc, mc, 0)]
    return sites


@pytest.mark.parametrize('net', ['body', 'upscaler'])
@pytest.mark.parametrize('N', [1, 5])
def test_linear_wgrad(net, N):
    mc = 64 if net == 'body' else 32
    table = _film1_layout(mc, [1, 2, 4, 4, 4] if net == 'body' else [1, 2, 4, 8, 8, 8])
    g = torch.Generator().manual_seed(N + mc)
    worst = 0.0
    for key, off, dy_ld, n, R_, x_ld, K, silu in _linear_sites(mc, table, N):
        name = '%s linear wgrad %s N %d' % (net, key, n)
        for dyadic in ((True, False) if not silu else (False,)):
            dyb = torch.full((n, dy_ld + 4), NAN, device=DEV)
            xb = torch.full((n, x_ld + 3), NAN, device=DEV)
            if dyadic:
                dy, x = _dyadic((n, R_), g), _dyadic((n, K), g)
            else:
                dy, x = torch.randn(n, R_, generator=g), torch.randn(n, K, generator=g) * 2
            dyb[:, off:off + R_] = dy.to(DEV)
            xb[:, :K] = x.to(DEV)
            wbuf, dW = _slot(R_ * K)
            bbuf, db = _slot(R_, 2, 6)
            _linear_wgrad(dyb, off, dyb.shape[1], n, R_, xb, xb.shape[1], K, silu, dW, db, 0)
            _outside_nan(name + ' dW', wbuf, 5, 5 + R_ * K)
            _outside_nan(name + ' db', bbuf, 2, 2 + R_)
            d64 = dy.double()
            u = F.silu(x.double()) if silu else x.double()
            ref_w, ref_b = (d64.t() @ u).reshape(-1), d64.sum(0)
            if dyadic:      # exact fp64 sums of exact products: the rounded exact values, bitwise
                _bitwise(name + ' dyadic dW', dW, ref_w.float())
                _bitwise(name + ' dyadic db', db, ref_b.float())
            else:           # SiLU in fp32 (expf, a division): 2^-21 of each |dy| |u| term covers it and the rounding
                mag = (d64.abs().t() @ u.abs()).reshape(-1)
                bw = (2.0 ** -21 if silu else 0.0) * mag + 0.5 * R.ulp32(ref_w) + 2.0 ** -45 * mag
                worst = max(worst, _ratio(name + ' dW', dW, ref_w, bw))
                _ratio(name + ' db', db, ref_b, 0.5 * R.ulp32(ref_b) + 2.0 ** -45 * d64.abs().sum(0))
            # db written exactly once per row: accumulate adds one gradient onto the prefill
            first_w, first_b = dW.clone(), db.clone()
            pre_w, pre_b = torch.randn(R_ * K, generator=g).to(DEV), torch.randn(R_, generator=g).to(DEV)
            dW.copy_(pre_w)
            db.copy_(pre_b)
            _linear_wgrad(dyb, off, dyb.shape[1], n, R_, xb, xb.shape[1], K, silu, dW, db, 1)
            _bitwise(name + ' accumulate dW', dW, pre_w + first_w)
            _bitwise(name + ' accumulate db', db, pre_b + first_b)
            _linear_wgrad(dyb, off, dyb.shape[1], n, R_, xb, xb.shape[1], K, silu, dW, db, 0)
            assert torch.equal(dW, first_w) and torch.equal(db, first_b), name + ': two runs differ'
    print('worst ratio %.3e' % worst)


# ------------------------------------------------------------------------------------------ encoder-decoder head biases
@pytest.mark.parametrize('S', [128, 192])
@pytest.mark.parametrize('B', [1, 3])
@pytest.mark.parametrize('n', [8, 10, 12])
def test_head_bias(S, B, n):
    g = torch.Generator().manual_seed(S + B + n)
    pixels = B * S * S
    dhb = torch.full((pixels, 16), NAN, device=DEV)          # channels n..15 are never read
    dhb[:, :n] = _dyadic((pixels, n), g, device=DEV)
    exact = dhb[:, :n].double().sum(0)
    total = 64
    slots = torch.randperm(total - 2, generator=g)[:n] + 1
    slots[n // 2] = -1                                       # a bias-free head channel
    offs = (ctypes.c_int64 * 16)(*slots.tolist())
    out = torch.full((total,), NAN, device=DEV)

    def run(accumulate):
        c = G.ctx()
        c._call('tha4_test_head_bias', _ptr(dhb), ctypes.c_int64(pixels), offs, n, _ptr(out), accumulate, c._stream())
        torch.cuda.synchronize()
    run(0)
    name = 'head bias B %d %d^2 n %d' % (B, S, n)
    mapped = [d for d in range(n) if slots[d] >= 0]
    idx = slots[mapped].to(DEV)
    _bitwise(name, out[idx], exact[mapped].float())
    keep = torch.ones(total, dtype=torch.bool, device=DEV)
    keep[idx] = False
    assert torch.isnan(out[keep]).all(), name + ': a slot outside the map (or the offset -1 channel) was written'
    first = out[idx].clone()
    pre = torch.randn(len(mapped), generator=g).to(DEV)
    out[idx] = pre
    run(1)
    _bitwise(name + ' accumulate', out[idx], pre + first)
    assert torch.isnan(out[keep]).all(), name + ': accumulate wrote outside the map'
    run(0)
    assert torch.equal(out[idx], first), name + ': two runs differ'


# ------------------------------------------------------------------------------------------ encoder-decoder d(pose)
@pytest.mark.parametrize('P,ld', [(12, 528), (27, 544), (12, 544)])
@pytest.mark.parametrize('b', [16, 24])
@pytest.mark.parametrize('B', [1, 3])
def test_pose_sum(P, ld, b, B):
    g = torch.Generator().manual_seed(P + ld + b + B)
    hw = b * b
    dbin = torch.full((B, hw, ld), NAN, device=DEV)
    dbin[..., :512] = torch.randn(B, hw, 512, generator=g).to(DEV)   # the feature channels' gradient, not part of the sum
    dbin[..., 512:512 + P] = _dyadic((B, hw, P), g, device=DEV)
    exact = dbin[..., 512:512 + P].double().sum(1)
    dld = P + 5
    out = torch.full((B, dld), NAN, device=DEV)

    def run():
        c = G.ctx()
        c._call('tha4_test_pose_sum', _ptr(dbin), ld, ctypes.c_int64(hw), 512, P, B, _ptr(out), dld, c._stream())
        torch.cuda.synchronize()
    run()
    name = 'pose sum P %d ld %d %d^2 B %d' % (P, ld, b, B)
    _bitwise(name, out[:, :P], exact.float())
    assert torch.isnan(out[:, P:]).all(), name + ': written past P'
    first = out.clone()
    run()
    assert torch.equal(out[:, :P], first[:, :P]), name + ': two runs differ'
