"""The weight-gradient convolution's U-Net operand variants (tha4_test_unet_wgrad, the launcher the body morpher's backward
uses) at the distinct weight-gradient layers of Morpher00 (-m gpu): 3x3 conv0 / conv1 at each width and resolution (the
up path's concatenated inputs included), the 4 -> 64 first conv, the pooled down-sampling conv0, nearest x2 + 3x3 at each
level, the 1x1 skip / qkv / proj convs at 16x16 and the 7-channel last.2 head, each in the operand variant the network runs.

- Dyadic inputs with no operand transform are bit-exact against fp64 (pins the 1x1, x2 and pooled geometry).
- Random inputs in the network's transform (f16 GroupNorm + FiLM0 + FiLM1 + fast SiLU on xf_build_coef's coefficients,
  raw f16, fp32, the tail's fp32 affine + tanh.approx.f32 SiLU rounded to f16, strict fp32) are within
  (2^-10 + K 2^-23) sum |dz| |x^| of fp64 on the transformed operand, widened to 2^-8 where a tanh.approx SiLU sits in
  the transform (the forward-kernel row of DESIGN.md section 4).
- The coefficients the transform used are within 2^-9 of fp64 GroupNorm + FiLM, and the f16 transform they give equals
  bitwise the one the forward conv applies to the same inputs; the plan is asserted; the NaN guard after dW stays NaN; two
  runs are bit-identical.  Statistics come in the replica counts the networks give a tensor of that size, FiLM1 at the
  block's real column offset in the 11008-wide table."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import gpu_util as G
from tha4_b200._lib import _ptr

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
NAN = float('nan')
XF_NONE, XF_HALF, XF_FLOAT, XF_FLOAT16 = 0, 1, 2, 3
ACT_NONE, ACT_SILU, ACT_SILU_FAST = 0, 2, 3
K3, K1, KUP2, KHEAD = 0, 1, 2, 3

FILM1_LD = 11008             # Morpher00's FiLM table: 2 x the output channels of its 26 ResBlocks
# (name, kind, Cx, Cout, H of x, operand: 'gn' (f16 GroupNorm, FiLM when film), 'raw16', 'f32', 'head' / 'head_strict', film1
# column offset of the block or None)
CASES = [
    ('first_conv 4->64 @256', K3, 4, 64, 256, 'f32', False),
    ('down0 conv0 64 @256', K3, 64, 64, 256, 'gn', False),
    ('down0 conv1 64 @256', K3, 64, 64, 256, 'gn', 0),
    ('down1 conv0 64->128 @128', K3, 64, 128, 128, 'gn', False),
    ('down-sampler conv0 pooled 64 @128', K3, 64, 64, 128, 'raw16', False),
    ('mid0 conv1 256 @16', K3, 256, 256, 16, 'gn', 3328),
    ('up4.1 conv1 64 @256', K3, 64, 64, 256, 'gn', 10880),
    ('up0 conv0 cat 512 @16', K3, 512, 256, 16, 'gn', False),
    ('up2 conv0 cat 384->256 @64', K3, 384, 256, 64, 'gn', False),
    ('up3 conv0 cat 192->128 @128', K3, 192, 128, 128, 'gn', False),
    ('up4 conv0 cat 128 @256', K3, 128, 64, 256, 'gn', False),
    ('up-sampler conv0 x2 256 @16', KUP2, 256, 256, 16, 'gn', False),
    ('up-sampler conv0 x2 256 @32', KUP2, 256, 256, 32, 'gn', False),
    ('up-sampler conv0 x2 256 @64', KUP2, 256, 256, 64, 'gn', False),
    ('up-sampler conv0 x2 128 @128', KUP2, 128, 128, 128, 'gn', False),
    ('skip 1x1 512->256 @16', K1, 512, 256, 16, 'raw16', False),
    ('qkv 1x1 256->768 @16', K1, 256, 768, 16, 'gn_none', False),
    ('proj 1x1 256 @16', K1, 256, 256, 16, 'f32', False),
    ('last.2 head 64->7 @256', KHEAD, 64, 7, 256, 'head', False),
    ('last.2 head strict 64->7 @256', KHEAD, 64, 7, 256, 'head_strict', False),
]
CASES = [c[:6] + (None if c[6] is False else c[6],) for c in CASES]


def _rep(H):
    """statistics replicas the networks give an H x H tensor (nets.cu make_view: about one per 32 conv tiles, at most 16)"""
    tiles = ((H + 15) // 16) * ((H + 7) // 8)
    r = 1
    while r < 16 and r * 32 <= tiles:
        r *= 2
    return r


def _stats(x, N, C, rep):
    """[rep][N][C][2] fp64 statistics of the tensor, its rows spread over the replicas as a producer's tiles spread them"""
    v = x.double()
    st = torch.zeros(rep, N, C, 2, dtype=torch.float64, device=DEV)
    H = v.shape[1]
    for r, rows in enumerate(torch.arange(H, device=DEV).chunk(rep)):
        st[r, :, :, 0] = v[:, rows].sum(dim=(1, 2))
        st[r, :, :, 1] = (v[:, rows] ** 2).sum(dim=(1, 2))
    return st


def _ref_coef(x16, gamma, beta, f0, f1, groups, halve):
    N, H, W, C = x16.shape
    v = x16.double().reshape(N, H * W, groups, C // groups)
    mean = v.mean(dim=(1, 3))
    var = (v * v).mean(dim=(1, 3)) - mean * mean
    rstd = (var + 1e-5).rsqrt()
    A = rstd.repeat_interleave(C // groups, dim=1) * gamma.double()
    B = beta.double() - mean.repeat_interleave(C // groups, dim=1) * A
    if f0 is not None:
        A = A * (1 + f0[:C].double()); B = B * (1 + f0[:C].double()) + f0[C:].double()
    if f1 is not None:
        A = A * (1 + f1[:, :C].double()); B = B * (1 + f1[:, :C].double()) + f1[:, C:].double()
    if halve:
        A, B = A / 2, B / 2
    return torch.stack([A, B], dim=-1)


def _run(kind, strict, x, x16, N, H, Cx, xf, act, stats, gamma, beta, f0, f1, f1_ld, f1_off, dz, Cout, dW_shape, ksplit=0):
    rep = stats.shape[0] if stats is not None else 1
    c = G.ctx()
    k = dW_shape[2]
    n = Cout * Cx * k * k
    buf = torch.full((n + 64,), NAN, device=DEV)
    coef = torch.full((N, Cx, 2), NAN, device=DEV)
    plan = torch.zeros(4, dtype=torch.int32)
    c._call('tha4_test_unet_wgrad', kind, strict, ksplit, _ptr(x), x16, Cx, N, H, H, Cx, xf, act, _ptr(stats), rep, 32,
            _ptr(gamma), _ptr(beta), _ptr(f0), _ptr(f1), f1_ld, f1_off, _ptr(dz), Cout, Cout, _ptr(buf), _ptr(coef),
            plan.numpy().ctypes.data, c._stream())
    torch.cuda.synchronize()
    assert torch.isnan(buf[n:]).all().item()
    return buf[:n].view(dW_shape), coef, plan.tolist()


def _ref_dw(xt, dz, kind, k):
    """fp64 weight gradient of the conv whose operand is xt (NHWC), dz NHWC"""
    xi = xt.permute(0, 3, 1, 2).double()
    if kind == KUP2:
        xi = F.interpolate(xi, scale_factor=2, mode='nearest')
    g = dz.permute(0, 3, 1, 2).double()
    return torch.nn.grad.conv2d_weight(xi, (g.shape[1], xi.shape[1], k, k), g, padding=(k - 1) // 2)


def _bound(xt, dz, kind, k, rel):
    K = dz.shape[0] * dz.shape[1] * dz.shape[2]
    return (rel + K * 2.0 ** -23) * _ref_dw(xt.abs(), dz.abs(), kind, k) + 1e-30


@pytest.mark.parametrize('N', [1, 3])
@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_unet_wgrad_layer(case, N):
    name, kind, Cx, Cout, H, op, f1_off = case
    film = f1_off is not None
    g = torch.Generator(device='cpu').manual_seed(sum(map(ord, name)) + N)
    k = 1 if kind == K1 else 3
    Ho = 2 * H if kind == KUP2 else H
    dW_shape = (Cout, Cx, k, k)
    # ---- dyadic, no transform: bit-exact against fp64 (default and strict) ----
    xd = (torch.randint(-4, 5, (N, H, H, Cx), generator=g).float() / 4).to(DEV)
    dzd = (torch.randint(-4, 5, (N, Ho, Ho, Cout), generator=g).float() / 8).to(DEV)
    for strict in (0, 1):
        dw, _, plan = _run(kind, strict, xd, 0, N, H, Cx, XF_NONE, ACT_NONE, None, None, None, None, None, 0, 0, dzd, Cout, dW_shape)
        assert torch.equal(dw.double(), _ref_dw(xd, dzd, kind, k)), (name, strict)
        assert plan[0] == (16 if Cout <= 16 else (64 if Cout <= 64 else 128)) and plan[1] == -(-(k * k * Cx) // 64), plan
    # ---- random, in the network's operand variant ----
    x = torch.randn(N, H, H, Cx, generator=g) * 1.5 + 0.3
    dz = (torch.randn(N, Ho, Ho, Cout, generator=g) * 1e-2).to(DEV)
    gamma = (torch.rand(Cx, generator=g) + 0.5).to(DEV)
    beta = (torch.randn(Cx, generator=g) * 0.3).to(DEV)
    f0 = (torch.randn(2 * Cx, generator=g) * 0.2).to(DEV) if film else None
    f1_ld, f1_off = FILM1_LD, f1_off or 0           # the block's row slice of the network's FiLM table
    f1 = (torch.randn(N, f1_ld, generator=g) * 0.2).to(DEV) if film else None
    if op in ('gn', 'gn_none', 'raw16', 'head', 'head_strict'):
        x16 = x.half().to(DEV)
        if op == 'raw16':
            args = (x16, 1, XF_NONE, ACT_NONE)
        elif op == 'head':
            args = (x16, 1, XF_FLOAT16, ACT_SILU_FAST)
        elif op == 'head_strict':                   # the strict tail: fp32 feature map, fp32 affine + SiLU
            args = (x.to(DEV), 0, XF_FLOAT, ACT_SILU)
        else:
            args = (x16, 1, XF_HALF, ACT_SILU_FAST if op == 'gn' else ACT_NONE)
    else:
        args = (x.to(DEV), 0, XF_NONE, ACT_NONE)
    xin, is16, xf, act = args
    stats = _stats(xin, N, Cx, _rep(H)) if xf != XF_NONE else None
    film1 = f1[:, f1_off:f1_off + 2 * Cx] if film else None
    strict_runs = (0, 1) if xf == XF_NONE else ((1,) if op == 'head_strict' else (0,))
    for strict in strict_runs:
        dw, coef, plan = _run(kind, strict, xin, is16, N, H, Cx, xf, act, stats, gamma, beta, f0, f1, f1_ld, f1_off, dz, Cout, dW_shape)
        again, _, _ = _run(kind, strict, xin, is16, N, H, Cx, xf, act, stats, gamma, beta, f0, f1, f1_ld, f1_off, dz, Cout, dW_shape)
        assert torch.equal(dw, again), 'two runs differ'
        xv = xin.double()
        rel = 2.0 ** -10
        if xf != XF_NONE:
            cref = _ref_coef(xin, gamma, beta, f0, film1, 32, xf == XF_HALF and act == ACT_SILU_FAST)
            cerr = ((coef.double() - cref).abs() / (cref.abs() + 2.0 ** -14)).max().item()
            assert cerr <= 2.0 ** -9, (name, cerr)
            A, B = coef.double()[..., 0], coef.double()[..., 1]
            if xf == XF_HALF:           # the f16 FMA is exact in fp64 before its rounding
                h = (xv * A[:, None, None, :] + B[:, None, None, :]).half().double()
                xv = (h + h * torch.tanh(h)) if act == ACT_SILU_FAST else h
            else:                       # the tail: fp32 affine, SiLU (f16 in the default mode)
                xv = F.silu(xv * A[:, None, None, :] + B[:, None, None, :])
                xv = xv.half().double() if xf == XF_FLOAT16 else xv
            if act == ACT_SILU_FAST:
                rel = 2.0 ** -8
            elif strict:                # strict: 3xTF32 products, fp32 affine and expf SiLU on the operand
                rel = 2.0 ** -20 + 2.0 ** -21
        ref = _ref_dw(xv, dz, kind, k)
        ratio = ((dw.double() - ref).abs() / _bound(xv, dz, kind, k, rel)).max().item()
        print('\n%s N=%d strict=%d: worst error / bound %.3f, plan %s' % (name, N, strict, ratio, plan))
        assert ratio <= 1.0, (name, strict, ratio)


def test_split_plan_matches_unsplit():
    """A forced pixel split sums its partials in split order: within rounding of the unsplit launch, and reproducible."""
    N, H, Cx, Cout = 1, 16, 256, 256
    g = torch.Generator().manual_seed(5)
    x = torch.randn(N, H, H, Cx, generator=g).to(DEV)
    dz = torch.randn(N, H, H, Cout, generator=g).to(DEV)
    one, _, p1 = _run(K1, 0, x, 0, N, H, Cx, XF_NONE, ACT_NONE, None, None, None, None, None, 0, 0, dz, Cout, (Cout, Cx, 1, 1), 1)
    two, _, p2 = _run(K1, 0, x, 0, N, H, Cx, XF_NONE, ACT_NONE, None, None, None, None, None, 0, 0, dz, Cout, (Cout, Cx, 1, 1), 4)
    assert p1[3] == 1 and p2[3] == 2, (p1, p2)           # 8 k-blocks: at least 4 per split
    assert ((one - two).abs().max() / one.abs().max()).item() <= 1e-5


@pytest.mark.parametrize('C,H,groups,film', [(64, 256, 32, False), (256, 16, 32, True), (128, 64, 32, True), (512, 16, 32, False)])
def test_coefficients_equal_the_forward_convs(C, H, groups, film):
    """The f16 transform of the weight-gradient operand equals bitwise the one the forward conv applies: a 1x1 forward conv
    with identity weights, no bias and no activation returns its transformed operand exactly (f16 products by 1, fp32 sums),
    and the coefficients the wgrad hook returns give the same f16 values (the FMA is exact in fp64 before its rounding)."""
    N = 2
    g = torch.Generator().manual_seed(C + H)
    x16 = (torch.randn(N, H, H, C, generator=g) * 1.5 + 0.3).half().to(DEV)
    stats = _stats(x16, N, C, _rep(H))
    gamma = (torch.rand(C, generator=g) + 0.5).to(DEV)
    beta = (torch.randn(C, generator=g) * 0.3).to(DEV)
    f0 = (torch.randn(2 * C, generator=g) * 0.2).to(DEV) if film else None
    f1 = (torch.randn(N, FILM1_LD, generator=g) * 0.2).to(DEV) if film else None
    off = 3328 if film else 0
    dz = torch.zeros(N, H, H, C, device=DEV)
    _, coef, _ = _run(K1, 0, x16, 1, N, H, Cx=C, xf=XF_HALF, act=ACT_NONE, stats=stats, gamma=gamma, beta=beta, f0=f0, f1=f1,
                      f1_ld=FILM1_LD, f1_off=off, dz=dz, Cout=C, dW_shape=(C, C, 1, 1))
    c = G.ctx()
    w = torch.eye(C, device=DEV).reshape(C, C, 1, 1).contiguous()
    out = torch.full((N, H, H, C), NAN, device=DEV)
    c._call('tha4_test_conv_forward_ex', 3, _ptr(w), None, C, C, None, None, 0, _ptr(x16), C, N, H, H, None, 0, _ptr(out), C,
            None, 0, None, 0, 0, ctypes.c_int64(0), None, 0, 0, _ptr(stats), C, stats.shape[0], ctypes.c_int64(N * C * 2), C, groups, 0,
            _ptr(gamma), _ptr(beta), _ptr(f0), _ptr(f1[:, off:] if film else None),
            FILM1_LD, 0, None, c._stream())
    torch.cuda.synchronize()
    A, B = coef.double()[..., 0], coef.double()[..., 1]
    exact = (x16.double() * A[:, None, None, :] + B[:, None, None, :]).cpu().numpy()
    # rounded once, fp64 -> f16 (numpy converts directly; a conversion through fp32 could round twice)
    mine = torch.from_numpy(exact.astype(np.float16).astype(np.float32)).to(DEV)
    assert torch.equal(out, mine), (out - mine).abs().max().item()
