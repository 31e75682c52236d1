"""The weight-gradient convolution's U-Net operand variants (tha4_test_unet_wgrad, the launcher the upscaler's backward uses) at
every distinct weight-gradient layer of Upscaler02 (-m gpu), at N = 1 and 2, in the operand variant the network runs.  The
list comes from the developer script's layer table, layers(512, 32, (1, 2, 4, 8, 8, 8)); its 4 -> 32 first conv is replaced
by what the upscaler runs instead: body.first_conv and coarse_image_conv as two convs on channel views (0-3 and 4-13) of the
16-channel fp32 prologue output, read with a row stride of 16.  The cases include 3x3 at 32 channels on 512x512 with
GroupNorm(32) at one channel per group, FiLM1 at each block's real offset in the 11392-wide table, the up path's concatenated
inputs at every resolution, nearest x2 + 3x3 into 512x512, the pooled 256x256 conv0, the 16x16 attention 1x1s and the
32 -> 7 last.2 head in the default and the strict tail's variant.

The assertions and bounds are those of test_gpu_unet_wgrad_kernels.py (the body morpher's), through its helpers: dyadic
inputs bit-exact against fp64, random inputs within the stated bound, coefficients within 2^-9, the plan that ran, the NaN
guard after dW, run-to-run identity.  The first-conv views also carry NaN in the padding channels 14 and 15, which no view
may read."""
import os
import sys

import pytest
import torch

import gpu_util as G
from tha4_b200._lib import _ptr
from test_gpu_unet_wgrad_kernels import (ACT_NONE, ACT_SILU, ACT_SILU_FAST, DEV, K1, K3, KHEAD, KUP2, NAN, XF_FLOAT, XF_FLOAT16,
                                         XF_HALF, XF_NONE, _bound, _ref_coef, _ref_dw, _rep, _run, _stats)

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'scripts', 'dev'))
from body_morpher_finetune_step import layers  # noqa: E402

pytestmark = pytest.mark.gpu
S, MC, MULTS = 512, 32, (1, 2, 4, 8, 8, 8)
FILM1_LD = 11392             # Upscaler02's FiLM table: 2 x the output channels of its 32 ResBlocks


def _film1_offsets():
    """block name -> column offset of its FiLM rows, in the order UNetNet::load stacks them (the layer table's block order)"""
    offs, total = {}, 0
    for name, kind, Cx, Cout, H, x16, xf, act in layers(S, MC, MULTS):
        block, _, conv = name.rpartition('.')
        if conv == 'conv1':
            offs[block] = total
            total += 2 * Cout
    assert total == FILM1_LD, total
    return offs


def _cases():
    """(name, kind, Cx, Cout, H of x, operand, film1 offset or None): one per distinct layer (a conv1, whose operand has the
    block's FiLM, is distinct from a conv0 of the same shape), named after its first use"""
    offs = _film1_offsets()
    seen, out = set(), []
    for name, kind, Cx, Cout, H, x16, xf, act in layers(S, MC, MULTS):
        block, _, conv = name.rpartition('.')
        key = (kind, Cx, Cout, H, x16, xf, act, conv == 'conv1')
        if name == 'first_conv' or key in seen:
            continue
        seen.add(key)
        if kind == KHEAD:
            out += [(name, kind, Cx, Cout, H, 'head', None), (name + ' strict', kind, Cx, Cout, H, 'head_strict', None)]
            continue
        if xf == XF_HALF:
            op = 'gn' if act == ACT_SILU_FAST else 'gn_none'
        else:
            op = 'raw16' if x16 else 'f32'
        out.append(('%s %d->%d @%d' % (name, Cx, Cout, H), kind, Cx, Cout, H, op, offs[block] if conv == 'conv1' else None))
    return out


CASES = _cases()


def test_cases_cover_the_network():
    kinds = {c[1] for c in CASES}
    assert kinds == {K3, K1, KUP2, KHEAD}
    assert len(CASES) == 55                  # 54 distinct layers besides the first conv, and the head's strict variant
    assert any(c[2] == 32 and c[4] == 512 and c[5] == 'gn' and c[6] is not None for c in CASES)     # conv1 at 512, FiLM
    assert any(c[1] == KUP2 and 2 * c[4] == 512 for c in CASES)
    assert any(c[5] == 'raw16' and c[1] == K3 and c[4] == 256 for c in CASES)                      # pooled conv0 at 256
    assert {c[2] for c in CASES if c[1] == K3 and c[5] == 'gn' and c[6] is None and c[2] > c[3]} >= {96, 192, 384, 512}


@pytest.mark.parametrize('N', [1, 2])
@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_upscaler_wgrad_layer(case, N):
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
    f1 = (torch.randn(N, FILM1_LD, generator=g) * 0.2).to(DEV) if film else None
    f1_off = f1_off or 0
    if op == 'raw16':
        args = (x.half().to(DEV), 1, XF_NONE, ACT_NONE)
    elif op == 'head':
        args = (x.half().to(DEV), 1, XF_FLOAT16, ACT_SILU_FAST)
    elif op == 'head_strict':                       # the strict tail: fp32 feature map, fp32 affine + SiLU
        args = (x.to(DEV), 0, XF_FLOAT, ACT_SILU)
    elif op in ('gn', 'gn_none'):
        args = (x.half().to(DEV), 1, XF_HALF, ACT_SILU_FAST if op == 'gn' else ACT_NONE)
    else:
        args = (x.to(DEV), 0, XF_NONE, ACT_NONE)
    xin, is16, xf, act = args
    stats = _stats(xin, N, Cx, _rep(H)) if xf != XF_NONE else None
    film1 = f1[:, f1_off:f1_off + 2 * Cx] if film else None
    strict_runs = (0, 1) if xf == XF_NONE else ((1,) if op == 'head_strict' else (0,))
    for strict in strict_runs:
        dw, coef, plan = _run(kind, strict, xin, is16, N, H, Cx, xf, act, stats, gamma, beta, f0, f1, FILM1_LD, f1_off, dz, Cout, dW_shape)
        again, _, _ = _run(kind, strict, xin, is16, N, H, Cx, xf, act, stats, gamma, beta, f0, f1, FILM1_LD, f1_off, dz, Cout, dW_shape)
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
                xv = torch.nn.functional.silu(xv * A[:, None, None, :] + B[:, None, None, :])
                xv = xv.half().double() if xf == XF_FLOAT16 else xv
            if act == ACT_SILU_FAST:
                rel = 2.0 ** -8
            elif strict:                # strict: 3xTF32 products, fp32 affine and expf SiLU on the operand
                rel = 2.0 ** -20 + 2.0 ** -21
        ref = _ref_dw(xv, dz, kind, k)
        ratio = ((dw.double() - ref).abs() / _bound(xv, dz, kind, k, rel)).max().item()
        print('\n%s N=%d strict=%d: worst error / bound %.3f, plan %s' % (name, N, strict, ratio, plan))
        assert ratio <= 1.0, (name, strict, ratio)


def _run_view(strict, x0, c0, C, dz):
    """the weight gradient of a conv on channels [c0, c0 + C) of the 16-channel x0, as the upscaler's backward launches it"""
    N, H = x0.shape[0], x0.shape[1]
    Cout = dz.shape[3]
    n = Cout * C * 9
    buf = torch.full((n + 64,), NAN, device=DEV)
    plan = torch.zeros(4, dtype=torch.int32)
    c = G.ctx()
    c._call('tha4_test_unet_wgrad', K3, strict, 0, _ptr(x0[..., c0:]), 0, 16, N, H, H, C, XF_NONE, ACT_NONE, None, 1, 32,
            None, None, None, None, 0, 0, _ptr(dz), Cout, Cout, _ptr(buf), None, plan.numpy().ctypes.data, c._stream())
    torch.cuda.synchronize()
    assert torch.isnan(buf[n:]).all().item()
    return buf[:n].view(Cout, C, 3, 3), plan.tolist()


@pytest.mark.parametrize('N', [1, 2])
@pytest.mark.parametrize('c0,C,name', [(0, 4, 'body.first_conv'), (4, 10, 'coarse_image_conv')])
def test_first_conv_views(c0, C, name, N):
    """body.first_conv (rest image, channels 0-3) and coarse_image_conv (posed, warped, grid: 4-13) of the fused first conv,
    32 output channels at 512x512, each read from the 16-channel prologue output whose padding channels hold NaN."""
    g = torch.Generator().manual_seed(c0 + 10 * N)
    x0 = torch.full((N, S, S, 16), NAN)
    x0[..., :14] = torch.randint(-4, 5, (N, S, S, 14), generator=g).float() / 4
    x0 = x0.to(DEV)
    dz = (torch.randint(-4, 5, (N, S, S, MC), generator=g).float() / 8).to(DEV)
    xs = x0[..., c0:c0 + C]
    for strict in (0, 1):
        dw, plan = _run_view(strict, x0, c0, C, dz)
        assert torch.equal(dw.double(), _ref_dw(xs, dz, K3, 3)), (name, strict)
        assert plan[:2] == [64, -(-(9 * C) // 64)], plan
    x0[..., :14] = (torch.randn(N, S, S, 14, generator=g) * 0.5).to(DEV)
    dz = (torch.randn(N, S, S, MC, generator=g) * 1e-2).to(DEV)
    xs = x0[..., c0:c0 + C]
    for strict, rel in ((0, 2.0 ** -10), (1, 2.0 ** -20 + 2.0 ** -21)):
        dw, plan = _run_view(strict, x0, c0, C, dz)
        again, _ = _run_view(strict, x0, c0, C, dz)
        assert torch.equal(dw, again), 'two runs differ'
        ratio = ((dw.double() - _ref_dw(xs, dz, K3, 3)).abs() / _bound(xs.double(), dz, K3, 3, rel)).max().item()
        print('\n%s N=%d strict=%d: worst error / bound %.3f, plan %s' % (name, N, strict, ratio, plan))
        assert ratio <= 1.0, (name, strict, ratio)
