"""Kernel-level parity of the encoder-decoders' weight-gradient convolution (-m gpu, conv_wgrad.cu through
tha4_test_conv_wgrad, the launcher the network backward uses) at every layer shape of the three networks (S = 128 / 192,
pose pads 0 / 16 / 32), in the operand variants the networks run: the fp32 image, f16 raw conv outputs with their producers'
statistics replicas (the default mode's fused InstanceNorm + ReLU), the f16 residual-stream copy, bin16 with 0 / 12 / 27 pose
columns, the heads' normalised f16 / fp32 feature map, and the fp32 tensors of strict mode.

- dyadic inputs (every partial sum exact): bit-exact against fp64, which pins the tap, stride, transpose and padding geometry;
- random inputs: within (2^-10 + K 2^-23) sum |dz| |x^| in the default mode (+ 2^-11 sum |dz| |x^|, the f16 affine term, for
  the normalised operands), (2^-20 + K 2^-23) sum |dz| |x^| in strict mode;
- the plan that ran is asserted; NaN guards around each destination slot stay NaN; two runs are bit-identical.
The transform's coefficients are checked against fp64 InstanceNorm moments, which pins the statistics replicas."""
import ctypes

import pytest
import torch

import gpu_util as G
import teacher_backward_ref as BR
import teacher_wgrad_ref as R
from tha4_b200._lib import _ptr

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
NAN = float('nan')
GUARD = 37

# (name, kind, Cx, Cout, H of x, variant, real channels of x, statistics replicas of the producer)
# kind 0 3x3, 1 4x4 s2, 2 transposed 4x4 s2 (x at H, dz at 2H), 3 head; variant: image / raw16 / res16 / bin16 / head
CASES = [
    ('dec down0', 0, 4, 64, 128, 'image', 4, 1), ('comb down0', 0, 8, 64, 128, 'image', 8, 1),
    ('S128 down1', 1, 64, 128, 128, 'raw16', 64, 4), ('S128 down2', 1, 128, 256, 64, 'raw16', 128, 1),
    ('S128 down3', 1, 256, 512, 32, 'raw16', 256, 1),
    ('dec bott0 P0', 0, 512, 512, 16, 'bin16', 512, 1), ('comb bott0 P12', 0, 528, 512, 16, 'bin16', 524, 1),
    ('S128 res conv0', 0, 512, 512, 16, 'res16', 512, 1), ('S128 res conv1', 0, 512, 512, 16, 'raw16', 512, 1),
    ('S128 up0', 2, 512, 256, 16, 'res16', 512, 1), ('S128 up1', 2, 256, 128, 32, 'raw16', 256, 1),
    ('S128 up2', 2, 128, 64, 64, 'raw16', 128, 1),
    ('dec head', 3, 64, 10, 128, 'head', 64, 4), ('comb head', 3, 64, 8, 128, 'head', 64, 4),
    ('face down0', 0, 4, 64, 192, 'image', 4, 1), ('face down1', 1, 64, 128, 192, 'raw16', 64, 8),
    ('face down2', 1, 128, 256, 96, 'raw16', 128, 2), ('face down3', 1, 256, 512, 48, 'raw16', 256, 1),
    ('face bott0 P27', 0, 544, 512, 24, 'bin16', 539, 1), ('face res conv0', 0, 512, 512, 24, 'res16', 512, 1),
    ('face res conv1', 0, 512, 512, 24, 'raw16', 512, 1), ('face up0', 2, 512, 256, 24, 'res16', 512, 1),
    ('face up1', 2, 256, 128, 48, 'raw16', 256, 1), ('face up2', 2, 128, 64, 96, 'raw16', 128, 2),
    ('face head', 3, 64, 12, 192, 'head', 64, 8),
]


def _dz_geom(kind, H):
    return H // 2 if kind == 1 else (2 * H if kind == 2 else H)


def _run(kind, strict, x, x_f16, xf, stats, rep, gamma, beta, norm_C, dz, dz_ld, Cout, c_real, ksplit=0):
    """-> (flat dW from a NaN-guarded slot, the transform's coefficients or None, plan)"""
    c = G.ctx()
    N, Cx, H, W = x.shape
    xd = x.permute(0, 2, 3, 1).contiguous().to(DEV, torch.float16 if x_f16 else torch.float32)
    Ho = _dz_geom(kind, H)
    dzb = torch.full((N, Ho, Ho, dz_ld), 1e4, device=DEV)           # columns past Cout must never be read
    dzb[..., :Cout] = dz.permute(0, 2, 3, 1).to(DEV)
    cr = c_real or Cx
    n = Cout * cr * (16 if kind in (1, 2) else 9)
    buf = torch.full((n + 2 * GUARD,), NAN, device=DEV)
    coef = torch.empty(N, norm_C, 2, device=DEV) if xf else None
    plan = (ctypes.c_int * 4)()
    gd, bd = (G.dev(gamma), G.dev(beta)) if xf else (None, None)
    c._call('tha4_test_conv_wgrad', kind, strict, ksplit, _ptr(xd), x_f16, Cx, N, H, W, Cx, xf, _ptr(stats), rep, _ptr(gd), _ptr(bd),
            norm_C, _ptr(dzb), dz_ld, Cout, c_real, _ptr(buf[GUARD:GUARD + n]), _ptr(coef), plan, c._stream())
    torch.cuda.synchronize()
    assert torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[GUARD + n:]).all(), 'written outside the slot'
    out = buf[GUARD:GUARD + n]
    assert torch.isfinite(out).all(), 'slot not fully written'
    return out.cpu(), (coef.cpu() if coef is not None else None), list(plan)


def _inputs(g, name, kind, Cx, Cout, H, variant, creal, N, strict):
    """(x stored, x_f16, xf, norm_C, gamma, beta, dz, dz_ld, c_real)"""
    x_f16 = 0 if strict or variant == 'image' else 1
    xf, norm_C, gamma, beta = R.XF_NONE, 0, None, None
    if variant == 'image':
        x = torch.rand(N, Cx, H, H, generator=g) * 2 - 1
    elif strict and variant != 'head':
        x = (torch.randn(N, Cx, H, H, generator=g)).clamp_min(0.0)          # the fp32 normalised tensor strict mode keeps
    else:
        x = torch.randn(N, Cx, H, H, generator=g) * 2 + 0.5
        if variant in ('raw16', 'bin16', 'head'):
            norm_C = 512 if variant == 'bin16' else Cx
            xf = R.XF_HALF if variant != 'head' else (R.XF_FLOAT if strict else R.XF_FLOAT16)
            gamma, beta = torch.rand(norm_C, generator=g) + 0.5, torch.randn(norm_C, generator=g) * 0.3
    if variant == 'bin16':
        x[:, creal:] = 0.0                                                     # pose padding planes
        x[:, 512:creal] = torch.rand(N, creal - 512, 1, 1, generator=g).expand(N, creal - 512, H, H) * 2 - 1   # tiled pose
    if x_f16:
        x = x.half().float()
    dz = torch.randn(N, Cout, _dz_geom(kind, H), _dz_geom(kind, H), generator=g)
    dz_ld = 16 if kind == 3 else Cout
    return x, x_f16, xf, norm_C, gamma, beta, dz, dz_ld, (creal if creal != Cx else 0)


@pytest.mark.parametrize('strict', [0, 1])
@pytest.mark.parametrize('N', [1, 3])
@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_wgrad_random(case, N, strict):
    name, kind, Cx, Cout, H, variant, creal, rep = case
    g = torch.Generator().manual_seed(sum(map(ord, name)) + N + 7 * strict)
    x, x_f16, xf, norm_C, gamma, beta, dz, dz_ld, c_real = _inputs(g, name, kind, Cx, Cout, H, variant, creal, N, strict)
    stats = BR.split_replicas(BR.stats_of(x[:, :norm_C]), rep, seed=3).contiguous().to(DEV) if xf else None
    ksplit = 3 if (N == 3 and kind == 0 and Cx >= 512) else 0            # the many-tile layers do not split by themselves
    out, coef, plan = _run(kind, strict, x, x_f16, xf, stats, rep, gamma, beta, norm_C, dz, dz_ld, Cout, c_real, ksplit)
    Ho = _dz_geom(kind, H)
    M, D, pix = (16 * Cout, Cx, N * H * H) if kind == 2 else ((16 if kind == 1 else 9) * Cx, Cout, N * Ho * Ho)
    assert plan == R.expected_plan(M, D, pix, ksplit), (plan, R.expected_plan(M, D, pix, ksplit))
    if xf:
        cr = R.coef_ref(x[:, :norm_C], gamma, beta)
        scale = (cr[..., 1].abs() + (cr[..., 1] - beta.double()[None]).abs())
        assert ((coef[..., 0].double() - cr[..., 0]).abs() <= 2.0 ** -9 * cr[..., 0].abs()).all(), 'coefficient A'
        assert ((coef[..., 1].double() - cr[..., 1]).abs() <= 2.0 ** -9 * scale + 1e-6).all(), 'coefficient B'
    xh = R.operand(x, xf, coef, norm_C)
    ref, absum = R.wgrad(0 if kind == 3 else kind, xh, dz)
    if c_real:
        ref, absum = ref[:, :c_real], absum[:, :c_real]
    K = pix
    rel = (2.0 ** -20 if strict else 2.0 ** -10 + (2.0 ** -11 if xf else 0.0)) + K * 2.0 ** -23
    bound = rel * absum + 1e-30
    got = out.double().view(ref.shape)
    ratio = ((got - ref).abs() / bound).max().item()
    print('\nwgrad %s N %d strict %d plan %s: max |err| / bound %.3e' % (name, N, strict, plan, ratio))
    assert ratio <= 1.0, ratio
    again, _, _ = _run(kind, strict, x, x_f16, xf, stats, rep, gamma, beta, norm_C, dz, dz_ld, Cout, c_real, ksplit)
    assert torch.equal(again, out), 'two runs differ'


# dyadic: values k 2^-3 (operand) and k 2^-4 (dz), |k| <= 2: every product and partial sum is exact in TF32 / fp32
DYADIC = [('3x3 image', 0, 4, 64, 64, 0, 0), ('3x3 f16 bin16 P12', 0, 528, 64, 16, 1, 524), ('4x4 s2 f16', 1, 64, 128, 64, 1, 0),
          ('transposed f16', 2, 256, 128, 32, 1, 0), ('head', 3, 64, 12, 64, 1, 0)]


@pytest.mark.parametrize('strict', [0, 1])
@pytest.mark.parametrize('ksplit', [0, 5])
@pytest.mark.parametrize('case', DYADIC, ids=[c[0] for c in DYADIC])
def test_wgrad_dyadic_bit_exact(case, ksplit, strict):
    name, kind, Cx, Cout, H, x_f16, c_real = case
    g = torch.Generator().manual_seed(len(name) + ksplit)
    N = 2
    x = torch.randint(-2, 3, (N, Cx, H, H), generator=g).double() / 8
    dz = torch.randint(-2, 3, (N, Cout, _dz_geom(kind, H), _dz_geom(kind, H)), generator=g).double() / 16
    out, _, plan = _run(kind, strict, x.float(), x_f16, R.XF_NONE, None, 1, None, None, 0, dz.float(), 16 if kind == 3 else Cout,
                        Cout, c_real, ksplit)
    if ksplit:
        assert plan[3] > 1, plan
    ref, _ = R.wgrad(0 if kind == 3 else kind, x, dz)
    if c_real:
        ref = ref[:, :c_real]
    assert torch.equal(out.double().view(ref.shape), ref), name
