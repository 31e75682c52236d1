"""CPU checks of the fp64 references the student training kernel tests rely on (tests/distill_kernel_ref.py)."""
import struct

import pytest
import torch

import distill_kernel_ref as D


def _f(bits):
    return struct.unpack('<f', struct.pack('<I', bits))[0]


def _bits(x):
    return struct.unpack('<I', struct.pack('<f', x))[0]


@pytest.mark.parametrize('inp, out', [
    (0x3F800000, 0x3F800000),          # 1.0 stays
    (0x3F800FFF, 0x3F800000),          # below half a TF32 ulp: down
    (0x3F801000, 0x3F802000),          # exact tie: away from zero
    (0xBF801000, 0xBF802000),          # negative tie: away from zero
    (0x3F803000, 0x3F804000),          # tie with an odd kept mantissa: still away (not to even)
    (0x3F805000, 0x3F806000),          # tie with an even kept mantissa: away, not to even
    (0x3F801001, 0x3F802000),          # above the tie
    (0x3FFFF000, 0x40000000),          # just below 2: carries into the exponent
    (0x3F7FF000, 0x3F800000),          # just below 1 (tie): rounds up to the power of two
    (0x3F7FEFFF, 0x3F7FE000),          # just below that: stays below 1
    (0x00000000, 0x00000000), (0x80000000, 0x80000000),
    (0x00001000, 0x00002000),          # subnormal tie
    (0x7F800000, 0x7F800000), (0xFF800000, 0xFF800000),
])
def test_round_tf32_bit_patterns(inp, out):
    r = D.round_tf32(torch.tensor([_f(inp)]))
    assert _bits(r.item()) == out, hex(_bits(r.item()))


def test_round_tf32_is_nearest_with_ties_away():
    x = torch.randn(100000, generator=torch.Generator().manual_seed(0)) * 1e3
    r = D.round_tf32(x).double()
    xd = x.double()
    ulp = torch.exp2(torch.floor(torch.log2(xd.abs())) - 10)
    err = (r - xd).abs()
    assert torch.all(err <= ulp / 2)
    ties = err == ulp / 2
    assert torch.all(r[ties].abs() > xd[ties].abs())
    assert torch.equal(D.round_tf32(r.float()), r.float())                    # idempotent: 10 explicit bits
    assert torch.all((r.float().view(torch.int32) & 0x1FFF) == 0)


def test_dyadic_values_and_exactness_claim():
    a = D.dyadic((64, 360), bits=4, exp=4, seed=1)
    b = D.dyadic((360, 64), bits=6, exp=6, seed=2)
    assert torch.equal(D.round_tf32(a), a) and torch.equal(D.round_tf32(b), b)
    amax, au = D.dyadic_unit(4, 4)
    bmax, bu = D.dyadic_unit(6, 6)
    assert a.abs().max().item() <= amax and torch.all(a.double() / au == torch.round(a.double() / au))
    D.assert_exact_sums(360, amax * bmax, au * bu)
    # the claim: fp32 in any order equals fp64
    exact = a.double() @ b.double()
    assert torch.equal((a @ b).double(), exact)
    assert torch.equal((a.flip(1) @ b.flip(0)).double(), exact)
    acc = torch.zeros(64, 64)
    for k in torch.randperm(360, generator=torch.Generator().manual_seed(3)).tolist():
        acc += a[:, k:k + 1] * b[k:k + 1, :]
    assert torch.equal(acc.double(), exact)
    # and the guard refuses what it cannot promise
    with pytest.raises(AssertionError):
        D.assert_exact_sums(2 ** 21, 16.0, 1.0)
    with pytest.raises(AssertionError):
        D.assert_exact_sums(4, 1.5, 1.0)


def test_bilinear_pair_is_adjoint(oracle_clib):
    g = torch.Generator().manual_seed(4)
    p = torch.randn(2, 3, 16, 16, generator=g)
    d = torch.randn(2, 3, 32, 32, generator=g, dtype=torch.float64)
    up = D.upsample2(oracle_clib, p).double()
    ref = torch.nn.functional.interpolate(p.double(), scale_factor=2, mode='bilinear', align_corners=False)
    assert (up - ref).abs().max().item() <= 4 * D.U32 * ref.abs().max().item()
    # <U p, d> = <p, U^T d> with the fp64 forward (the fp32 one above differs from it by its own rounding only)
    rhs = (p.double() * D.upsample2_adjoint(d)).sum().item()
    lhs64 = (ref * d).sum().item()
    assert abs(lhs64 - rhs) <= 1e-12 * (ref.abs() * d.abs()).sum().item(), (lhs64, rhs)


def test_adjoint_folds_both_taps_at_the_border():
    # source column 0 is read by output columns 0 (weight 1: both taps clamp onto it), 1 (0.75) and 2 (0.25)
    d = torch.zeros(1, 1, 4, 8, dtype=torch.float64)
    d[0, 0, 0, 0] = 1.0                        # the corner: both taps on both axes land on source (0, 0)
    a = D.upsample2_adjoint(d)
    assert a[0, 0, 0, 0].item() == 1.0 and a.abs().sum().item() == 1.0


def test_body_loss_reference_gradient_signs(oracle_clib):
    """sgn(0) = 0 at exact ties, the grid weight on clamped samples only from the |grid - T3| term."""
    R, N = 8, 1
    g = torch.Generator().manual_seed(5)
    out7 = torch.zeros(N, R, R, 8)
    out7[..., 2] = 0.5
    out7[..., 3:7] = torch.rand(N, R, R, 4, generator=g)
    out7[0, :, :4, 0] = 2.0                    # clamped columns
    image = torch.rand(N, 4, R, R, generator=g)
    T0 = out7[..., 3:7].permute(0, 3, 1, 2).contiguous()       # colour ties everywhere
    T2 = torch.rand(N, 4, R, R, generator=g) + 2.0
    T3 = out7[..., 0:2].permute(0, 3, 1, 2).contiguous()       # grid ties everywhere
    w = [1.0, 2.0, 3.0, 4.0]
    sums, d = D.body_loss_ref(oracle_clib, out7, image, T0, T2, T3, w)
    assert sums[2].item() == 0 and sums[3].item() == 0
    assert torch.all(d[0, :, :4, 0] == 0)      # clamped: no sampling term; tie: no grid term
    assert torch.all(d[..., 7] == 0)
