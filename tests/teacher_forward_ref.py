"""Plain fp64 references of the default-mode teacher forward kernels (conv_halo.cu / conv_tc.cu with the fused input
normalisation), CPU only.

Each reference runs on exactly the operands the kernel sees: the f16 raw input, normalised with the fp64 sum of the
statistics replicas it is handed; the weights after the pack's TF32 rounding, power-of-two scaling and f16 rounding.  Next
to each result it returns an elementwise worst-case bound on the kernel's error, computed from the same operands:
  * the normalisation affine (A, B) is formed in fp32 from the fp64 sums and rounded to f16; the kernel evaluates
    x A + B with one f16 FMA (conv_tc_device.cuh: xf_build_coef / xf_chunks);
  * SiLU runs in f16 as h + h tanh.approx(h) with h = (x A + B) / 2;
  * the products of f16 operands are exact, the fp32 accumulation over K terms in any order (split-K and cluster
    partials included) is bounded by 2 K 2^-23 of sum |a| |w|, as in test_gpu_halo_split.py;
  * bias and residual are added in fp32.
A cancelling sum is bounded by the sum of its absolute terms rather than by its result.
"""
import math

import torch
import torch.nn.functional as F

from distill_kernel_ref import round_tf32
from teacher_backward_ref import attention_ref, split_replicas, stats_of  # noqa: F401  (the GPU tests take them from here)

U32 = 2.0 ** -24           # unit roundoff of fp32
U16 = 2.0 ** -11           # unit roundoff of f16
F16_FLOOR = 2.0 ** -25     # half the spacing of f16 subnormals: the absolute rounding error of a value near 0
# Assumption: tanh.approx.f16 has an absolute error of at most 2^-10.987 (the PTX ISA's stated maximum for the f16 type),
# rounded up here to 2^-10.  It cannot be checked without the GPU; the GPU tests would fail if it were exceeded.
TANH16_ABS = 2.0 ** -10
# |d/dh h (1 + tanh h)| <= 1 + 1 + max_h h sech^2 h (0.4477): the Lipschitz constant of SiLU in its half argument
SILU_HALF_LIP = 2.45
EPS = 1e-5


# ------------------------------------------------------------------------------------------ weights
def up2_phase_weights(w):
    """CONV_UP2_3x3 (nearest x2 upsample, then 3x3) as four phases of 2x2 taps on the low-resolution input, summed in fp32
    in conv_pack_kernel's order (ky outer, kx inner, from 0): [4][Cout, Cin, 2, 2] fp32, phase = 2 py + px."""
    w = w.float()
    out = torch.zeros(4, w.shape[0], w.shape[1], 2, 2, dtype=torch.float32)
    rng = {0: [(0, 0), (1, 2)], 1: [(0, 1), (2, 2)]}       # parity -> tap -> (k0, k1) of the 3x3 kernel read at that tap
    for ph in range(4):
        py, px = ph >> 1, ph & 1
        for ty in range(2):
            for tx in range(2):
                ky0, ky1 = rng[py][ty]
                kx0, kx1 = rng[px][tx]
                v = torch.zeros(w.shape[0], w.shape[1], dtype=torch.float32)
                for ky in range(ky0, ky1 + 1):
                    for kx in range(kx0, kx1 + 1):
                        v = v + w[:, :, ky, kx]
                out[ph, :, :, ty, tx] = v
    return out


def packed_f16(wp):
    """fp64 value of the f16 copy the kernel multiplies (conv_make_half), unscaled: TF32-rounded weights times the power of
    two that puts max |w| in [0.5, 1), rounded to f16 (round to nearest even), divided by the same power."""
    wt = round_tf32(wp)
    mx = wt.abs().max().item()
    scale = 1.0
    if mx > 0:
        e = math.frexp(mx)[1]
        scale = 2.0 ** -max(-24, min(8, e))
    return (wt * scale).half().double() / scale


def kernel_weights(kind, w):
    """kind 0 (3x3) / 1 (4x4 stride 2) / 3 (1x1): [Cout, Cin, k, k]; kind 4 (CONV_UP2_3x3): [4][Cout, Cin, 2, 2] -- as the kernel holds them."""
    if kind == 4:
        return packed_f16(up2_phase_weights(w))
    return packed_f16(w.float())


# ------------------------------------------------------------------------------------------ fused input normalisation
def _group_sums(sums, groups):
    """[N, C, 2] -> per-channel (mean numerator, square numerator) of its group (InstanceNorm: groups == 0)."""
    N, C, _ = sums.shape
    if groups == 0:
        return sums, 1
    cpg = C // groups
    g = sums.view(N, groups, cpg, 2).sum(2)
    return g.repeat_interleave(cpg, 1), cpg


def normalized_operand(x16, sums, norm_C, groups, gamma, beta, act, film0=None, film1=None, hw=None):
    """The operand the conv multiplies: act(FiLM1(FiLM0(GroupNorm(x)))) of the first norm_C channels of the f16 input x16
    [N, Cin, H, W] (fp64 values of f16 numbers), the rest passed through.  sums [N, norm_C, 2]: the fp64 total of the
    statistics replicas.  film1: [N, 2 norm_C] rows.  act 0 none, 1 ReLU, 2 SiLU.  hw: pixels per channel the sums cover
    (default: all of x16's; a band of rows may be passed).  Returns (operand, elementwise bound)."""
    x = x16.double()
    N, Cin, H, W = x.shape
    C = norm_C
    gs, cpg = _group_sums(sums.double(), groups)
    cnt = float((hw if hw is not None else H * W) * cpg)
    mean = gs[..., 0] / cnt
    var = (gs[..., 1] / cnt - mean * mean).clamp_min(0.0)
    rstd = 1.0 / torch.sqrt(var + EPS)
    A = rstd * gamma.double().view(1, C)
    B = beta.double().view(1, C) - mean * A
    Bmag = beta.double().abs().view(1, C) + (mean * A).abs()
    for film in (film0, film1):
        if film is None:
            continue
        f = film.double().view(-1, 2 * C)
        sc, sh = 1 + f[:, :C], f[:, C:]
        A, B, Bmag = A * sc, B * sc + sh, Bmag * sc.abs() + sh.abs()
    xa = x[:, :C]
    A4, B4, Bm4 = (t.view(-1, C, 1, 1) for t in (A, B, Bmag))
    z = xa * A4 + B4
    terms = xa.abs() * A4.abs() + Bm4
    # A and B: fp32 arithmetic (a few u) and one f16 rounding each; the f16 FMA rounds once more
    e_coef = (U16 + 16 * U32) * terms + F16_FLOOR * (xa.abs() + 1.0)
    if act == 2:
        h = 0.5 * z
        e_h = 0.5 * e_coef + U16 * (h.abs() + 0.5 * e_coef) + F16_FLOOR
        a = h * (1 + torch.tanh(h))
        e_pre = SILU_HALF_LIP * e_h + (h.abs() + e_h) * TANH16_ABS
        e = e_pre + U16 * (a.abs() + e_pre) + F16_FLOOR
    else:
        e = e_coef + U16 * (z.abs() + e_coef) + F16_FLOOR
        a = F.relu(z) if act == 1 else z
    if Cin > C:
        a = torch.cat([a, x[:, C:]], 1)
        e = torch.cat([e, torch.zeros_like(x[:, C:])], 1)
    return a, e


# ------------------------------------------------------------------------------------------ conv
def _conv(kind, a, wk, pad=None):
    if kind == 4:          # four phases of 2x2 taps on the low-resolution input
        N, _, H, W = a.shape
        out = torch.zeros(N, wk.shape[1], 2 * H, 2 * W, dtype=torch.float64)
        for ph in range(4):
            py, px = ph >> 1, ph & 1
            ap = F.pad(a, (1 - px, px, 1 - py, py))        # (left, right, top, bottom): taps at offsets -1/0 or 0/+1
            out[:, :, py::2, px::2] = F.conv2d(ap, wk[ph])
        return out
    if kind == 1:          # 4x4 stride 2 pad 1
        return F.conv2d(a, wk, None, 2, 1)
    return F.conv2d(a, wk, None, 1, wk.shape[-1] // 2 if pad is None else pad)


def conv_ref(kind, a, e_a, wk, bias=None, res=None, res_mode=0, a2=None, wk2=None, pad=None):
    """conv_forward on the operand a (bound e_a) with the kernel's weights wk (kernel_weights), plus a folded 1x1 conv of the
    raw f16 input a2 with wk2, bias and a residual (res_mode 1 same resolution, 2 nearest x2 of a half-resolution res).
    pad 0: a and e_a already carry the zero padding (a window of a larger map).  Returns (fp64 reference, elementwise bound)."""
    out = _conv(kind, a, wk, pad)
    mag = _conv(kind, a.abs(), wk.abs(), pad)
    err = _conv(kind, e_a, wk.abs(), pad)
    taps = 4 if kind == 4 else wk.shape[-1] * wk.shape[-2]
    K = taps * wk.shape[-3]
    if a2 is not None:
        out = out + F.conv2d(a2.double(), wk2)
        mag = mag + F.conv2d(a2.double().abs(), wk2.abs())
        K += wk2.shape[1]
    bound = err + 2 * K * 2.0 ** -23 * mag
    extra = torch.zeros_like(out)
    if bias is not None:
        out = out + bias.double().view(1, -1, 1, 1)
        extra = extra + bias.double().abs().view(1, -1, 1, 1)
    if res is not None:
        r = res.double() if res_mode == 1 else F.interpolate(res.double(), scale_factor=2, mode='nearest')
        out = out + r
        extra = extra + r.abs()
    bound = bound + 4 * U32 * (mag + extra) + 1e-30
    return out, bound


# ------------------------------------------------------------------------------------------ outputs the epilogue derives
def f16_copy_bound(y32):
    """|y16 - y32| for the f16 copy of an fp32 output: one f16 rounding."""
    return U16 * y32.double().abs() + F16_FLOOR


def stats_bound(y):
    """Bound on the epilogue's statistics of the output y [N, C, H, W] (fp32 sums of 32 rows per lane, the lanes' partials
    added in fp64): [N, C, 2] of 64 u times the sums of |y| and of y^2."""
    y = y.double()
    return 64 * U32 * torch.stack([y.abs().sum((2, 3)), (y * y).sum((2, 3))], -1)


def stats_ref_from_f16(y16):
    """The statistics of an output stored in f16 only, from its f16 copy: (fp64 sums [N, C, 2], bound).  The kernel summed the
    fp32 values, each within one f16 rounding of the copy."""
    y = y16.double()
    s = stats_of(y)
    a = y.abs()
    d = U16 * a / (1 - U16) + F16_FLOOR
    b = torch.stack([d.sum((2, 3)), (2 * a * d + d * d).sum((2, 3))], -1)
    return s, b + stats_bound(y) * 1.01


# ------------------------------------------------------------------------------------------ fused tail
def _sig(h, e):
    """sigmoid (Lipschitz 1/4), evaluated in fp32 with expf and one division."""
    return torch.sigmoid(h), 0.25 * e + 8 * U32


def _tanh(h, e):
    """tanhf (Lipschitz 1), a few ulp."""
    return torch.tanh(h), e + 8 * U32


def _color(alpha, color, image):
    """apply_color_change: color alpha + image (1 - alpha), each operand a (value, bound) pair."""
    (a, ea), (c, ec), (i, ei) = alpha, color, image
    v = c * a + i * (1 - a)
    return v, (c - i).abs() * ea + a.abs() * ec + (1 - a).abs() * ei + 4 * U32 * ((c * a).abs() + (i * (1 - a)).abs())


def _rgb(alpha, color, image):
    """apply_rgb_change: RGB blended as _color, the image's own alpha kept."""
    v, e = _color(alpha, (color[0][:, 0:3], color[1][:, 0:3]), (image[0][:, 0:3], image[1][:, 0:3]))
    return torch.cat([v, image[0][:, 3:4]], 1), torch.cat([e, image[1][:, 3:4]], 1)


def _warp(gc, image):
    """apply_grid_change (bilinear, border, align_corners False) of an exact image by the offsets gc (value, bound).  The
    sample moves by S / 2 pixels per unit of offset, and bilinear interpolation of a border-clamped image changes by at most
    L = the largest difference of two adjacent pixels per pixel moved; the fp32 source coordinate is off by a few u S
    pixels; the blend of four corners rounds a few times."""
    from oracle import tha4_oracle as O
    g, eg = gc
    img = image.double()
    N, _, H, W = img.shape
    v = O.apply_grid_change(g, img)
    L = torch.maximum((img[..., 1:, :] - img[..., :-1, :]).abs().amax((1, 2, 3)),
                      (img[..., :, 1:] - img[..., :, :-1]).abs().amax((1, 2, 3))).view(N, 1, 1, 1)
    pos = 0.5 * W * (eg[:, 0:1] + eg[:, 1:2]) + 16 * U32 * W
    e = L * pos + 8 * U32 * img.abs().amax((1, 2, 3)).view(N, 1, 1, 1)
    return v, e.expand_as(v)


def tail_ref(kind, x16, sums, groups, act, gamma, beta, ws, bs, image0, image1=None):
    """The fused tail (tail_tc.cu) of one site: the pending normalisation of the raw f16 feature map x16 (from the fp64 sum of
    the replicas; the kernel forms fp32 coefficients and one fp32 FMA, rounded to f16 -- inside normalized_operand's bound),
    the 3x3 head conv (weights TF32- and f16-rounded: 2^-10 of |a| |w| for the weights, 2 K 2^-23 for the fp32
    accumulation), then the reference's ops of the site (as test_gpu_kernels._tail_reference) in fp64 with the head bound
    carried through sigmoid / tanh / the blends / the warp.  ws, bs: the head convs in tail.cu order.  Returns the outputs
    in the kernel's order as (value, bound) pairs."""
    C = x16.shape[1]
    a, e = normalized_operand(x16, sums, C, groups, gamma, beta, act)
    w = torch.cat([t.double() for t in ws], 0)
    b = torch.cat([(t.double() if t is not None else torch.zeros(u.shape[0], dtype=torch.float64)) for t, u in zip(bs, ws)])
    h = F.conv2d(a, w, b, 1, 1)
    mag = F.conv2d(a.abs(), w.abs(), None, 1, 1)
    K = 9 * C
    eh = F.conv2d(e, w.abs(), None, 1, 1) + (2.0 ** -10 + 2 * K * 2.0 ** -23) * mag + 4 * U32 * b.abs().view(1, -1, 1, 1)
    eh = eh + 2.0 ** -24 * w.abs().max() * F.conv2d(a.abs(), torch.ones_like(w[:1]), None, 1, 1)    # f16 weights near 0
    H = lambda i, j: (h[:, i:j], eh[:, i:j])                                                    # noqa: E731
    im0 = (image0.double(), torch.zeros_like(image0.double()))
    if kind == 0:
        alpha, warped = _sig(*H(6, 7)), _warp(H(4, 6), image0)
        return [_color(alpha, H(0, 4), warped), alpha, warped, H(4, 6), H(0, 4)]
    if kind == 1:
        bga, bgc, eba, ebc = _sig(*H(0, 1)), _tanh(*H(1, 5)), _sig(*H(5, 6)), _tanh(*H(6, 10))
        return [_color(eba, im0, ebc), eba, ebc, _color(bga, bgc, im0), bga, bgc]
    if kind == 2:
        im1 = (image1.double(), torch.zeros_like(image1.double()))
        alpha, color, ca = _sig(*H(2, 3)), _tanh(*H(3, 7)), _sig(*H(7, 8))
        warped = _warp(H(0, 2), image0)
        morphed = _color(alpha, color, warped)
        half = ((morphed[0][:, 3:4] + 1) / 2, morphed[1][:, 3:4] / 2 + 2 * U32)
        return [_rgb(ca, morphed, im1), ca, _rgb(half, morphed, im1), morphed, alpha, color, warped, H(0, 2)]
    imc, ima, eyc, eya = _tanh(*H(2, 6)), _sig(*H(6, 7)), _tanh(*H(7, 11)), _sig(*H(11, 12))
    w0 = _warp(H(0, 2), image0)
    w1 = _color(ima, imc, w0)
    return [_color(eya, eyc, w1), eya, eyc, w1, ima, imc, w0, H(0, 2)]
