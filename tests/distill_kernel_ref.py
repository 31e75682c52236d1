"""Plain fp64 references of the student training kernels (tha4_b200/csrc/distill.cu), CPU only.

Each reference rounds where the kernel rounds (TF32 weights, the fp32 sample position of grid_sample) and is exact
everywhere else, so that the tests can bound the remaining difference from the inputs.  Dyadic inputs (few significant
bits) make every product and partial sum exact in fp32: on them a kernel must equal its reference bit for bit, whatever
its summation order or atomics.
"""
import ctypes

import torch
import torch.nn.functional as F

U32 = 2.0 ** -24          # unit roundoff of fp32


# ------------------------------------------------------------------------------------------ rounding and dyadic values
def round_tf32(x: torch.Tensor) -> torch.Tensor:
    """cvt.rna.tf32.f32: the nearest fp32 value with 10 explicit mantissa bits, ties away from zero."""
    x = x.float().contiguous()
    b = x.view(torch.int32)
    r = ((b + 0x1000) & ~0x1FFF).view(torch.float32)     # add half a TF32 ulp to the magnitude, drop 13 bits
    return torch.where(torch.isfinite(x), r, x)


def ulp32(x: torch.Tensor) -> torch.Tensor:
    """Spacing of fp32 numbers at |x| (fp64 result; the subnormal spacing below the smallest normal)."""
    a = x.double().abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 23)


def dyadic(shape, bits: int, exp: int, seed: int, device='cpu') -> torch.Tensor:
    """k * 2**-exp with integer |k| < 2**bits (fp32).  bits <= 11 keeps the values exact in TF32."""
    g = torch.Generator(device=device).manual_seed(seed)
    k = torch.randint(-(2 ** bits) + 1, 2 ** bits, tuple(shape), generator=g, dtype=torch.int32, device=device)
    return k.float() * 2.0 ** -exp


def dyadic_unit(bits: int, exp: int):
    """(largest magnitude, unit) of dyadic(bits, exp)"""
    return (2 ** bits - 1) * 2.0 ** -exp, 2.0 ** -exp


def assert_exact_sums(n_terms: int, max_term: float, unit: float, start: float = 0.0):
    """Precondition of a bit-exact comparison: every partial sum of `start` and up to n_terms terms, each a multiple of
    `unit` of magnitude <= max_term, is a multiple of `unit` below 2**24 units, hence exact in fp32 in any order."""
    worst = abs(start) + n_terms * max_term
    assert start / unit == round(start / unit) and max_term / unit == round(max_term / unit), (start, max_term, unit)
    assert worst / unit < 2 ** 24, 'dyadic inputs too wide for exact fp32 sums: %g units' % (worst / unit)


# ------------------------------------------------------------------------------------------ bilinear x2 and the base grid
def base_grid(oracle_clib, size: int) -> torch.Tensor:
    b = torch.empty(size)
    oracle_clib.tha4o_base_grid(size, ctypes.c_void_p(b.data_ptr()))
    return b


def upsample2(oracle_clib, x: torch.Tensor) -> torch.Tensor:
    """interpolate(x [N,C,h,w], x2, bilinear, align_corners=False) in fp32, bit-exact to the library (the C oracle)."""
    x = x.float().contiguous()
    n, c, h, w = x.shape
    out = torch.empty(n, c, 2 * h, 2 * w)
    oracle_clib.tha4o_resize_bilinear(ctypes.c_void_p(x.data_ptr()), n, c, h, w, 2 * h, 2 * w, ctypes.c_void_p(out.data_ptr()))
    return out


def upsample2_adjoint(d: torch.Tensor) -> torch.Tensor:
    """Adjoint of the bilinear x2 map (align_corners=False) in fp64: d [N,C,2h,2w] -> [N,C,h,w], by autograd."""
    n, c, H, W = d.shape
    p = torch.zeros(n, c, H // 2, W // 2, dtype=torch.float64, requires_grad=True)
    F.interpolate(p, scale_factor=2, mode='bilinear', align_corners=False).backward(d.double())
    return p.grad


def upsample2_weights_abs(d: torch.Tensor) -> torch.Tensor:
    """sum over the taps of |w| |d| for each source pixel (the magnitude the adjoint's rounding is relative to)"""
    return upsample2_adjoint(d.double().abs())


# ------------------------------------------------------------------------------------------ loss and gradient tails
def sample_grid64(oracle_clib, gc: torch.Tensor):
    """gc [N,2,R,R] fp32 (a leaf of fp64 autograd as gc64) -> the fp64 grid for F.grid_sample whose unnormalised position
    is the kernel's fp32 one, ((base + gc + 1) R - 1) / 2 rounded at every step, and whose gradient is that of base + gc."""
    R = gc.shape[-1]
    b = base_grid(oracle_clib, R)
    gc = gc.float()
    gx, gy = b.view(1, 1, R) + gc[:, 0], b.view(1, R, 1) + gc[:, 1]
    ix, iy = (((gx + 1) * R) - 1) / 2, (((gy + 1) * R) - 1) / 2          # fp32, as sample_locate
    gc64 = gc.double().requires_grad_()
    pos = torch.stack([(2 * ix.double() + 1) / R - 1, (2 * iy.double() + 1) / R - 1], dim=-1)
    grid = pos + (gc64 - gc64.detach()).permute(0, 2, 3, 1)
    return gc64, grid


def body_outputs64(oracle_clib, out7: torch.Tensor, image: torch.Tensor):
    """out7 [N,R,R,8] fp32 -> fp64 leaves (gc, alpha, colour) and the outputs blended, alpha, colour, warped, grid_change"""
    gc64, grid = sample_grid64(oracle_clib, out7[..., 0:2].permute(0, 3, 1, 2).contiguous())
    alpha = out7[..., 2:3].permute(0, 3, 1, 2).double().requires_grad_()
    col = out7[..., 3:7].permute(0, 3, 1, 2).double().requires_grad_()
    warped = F.grid_sample(image.double(), grid, mode='bilinear', padding_mode='border', align_corners=False)
    blended = (1 - alpha) * warped + alpha * col
    return (gc64, alpha, col), (blended, alpha, col, warped, gc64)


def _d_out7(leaves):
    gc, alpha, col = leaves
    z = lambda t: torch.zeros_like(t) if t.grad is None else t.grad
    d = torch.cat([z(gc), z(alpha), z(col), torch.zeros_like(alpha)], dim=1)
    return d.permute(0, 2, 3, 1).contiguous()


def body_loss_ref(oracle_clib, out7, image, T0, T2, T3, w):
    """train_tail_kernel in fp64: the four sums of |a - b| and d out7 of sum_i w_i mean|term_i| (torch's sgn(0) = 0)"""
    leaves, (bl, _, col, wp, gc) = body_outputs64(oracle_clib, out7, image)
    terms = [bl - T0.double(), wp - T2.double(), gc - T3.double(), col - T0.double()]
    loss = sum(wi * t.abs().mean() for wi, t in zip(w, terms))
    loss.backward()
    return torch.tensor([t.detach().abs().sum().item() for t in terms], dtype=torch.float64), _d_out7(leaves)


def body_grad_ref(oracle_clib, out7, image, g):
    """grad_tail_kernel in fp64: d out7 of sum_i <g_i, output_i> (g: five NCHW tensors or None)"""
    leaves, outs = body_outputs64(oracle_clib, out7, image)
    pairs = [(o, gi.double()) for o, gi in zip(outs, g) if gi is not None]
    if pairs:
        torch.autograd.backward([o for o, _ in pairs], [gi for _, gi in pairs])
    return _d_out7(leaves)


def face_loss_ref(out4, target, mask, w):
    """face_tail_kernel in fp64: out4 [N,R,R,4] -> sums of |o - t| and |(t - o) m|, d out4 of w0 mean|o-t| + w1 mean|(t-o) m|"""
    o = out4.permute(0, 3, 1, 2).double().requires_grad_()
    t, m = target.double(), mask.double()
    a, b = o - t, (t - o) * m
    (w[0] * a.abs().mean() + w[1] * b.abs().mean()).backward()
    sums = torch.tensor([a.detach().abs().sum().item(), b.detach().abs().sum().item()], dtype=torch.float64)
    return sums, o.grad.permute(0, 2, 3, 1).contiguous()
