"""Plain fp64 references of the teacher backward kernels (tha4_b200/csrc/unet_backward.cu, encdec_backward.cu), CPU only.

Each reference is torch's fp64 autograd of the forward op, run on exactly the inputs the kernel sees: the f16 values of an f16
tape, the TF32-rounded weights where the conv pack rounds them, and the ReLU mask of the float affine A x + B the kernel forms.
Next to each result it returns an elementwise worst-case bound on the kernel's error, computed from the same inputs: the
kernel's roundings (fp32 per-thread accumulation, fp32 affine coefficients, TF32 operands) applied to the magnitudes of the
terms, so that a cancelling sum is bounded by the sum of its absolute terms rather than by its result.
"""
import math

import torch
import torch.nn.functional as F

from distill_kernel_ref import round_tf32, ulp32

U32 = 2.0 ** -24          # unit roundoff of fp32
U_TF32_TRUNC = 2.0 ** -10  # relative error of an fp32 operand read as TF32 by truncation (wgmma kind::tf32)
U_3XTF32 = 2.0 ** -20      # relative error of one 3xTF32 product (the low x low term dropped, the split rounded)
EPS = 1e-5


# ------------------------------------------------------------------------------------------ helpers
def split_replicas(sums: torch.Tensor, rep: int, seed: int) -> torch.Tensor:
    """[N, C, 2] fp64 sums -> [rep, N, C, 2] replicas that add up to them: uneven random shares, replica 1 (if any) all
    zero, the last one takes the remainder."""
    if rep == 1:
        return sums.unsqueeze(0).clone()
    g = torch.Generator().manual_seed(seed)
    w = torch.rand((rep,) + tuple(sums.shape), generator=g, dtype=torch.float64) ** 3
    w[1] = 0.0
    w = w / w.sum(0, keepdim=True)
    out = w * sums.unsqueeze(0)
    out[-1] = sums - out[:-1].sum(0)
    return out


def stats_of(x: torch.Tensor) -> torch.Tensor:
    """Per-(n, c) sum and sum of squares [N, C, 2] of x [N, C, H, W] in fp64 (the statistics a producing conv accumulates)."""
    x = x.double()
    return torch.stack([x.sum((2, 3)), (x * x).sum((2, 3))], dim=-1)


def _group_moments(x: torch.Tensor, groups: int):
    """mean and rstd [N, C] (each channel gets its group's) as the kernels derive them from the fp64 sums."""
    N, C = x.shape[:2]
    cpg = C // groups
    s = stats_of(x).view(N, groups, cpg, 2).sum(2)
    cnt = float(x.shape[2] * x.shape[3] * cpg)
    mean = s[..., 0] / cnt
    var = (s[..., 1] / cnt - mean * mean).clamp_min(0.0)
    rstd = 1.0 / torch.sqrt(var + EPS)
    return mean.repeat_interleave(cpg, 1), rstd.repeat_interleave(cpg, 1)


def _film_factors(N, C, film0, film1):
    """(1 + s0)(1 + s1) [N, C] and the exact FiLM shift terms' magnitude bound, fp64."""
    one = torch.ones(N, C, dtype=torch.float64)
    s0 = one if film0 is None else (1 + film0[:C].double()).view(1, C).expand(N, C)
    s1 = one if film1 is None else 1 + film1[:, :C].double()
    b0 = torch.zeros(N, C, dtype=torch.float64) if film0 is None else film0[C:].double().view(1, C).expand(N, C)
    b1 = torch.zeros(N, C, dtype=torch.float64) if film1 is None else film1[:, C:].double()
    return s0, s1, b0, b1


def _gsum(t: torch.Tensor, groups: int) -> torch.Tensor:
    """[N, C] -> each channel gets the sum over its group's channels."""
    N, C = t.shape
    cpg = C // groups
    return t.view(N, groups, cpg).sum(2).repeat_interleave(cpg, 1)


def _bcast(t):
    return t.view(t.shape[0], t.shape[1], 1, 1)


# ------------------------------------------------------------------------------------------ normalisation backward
def norm_backward_ref(x, groups, gamma, beta, dy, act, film0=None, film1=None, dy_pool=False, res=None, res_mode=0, add=None,
                      relu_mask=None):
    """d(x) (and d(film1) when film1 is given) of
        out = pool?(act(FiLM1(FiLM0(GroupNorm(groups)(x)))))   [+ resample(x) paired with res]  [+ x paired with add]
    for the upstream gradients dy (of out), res and add; groups == C is InstanceNorm.  act 0 none, 1 ReLU (mask relu_mask:
    the kernel's own), 2 SiLU.  res_mode 1: identity, 2: the forward added nearest-x2(x) (res at 2x), 3: AvgPool2d(2)(x)
    (res at 1/2).  All fp64; returns (dx, dfilm or None, bound_dx, bound_dfilm or None)."""
    x = x.double()
    N, C, H, W = x.shape
    xr = x.clone().requires_grad_()
    f1r = film1.double().clone().requires_grad_() if film1 is not None else None
    h = F.group_norm(xr, groups, gamma.double(), beta.double(), eps=EPS)
    if film0 is not None:
        h = h * (1 + film0[:C].double().view(1, C, 1, 1)) + film0[C:].double().view(1, C, 1, 1)
    if film1 is not None:
        h = h * (1 + _bcast(f1r[:, :C])) + _bcast(f1r[:, C:])
    y = {0: h, 1: h * relu_mask if relu_mask is not None else F.relu(h), 2: F.silu(h)}[act]
    outs, grads = [F.avg_pool2d(y, 2) if dy_pool else y], [dy.double()]
    if res is not None:
        outs.append({1: xr, 2: F.interpolate(xr, scale_factor=2, mode='nearest'), 3: F.avg_pool2d(xr, 2)}[res_mode])
        grads.append(res.double())
    if add is not None:
        outs.append(xr)
        grads.append(add.double())
    torch.autograd.backward(outs, grads)
    dx = xr.grad.detach()
    dfilm = f1r.grad.detach() if film1 is not None else None
    bdx, bdf = _norm_bound(x, groups, gamma, beta, h.detach(), dy, act, film0, film1, dy_pool, res, res_mode, add, dx, relu_mask)
    return dx, dfilm, bdx, bdf


def _norm_bound(x, groups, gamma, beta, h, dy, act, film0, film1, dy_pool, res, res_mode, add, dx, relu_mask):
    """Elementwise bound on the fp32 kernel's error: dx = K dz - r1 - xhat r2 (+ residual, + add) with
    K = rstd gamma M, r1 = rstd mean_g(gamma M dz), r2 = rstd mean_g(gamma M dz xhat), M = the FiLM scales.
      * the affine (A, B) and (mean, rstd) are fp32 roundings of fp64 values: xhat is off by a few u times
        xa = rstd (|x| + |mean|), the SiLU argument by a few u times hs = |A| (|x| + |mean|) + |B terms|;
      * SiLU' moves by at most 1/2 per unit of its argument (|silu''| <= 1/2), plus its own few-ulp evaluation;
      * the sums over a group are fp32 per thread (at most 32 pixels) and fp64 beyond: 64 u of the absolute terms;
      * r2 is bounded with xa in place of |xhat|, which also covers the error of xhat inside the sum."""
    u = U32
    N, C, H, W = x.shape
    mean, rstd = _group_moments(x, groups)
    s0, s1, b0, b1 = _film_factors(N, C, film0, film1)
    M = s0 * s1
    gm = gamma.double().view(1, C) * M
    K = rstd * gm
    dyu = dy.double()
    if dy_pool:
        dyu = 0.25 * F.interpolate(dyu, scale_factor=2, mode='nearest')
    if act == 2:
        sg = torch.sigmoid(h)
        dz = dyu * sg * (1 + h * (1 - sg))
    elif act == 1:
        dz = dyu * (relu_mask if relu_mask is not None else (h > 0).double())
    else:
        dz = dyu
    xa = _bcast(rstd) * (x.abs() + _bcast(mean.abs()))
    hs = _bcast(K.abs()) * (x.abs() + _bcast(mean.abs())) + _bcast(beta.double().abs().view(1, C) * M.abs() + b0.abs() * s1.abs() + b1.abs())
    e_dz = dyu.abs() * (0.5 * 16 * u * hs + 8 * u) if act == 2 else torch.zeros_like(dyu)
    adz = dz.abs()
    cnt = float(H * W * (C // groups))
    T1, T2 = adz.sum((2, 3)), (adz * xa).sum((2, 3))                 # [N, C]
    E1, E2 = e_dz.sum((2, 3)), (e_dz * xa).sum((2, 3))
    r1_abs = rstd * _gsum(gm.abs() * T1, groups) / cnt
    r2_abs = rstd * _gsum(gm.abs() * T2, groups) / cnt
    r1_err = rstd * _gsum(gm.abs() * E1, groups) / cnt
    r2_err = rstd * _gsum(gm.abs() * E2, groups) / cnt
    bound = (_bcast(K.abs()) * e_dz + _bcast(r1_err) + xa * _bcast(r2_err)
             + 64 * u * (_bcast(K.abs()) * adz + _bcast(r1_abs) + xa * _bcast(r2_abs)))
    extra = torch.zeros_like(x)
    if res is not None:
        r = res.double().abs()
        extra = extra + {1: r, 2: F.avg_pool2d(r, 2) * 4, 3: 0.25 * F.interpolate(r, scale_factor=2, mode='nearest')}[res_mode]
    if add is not None:
        extra = extra + add.double().abs()
    bound = bound + 4 * u * (extra + dx.abs())
    bdf = None
    if film1 is not None:
        g, bt = gamma.double().view(1, C), beta.double().view(1, C)
        dS1, dS2 = 64 * u * T1 + E1, 64 * u * T2 + E2
        bscale = (g.abs() * dS2 + bt.abs() * dS1) * s0.abs() + b0.abs() * dS1 + 8 * u * ((g.abs() * T2 + bt.abs() * T1) * s0.abs() + b0.abs() * T1)
        bshift = dS1 + 4 * u * T1
        bdf = torch.cat([bscale, bshift], dim=1)
    return bound, bdf


def kernel_affine_f32(x, gamma, beta):
    """InstanceNorm's per-(n, c) affine (A, B) in the fp32 arithmetic of encdec_backward.cu (mean and rstd from the fp64
    sums, rounded once), and the fp64 value of A x + B from those fp32 coefficients."""
    x = x.double()
    N, C, H, W = x.shape
    s = stats_of(x)
    mean = s[..., 0] / (H * W)
    var = (s[..., 1] / (H * W) - mean * mean).clamp_min(0.0)
    mf, rf = mean.float(), (1.0 / torch.sqrt(var + EPS)).float()
    A = rf * gamma.float().view(1, C)
    B = beta.float().view(1, C) - mf * A
    z = x * _bcast(A.double()) + _bcast(B.double())
    scale = x.abs() * _bcast(A.double().abs()) + _bcast((mf * A).double().abs() + beta.double().abs().view(1, C))
    return z, scale


def relu_mask_and_ambiguous(x, gamma, beta):
    """The ReLU mask of the kernel's float affine, and the elements whose pre-activation is within rounding of 0 (there the
    mask depends on whether the compiler fused the multiply-add: tests give those elements a zero upstream gradient)."""
    z, scale = kernel_affine_f32(x, gamma, beta)
    ambiguous = z.abs() <= 16 * U32 * scale
    return (z > 0).double(), ambiguous


# ------------------------------------------------------------------------------------------ conv data gradient
def conv_dgrad_ref(kind, w, dy, in_hw, add=None, strict=False, round_w=True):
    """d(x) of the forward conv `kind` (0: 3x3 s1 p1, w [Cout, Cin, 3, 3]; 3: 1x1, w [Cout, Cin, 1, 1]) for dy, plus add,
    in fp64 with the weights the pack holds (TF32-rounded unless strict / round_w False).  Returns (dx, bound):
      default: the TF32 read of dy truncates (2^-10 relative), products of TF32 values are exact, fp32 accumulation over
               K = taps * Cout terms (gamma_K = K 2^-23, any order, split-K partials included);
      strict:  3xTF32 products (2^-20 relative) and the same accumulation,
    both on |W| (*) |dy|, plus the rounding of the sum with add."""
    wr = w.double() if (strict or not round_w) else round_tf32(w).double()
    N = dy.shape[0]
    Cin = w.shape[1]
    taps = w.shape[2] * w.shape[3]
    pad = w.shape[2] // 2

    def adj(wt, g):
        x = torch.zeros(N, Cin, in_hw[0], in_hw[1], dtype=torch.float64, requires_grad=True)
        F.conv2d(x, wt, None, 1, pad).backward(g)
        return x.grad.detach()
    dx = adj(wr, dy.double())
    mag = adj(wr.abs(), dy.double().abs())
    K = taps * w.shape[0]
    op = U_3XTF32 if strict else U_TF32_TRUNC
    bound = (op + K * 2.0 ** -23) * mag
    if add is not None:
        dx = dx + add.double()
        bound = bound + 2 * U32 * (mag + add.double().abs())
    return dx, bound


# ------------------------------------------------------------------------------------------ pose MLP
def silu_grad64(h):
    sg = torch.sigmoid(h.double())
    return sg * (1 + h.double() * (1 - sg))


def linear_backward_ref(dy, W, pre=None):
    """dx = SiLU'(pre) * (dy @ W) for dy [N, R], W [R, K].  The kernel accumulates in fp64 and rounds once to fp32, then
    multiplies by an fp32 SiLU'.  Returns (fp64 reference, elementwise bound): 1 ulp of the result without SiLU'; with it,
    a few ulps of the non-cancelling magnitude |t| sg (1 + |h (1 - sg)|) (SiLU' itself cancels near h = -1.28)."""
    t = dy.double() @ W.double()
    if pre is None:
        return t, ulp32(t)
    h = pre.double()
    sg = torch.sigmoid(h)
    ref = t * sg * (1 + h * (1 - sg))
    mag = t.abs() * sg * (1 + (h * (1 - sg)).abs())
    return ref, ulp32(ref) + 8 * ulp32(mag)


# ------------------------------------------------------------------------------------------ attention
def attention_ref(qkv, heads):
    """qkv_attention, 'new order' (the reference's unet.py QKVAttention): qkv [N, 3C, 16, 16] -> [N, C, 16, 16]."""
    b, c3, hh, ww = qkv.shape
    c, L = c3 // 3, hh * ww
    ch = c // heads
    q, k, v = qkv.reshape(b, c3, L).chunk(3, dim=1)
    scale = 1.0 / math.sqrt(math.sqrt(ch))
    w = torch.einsum('bct,bcs->bts', (q * scale).reshape(b * heads, ch, L), (k * scale).reshape(b * heads, ch, L))
    w = torch.softmax(w, dim=-1)
    return torch.einsum('bts,bcs->bct', w, v.reshape(b * heads, ch, L)).reshape(b, c, hh, ww)


def attention_backward_ref(qkv, dout, heads):
    """d(qkv) by fp64 autograd, and an elementwise bound on the fp32 kernel (unet_backward.cu: one thread per query / key, S
    recomputed per pass, P = exp(S - m) / l, D_i = sum_j P_ij dP_ij, dS = P (dP - D)):
      dP_ij = dO_i . v_j and S_ij are fp32 dot products of 32 terms: 32 u of their absolute versions;
      P_ij carries the error of S_ij - m_i (32 u of |S|_ij and of the row maximum's |S|) plus that of the exp and of l
      (300 u): dP_rel_ij = 32 u (|S|_ij + |S|_i,max) + 300 u;
      every sum over 256 rows / keys is fp32: 256 u of its absolute terms."""
    q64 = qkv.double().clone().requires_grad_()
    attention_ref(q64, heads).backward(dout.double())
    ref = q64.grad.detach()
    b, c3, hh, ww = qkv.shape
    c, L = c3 // 3, hh * ww
    ch = c // heads
    s = 1.0 / math.sqrt(math.sqrt(ch))
    q, k, v = [t.reshape(b * heads, ch, L).transpose(1, 2) for t in qkv.double().reshape(b, c3, L).chunk(3, dim=1)]   # [bh, L, ch]
    go = dout.double().reshape(b * heads, ch, L).transpose(1, 2)
    u = U32
    S = s * s * q @ k.transpose(1, 2)
    Sabs = s * s * q.abs() @ k.abs().transpose(1, 2)
    P = torch.softmax(S, dim=-1)
    dP = go @ v.transpose(1, 2)
    dPabs = go.abs() @ v.abs().transpose(1, 2)
    D = (P * dP).sum(-1, keepdim=True)
    rel_p = 32 * u * (Sabs + Sabs.amax(-1, keepdim=True)) + 300 * u
    eP = P * rel_p
    e_dP = 32 * u * dPabs
    e_D = (eP * dP.abs() + P * e_dP).sum(-1, keepdim=True) + 256 * u * (P * dP.abs()).sum(-1, keepdim=True)
    dS = P * (dP - D)
    e_dS = eP * (dP - D).abs() + P * (e_dP + e_D) + 2 * u * dS.abs()
    Lu = 300 * u
    e_dq = s * s * (e_dS @ k.abs() + Lu * dS.abs() @ k.abs())
    e_dk = s * s * (e_dS.transpose(1, 2) @ q.abs() + Lu * dS.abs().transpose(1, 2) @ q.abs())
    e_dv = eP.transpose(1, 2) @ go.abs() + Lu * P.transpose(1, 2) @ go.abs()
    bound = torch.cat([t.transpose(1, 2).reshape(b, c, hh, ww) for t in (e_dq, e_dk, e_dv)], dim=1)
    return ref, bound
