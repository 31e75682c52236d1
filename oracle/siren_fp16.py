"""CPU restatement of the SIREN student kernels at their rounding points  --  TEST INFRASTRUCTURE, NOT PRODUCT.

tha4_oracle.py restates the students in fp32; the kernels (tha4_b200/csrc/siren_tc.cu, siren.cu) store every activation
in fp16, and that rounding is larger than anything a subtly wrong kernel changes.  This module computes one level the way
the kernels do, rounding exactly where they round:

  weights     fp16(fp32(30 W)), biases fp32(30 b); the head unscaled: fp16 weights, fp32 bias
  first layer per-sample term fp32(30 b + (30 W_pose) . pose) plus the xy terms at the tha4_base_grid coordinates
  GEMMs       the exact products of the fp16 operands, summed in fp64
  activations sin (fp64) of the fp32 argument, rounded to fp16 (round to nearest even)
  upsample    wgmma path: fp16 tap weights, HMUL2 then three HFMA2, each rounded once to fp16;
              mma.sync path: fp32 lerp, rounded once
  level 2     head -> grid_sample through the C oracle (oracle/gridsample_ref.c, the bit-exact index math) -> blend

A level is given in the reference's layout: a list of (weight [N, Cin], bias [N]) per sine layer, plus the head.  The
first layer's input channels are the previous level's channels (levels 1 / 2), then x, y, then the pose.

`mutate` injects one of the faults the tests must be able to see (MUTATIONS); the tests check that each is caught.
"""
import ctypes
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch
from torch import Tensor

RESOLUTION = {0: 128, 1: 256, 2: 512, 3: 128}      # mode -> R (0..2: body levels, 3: face)
ELEMENTWISE = (0, 3)                                # modes whose first layer has no GEMM

MUTATIONS = ('bias_slice', 'swap_xy', 'align_corners', 'drop_last_k', 'pose0', 'half_pixel')

# test 1 bound (single layers): 1 fp16 ulp of the reference + fp32 accumulation for |argument| <= 50 + st_sin's 3.6e-6
ULP_SLACK = 3e-5
# test 2 bounds (production levels, init-like weights): from a CPU perturbation proxy (~1e-3 max / 5e-5 mean)
LEVEL_MAX, LEVEL_MEAN = 4e-3, 2e-4


def f16(x: Tensor) -> Tensor:
    """round to fp16 (nearest even), kept as float64"""
    return x.to(torch.float16).to(torch.float64)


def f32(x: Tensor) -> Tensor:
    return x.to(torch.float32).to(torch.float64)


def base_grid(size: int, shift: float = 0.0) -> Tensor:
    """tha4o_base_grid (oracle/gridsample_ref.c) in fp32 arithmetic, as float64"""
    i = np.arange(size, dtype=np.float32)
    step = np.float32(2.0) / np.float32(size - 1)
    lo = np.float32(-1.0) + step * i
    hi = np.float32(1.0) - step * (np.float32(size - 1) - i)
    v = np.where(np.arange(size) < size // 2, lo, hi).astype(np.float32)
    v = (v * np.float32(size - 1)).astype(np.float32) / np.float32(size)
    return torch.from_numpy(v.astype(np.float64)) + shift


def _lerp_taps(out_size: int, in_size: int, align_corners: bool = False):
    """lerp_locate (gridsample.cuh) for scale 1/2 in fp32: indices i0, i1 and weights l0, l1 per output coordinate"""
    d = np.arange(out_size, dtype=np.float32)
    if align_corners:
        f = d * np.float32((in_size - 1) / (out_size - 1))
    else:
        f = np.float32(0.5) * (d + np.float32(0.5)) - np.float32(0.5)
    f = np.maximum(f, np.float32(0.0)).astype(np.float32)
    i0 = f.astype(np.int64)
    i1 = np.minimum(i0 + 1, in_size - 1)
    l1 = (f - i0.astype(np.float32)).astype(np.float32)
    l0 = (np.float32(1.0) - l1).astype(np.float32)
    return torch.from_numpy(i0), torch.from_numpy(i1), torch.from_numpy(l0.astype(np.float64)), torch.from_numpy(l1.astype(np.float64))


def upsample(prev: Tensor, variant: str = 'wgmma', align_corners: bool = False) -> Tensor:
    """bilinear x2 of prev [B, h, h, C] (fp16 values) -> [B, 2h, 2h, C] fp16 values, as the kernels' prologues compute it"""
    h = prev.shape[1]
    i0, i1, l0, l1 = _lerp_taps(2 * h, h, align_corners)
    a = prev[:, i0][:, :, i0]      # (y0, x0)
    b = prev[:, i0][:, :, i1]      # (y0, x1)
    c = prev[:, i1][:, :, i0]      # (y1, x0)
    d = prev[:, i1][:, :, i1]      # (y1, x1)
    ly0, ly1 = l0.view(1, -1, 1, 1), l1.view(1, -1, 1, 1)
    lx0, lx1 = l0.view(1, 1, -1, 1), l1.view(1, 1, -1, 1)
    if variant == 'wgmma':
        # HMUL2 + 3 HFMA2 on fp16 tap weights fp16(fp32(ly * lx)); fp64 holds every product and sum exactly here
        w00, w01, w10, w11 = f16(f32(ly0 * lx0)), f16(f32(ly0 * lx1)), f16(f32(ly1 * lx0)), f16(f32(ly1 * lx1))
        o = f16(w00 * a)
        o = f16(w01 * b + o)
        o = f16(w10 * c + o)
        return f16(w11 * d + o)
    return f16(ly0 * (lx0 * a + lx1 * b) + ly1 * (lx0 * c + lx1 * d))


def _sin16(arg: Tensor) -> Tensor:
    return f16(torch.sin(f32(arg)))


def level_forward(mode: int, layers: Sequence[Tuple[Tensor, Tensor]], pose: Tensor, head: Optional[Tuple[Tensor, Tensor]] = None,
                  prev: Optional[Tensor] = None, image: Optional[Tensor] = None, clib=None, variant: str = 'wgmma',
                  R: Optional[int] = None, mutate: Optional[str] = None, nb: int = 64):
    """One level.  pose [B, P]; prev [B, R/2, R/2, >= feat] (fp16 values, levels 1 / 2); image [B,4,R,R] and clib for a
    level-2 head.  Returns the last sine layer's activations [B, R, R, N] (fp16 values, float64) without a head, the
    tail outputs [blended, alpha, color, warped, grid_change] (NCHW) for level 2, or [B,4,R,R] for the face."""
    assert mutate is None or mutate in MUTATIONS, mutate
    R = R or RESOLUTION[mode]
    B, P = pose.shape
    pose = pose.double()
    if mutate == 'pose0':
        pose = pose[:1].expand(B, P)
    xs = base_grid(R, 1.0 / R if mutate == 'half_pixel' else 0.0)
    W0, b0 = layers[0]
    feat = W0.shape[1] - 2 - P
    assert (feat == 0) == (mode in ELEMENTWISE), (mode, feat)

    def scaled(W, b):
        return f32((W.float() * 30.0).double()), f32((b.float() * 30.0).double())

    def slice_bias(bias):
        if mutate != 'bias_slice' or bias.shape[-1] <= nb:
            return bias
        w = min(nb, bias.shape[-1] - nb)         # the real columns of the second slice
        bias = bias.clone()
        bias[..., nb:nb + w] = bias[..., :w]
        return bias

    def gemm(a, Wh):
        K = Wh.shape[1]
        if mutate == 'drop_last_k' and K > 64:
            Wh = Wh.clone()
            Wh[:, 64 * ((K - 1) // 64):] = 0
        return a.reshape(-1, K) @ Wh.t()

    # first layer: per-sample term fp32(30 b + (30 W_pose) . pose) + the xy terms
    W0s, b0s = scaled(W0, b0)
    wx, wy = W0s[:, feat], W0s[:, feat + 1]
    if mutate == 'swap_xy':
        wx, wy = wy, wx
    pb = f32(b0s + pose @ W0s[:, feat + 2:].t())                                                # [B, N0]
    first = pb.view(B, 1, 1, -1) + wx.view(1, 1, 1, -1) * xs.view(1, 1, R, 1) + wy.view(1, 1, 1, -1) * xs.view(1, R, 1, 1)
    if mode in ELEMENTWISE:
        a = _sin16(first)
    else:
        up = upsample(prev[..., :feat].double(), variant, mutate == 'align_corners')
        z = gemm(up, f16(W0s[:, :feat])).view(B, R, R, -1)
        a = _sin16(z + slice_bias(first))
    for W, b in layers[1:]:
        Ws, bs = scaled(W, b)
        z = gemm(a, f16(Ws)).view(B, R, R, -1)
        a = _sin16(z + slice_bias(bs))
    if head is None:
        return a
    Wh, bh = head
    o = gemm(a, f16(Wh.float().double())).view(B, R, R, -1) + bh.float().double()
    o = o.permute(0, 3, 1, 2)                                                                    # NCHW
    if mode == 3:
        return o[:, :4]
    gc = f32(o[:, 0:2]).float().contiguous()
    alpha, color = f32(o[:, 2:3]), f32(o[:, 3:7])
    warped = grid_sample(clib, image.float().contiguous(), gc).double()
    blended = (1 - alpha) * warped + alpha * color
    return [blended, alpha, color, warped, gc.double()]


def grid_sample(clib, image: Tensor, grid_change: Tensor) -> Tensor:
    N, C, H, W = image.shape
    out = torch.empty_like(image)
    p = lambda t: ctypes.c_void_p(t.data_ptr())     # noqa: E731
    clib.tha4o_grid_sample(p(image), p(grid_change), N, C, H, W, p(out), None, None, None, None)
    return out


def layer(sd, key: str) -> Tuple[Tensor, Tensor]:
    """(weight [N, Cin], bias [N]) of the 1x1 conv `key` of a student state_dict"""
    w = sd[key + '.weight']
    return w.reshape(w.shape[0], -1), sd[key + '.bias']


# ------------------------------------------------------------------------------------------------ comparisons
def ulp_ratio(out: Tensor, ref: Tensor) -> Tuple[float, float, float]:
    """max over elements of |out - ref| / (ulp_fp16(ref) + ULP_SLACK) (<= 1 passes), and the max / mean error"""
    ref = ref.double()
    d = (out.double() - ref).abs()
    ulp = torch.from_numpy(np.spacing(np.abs(ref.numpy().astype(np.float16))).astype(np.float64))
    return (d / (ulp + ULP_SLACK)).max().item(), d.max().item(), d.mean().item()


def level_ratio(out, ref) -> Tuple[float, float, float]:
    """max(max error / LEVEL_MAX, mean error / LEVEL_MEAN) over one tensor or a list of tensors (<= 1 passes)"""
    outs, refs = (out, ref) if isinstance(out, (list, tuple)) else ([out], [ref])
    mx = max((o.double() - r.double()).abs().max().item() for o, r in zip(outs, refs))
    mean = max((o.double() - r.double()).abs().mean().item() for o, r in zip(outs, refs))
    return max(mx / LEVEL_MAX, mean / LEVEL_MEAN), mx, mean


# ------------------------------------------------------------------------------------------------ test weights
def controlled_layer(g: torch.Generator, n: int, k: int, extra: int = 0, bias_max: float = 40.0, l1: float = 10.0):
    """A sine layer whose argument stays within |30 b| + l1 <= 50 for inputs in [-1, 1]: 30 b uniform in
    +-bias_max, each row of 30 W scaled to an L1 norm in [0.3, 1] * l1.  extra: input columns beyond k (xy + pose)."""
    W = torch.rand(n, k + extra, generator=g) * 2 - 1
    W = W / W.abs().sum(1, keepdim=True) * (0.3 + 0.7 * torch.rand(n, 1, generator=g)) * (l1 / 30.0)
    b = (torch.rand(n, generator=g) * 2 - 1) * (bias_max / 30.0)
    return W.float(), b.float()


def exact_first_layer(g: torch.Generator, n: int, pose: Tensor, margin: float = 1e-5):
    """An elementwise first layer whose activations the kernels compute bit-exactly: no xy weights, and 30 b, 30 W_pose and
    the pose on dyadic grids, so that every fp32 sum is exact in any order; biases are redrawn until sin of every
    argument lies `margin` away from an fp16 rounding midpoint (st_sin is within 4e-6 of sin).  pose entries must be
    multiples of 1/8 in [-1, 1].  Returns (W [n, 2 + P], b [n])."""
    B, P = pose.shape
    assert torch.equal(pose * 8, (pose * 8).round()) and pose.abs().max() <= 1
    Wp = torch.randint(-64, 65, (n, P), generator=g).double() * 2.0 ** -14          # 30 Wp: multiples of 15 * 2^-13, |.| < 0.12
    k = torch.randint(-19000, 19001, (n,), generator=g).double()                     # 30 b = 15 k 2^-13, |.| < 35
    for _ in range(100):
        arg = 30.0 * (k * 2.0 ** -14) + pose.double() @ (30.0 * Wp).t()              # exact
        s = torch.sin(arg)
        lo = s.to(torch.float16).double()
        nxt = torch.from_numpy(np.nextafter(lo.numpy().astype(np.float16), np.where(s.numpy() > lo.numpy(), 1, -1).astype(np.float16)).astype(np.float64))
        near = ((s - (lo + nxt) / 2).abs() < margin).any(0)
        if not near.any():
            break
        k[near] = torch.randint(-19000, 19001, (int(near.sum()),), generator=g).double()
    else:
        raise RuntimeError('exact_first_layer: no biases found')
    W = torch.cat([torch.zeros(n, 2, dtype=torch.float64), Wp], 1)
    return W.float(), (k * 2.0 ** -14).float()
