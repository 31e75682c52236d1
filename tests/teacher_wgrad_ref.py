"""fp64 references of the encoder-decoders' weight-gradient convolution (tests/test_gpu_teacher_wgrad_kernels.py), built from
the kernel's own inputs: the operand x^ exactly as the kernel forms it from the stored tensor and the (A, B) coefficients it
reports, then dW by CPU autograd in fp64, and the bound's sum of |dz| |x^| per weight."""
import numpy as np
import torch
import torch.nn.functional as F

XF_NONE, XF_HALF, XF_FLOAT, XF_FLOAT16 = 0, 1, 2, 3


def _round(v: torch.Tensor, dtype) -> torch.Tensor:
    # one correctly rounded conversion from fp64 (numpy converts float64 -> float16 / float32 directly)
    return torch.from_numpy(v.numpy().astype(dtype).astype(np.float64))


def operand(x: torch.Tensor, xf: int, coef: torch.Tensor = None, norm_C: int = 0) -> torch.Tensor:
    """x^ [N, C, H, W] fp64 from the stored values x (fp32, or f16 values) and coef [N, norm_C, 2] (A, B): XF_HALF = one
    f16 FMA with f16 coefficients + ReLU (the fused normalisation of the default mode), XF_FLOAT = fp32 FMA + ReLU, XF_FLOAT16
    = the same rounded to f16.  Channels >= norm_C pass through.  x * A + B is exact in fp64 for these operands."""
    x = x.double()
    if xf == XF_NONE:
        return x
    a = coef[..., 0].double()[:, :, None, None]
    b = coef[..., 1].double()[:, :, None, None]
    v = x[:, :norm_C] * a + b
    if xf == XF_HALF:
        v = _round(v, np.float16).clamp_min(0.0)
    else:
        v = _round(v, np.float32).clamp_min(0.0)
        if xf == XF_FLOAT16:
            v = _round(v, np.float16)
    return torch.cat([v, x[:, norm_C:]], 1)


def wgrad(kind: int, xh: torch.Tensor, dz: torch.Tensor):
    """(dW, sum |dz| |x^|) in the reference layout.  kind 0 / 3: 3x3 s1 p1, 1: 4x4 s2 p1, 2: transposed 4x4 s2 p1."""
    N, C = xh.shape[:2]
    Co = dz.shape[1]

    def grad(a, b):
        if kind == 2:
            w = torch.zeros(C, Co, 4, 4, dtype=torch.float64, requires_grad=True)
            F.conv_transpose2d(a, w, stride=2, padding=1).backward(b)
        else:
            k, st = (4, 2) if kind == 1 else (3, 1)
            w = torch.zeros(Co, C, k, k, dtype=torch.float64, requires_grad=True)
            F.conv2d(a, w, stride=st, padding=1).backward(b)
        return w.grad

    return grad(xh, dz.double()), grad(xh.abs(), dz.double().abs())


def coef_ref(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor):
    """fp64 (A, B) [N, C, 2] of InstanceNorm2d(affine) of x [N, C, H, W] (eps 1e-5)."""
    x = x.double()
    mean = x.mean((2, 3))
    var = (x * x).mean((2, 3)) - mean * mean
    a = gamma.double()[None] / torch.sqrt(var.clamp_min(0.0) + 1e-5)
    return torch.stack([a, beta.double()[None] - mean * a], -1)


def expected_plan(M: int, D: int, pixels: int, ksplit: int = 0, sms: int = 132):
    """[N tile, M tiles, N tiles, pixel splits] as conv_wgrad_plan chooses them."""
    nt = 16 if D <= 16 else (64 if D <= 64 else 128)
    mt, ntl = -(-M // 64), -(-D // nt)
    kb = pixels // 32
    tiles = mt * ntl
    splits = ksplit if ksplit > 0 else (1 if tiles >= sms else -(-2 * sms // tiles))
    splits = max(1, min(splits, max(1, kb // 4)))
    per = -(-kb // splits)
    return [nt, mt, ntl, -(-kb // per)]
