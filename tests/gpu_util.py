"""Helpers for the -m gpu tests: thin ctypes wrappers over the kernel-level entry points of the C ABI."""
import ctypes

import torch

from tha4_b200._lib import Context, _ptr

_ctx = None


def ctx() -> Context:
    global _ctx
    if _ctx is None:
        _ctx = Context(torch.device('cuda:0'))
    return _ctx


def dev(t):
    return t.to('cuda:0').contiguous()


def conv(kind, x, w, bias=None, res=None, res_mode=0, in_up=0, strict=1, ksplit=0):
    c = ctx()
    N, Cin, H, W = x.shape
    Cout = w.shape[1] if kind == 2 else w.shape[0]
    LH, LW = (2 * H, 2 * W) if in_up else (H, W)
    Ho, Wo = {0: (LH, LW), 1: (LH // 2, LW // 2), 2: (LH * 2, LW * 2), 3: (LH, LW), 4: (LH * 2, LW * 2)}[kind]
    y = torch.empty(N, Cout, Ho, Wo, device='cuda:0')
    xd, wd = dev(x), dev(w)
    bd = dev(bias) if bias is not None else None
    rd = dev(res) if res is not None else None
    c._call('tha4_test_conv', kind, _ptr(xd), _ptr(wd), _ptr(bd), _ptr(rd), res_mode, in_up, _ptr(y), N, Cin, H, W, Cout,
            strict, ksplit, c._stream())
    torch.cuda.synchronize()
    return y.cpu()


def conv_norm(kind, x, norm_C, groups, gamma, beta, film0, film1, act, w, bias=None, res=None, res_mode=0, ksplit=0):
    """conv(act(norm(x))) through the fused-input-normalisation wgmma kernel; returns (fp32 output, f16 copy widened)."""
    c = ctx()
    N, Cin, H, W = x.shape
    Cout = w.shape[1] if kind == 2 else w.shape[0]
    Ho, Wo = {0: (H, W), 1: (H // 2, W // 2), 2: (H * 2, W * 2), 3: (H, W), 4: (H * 2, W * 2)}[kind]
    y = torch.empty(N, Cout, Ho, Wo, device='cuda:0')
    y16 = torch.empty_like(y)
    t = [dev(v) if v is not None else None for v in (x, gamma, beta, film0, film1, w, bias, res)]
    c._call('tha4_test_conv_norm', kind, _ptr(t[0]), N, Cin, H, W, norm_C, groups, _ptr(t[1]), _ptr(t[2]), _ptr(t[3]), _ptr(t[4]), act,
            _ptr(t[5]), _ptr(t[6]), _ptr(t[7]), res_mode, Cout, ksplit, _ptr(y), _ptr(y16), c._stream())
    torch.cuda.synchronize()
    return y.cpu(), y16.cpu()


def norm(x, groups, gamma, beta, film0=None, film1=None, act=0, pool=0, out_f16=0):
    c = ctx()
    N, C, H, W = x.shape
    y = torch.empty(N, C, H // 2 if pool else H, W // 2 if pool else W, device='cuda:0')
    args = [dev(x), dev(gamma), dev(beta), dev(film0) if film0 is not None else None, dev(film1) if film1 is not None else None]
    c._call('tha4_test_norm', _ptr(args[0]), N, C, H, W, groups, _ptr(args[1]), _ptr(args[2]), _ptr(args[3]), _ptr(args[4]),
            act, pool, out_f16, _ptr(y), c._stream())
    torch.cuda.synchronize()
    return y.cpu()


TAIL_OUT_SPECS = {0: [4, 1, 4, 2, 4], 1: [4, 1, 4, 4, 1, 4], 2: [4, 1, 4, 4, 1, 4, 4, 2], 3: [4, 1, 4, 4, 1, 4, 4, 2]}


def tail(kind, feature, gamma, beta, groups, act, head_ws, head_bs, image0, image1=None, strict=0):
    """head_ws: list of [cout_i, C, 3, 3]; head_bs: list of [cout_i] or None (bias-free head)."""
    c = ctx()
    N, C, S, _ = feature.shape
    outs = [torch.empty(N, ch, S, S, device='cuda:0') for ch in TAIL_OUT_SPECS[kind]]
    hw = dev(torch.cat([w.reshape(-1) for w in head_ws]))
    hb = dev(torch.cat([(b if b is not None else torch.zeros(w.shape[0])) for w, b in zip(head_ws, head_bs)]))
    couts = (ctypes.c_int * len(head_ws))(*[w.shape[0] for w in head_ws])
    f, g, b, i0 = dev(feature), dev(gamma), dev(beta), dev(image0)
    i1 = dev(image1) if image1 is not None else None
    from tha4_b200._lib import _ptr_array
    c._call('tha4_test_tail', kind, _ptr(f), N, C, S, _ptr(g), _ptr(b), groups, act, _ptr(hw), _ptr(hb), couts, len(head_ws),
            _ptr(i0), _ptr(i1), _ptr_array(outs), strict, c._stream())
    torch.cuda.synchronize()
    return [o.cpu() for o in outs]


def attention(qkv, heads=8):
    c = ctx()
    N, C3 = qkv.shape[0], qkv.shape[1]
    out = torch.empty(N, C3 // 3, 16, 16, device='cuda:0')
    q = dev(qkv)
    c._call('tha4_test_attention', _ptr(q), N, C3 // 3, heads, _ptr(out), c._stream())
    torch.cuda.synchronize()
    return out.cpu()


def linear(x, W, b, silu_in):
    c = ctx()
    y = torch.empty(x.shape[0], W.shape[0], device='cuda:0')
    xd, wd, bd = dev(x), dev(W), dev(b)
    c._call('tha4_test_linear', _ptr(xd), x.shape[0], x.shape[1], _ptr(wd), _ptr(bd), W.shape[0], silu_in, _ptr(y), c._stream())
    torch.cuda.synchronize()
    return y.cpu()


SIREN_R = {0: 128, 1: 256, 2: 512, 3: 128}


def siren_level(path, mode, layers, pose, pose_dim, head=None, npad=None, nb=None, prev=None, image=None, out_f16=0):
    """One student level (tha4_test_siren_level).  layers: [(W [N, Cin], b [N])] in the reference layout; pose [B, pose_ld]
    of which the first pose_dim entries are the pose; prev: fp16 [B, R/2, R/2, prev_c].  npad defaults to N rounded up to
    32, nb to 96 (or 64 / 16 where 96 does not fit).  Returns the activations [B, R, R, N] as fp16 (no head), the five
    tail planes (level 2) or the face [B,4,R,R], on the CPU."""
    from tha4_b200._lib import _ptr_array
    c = ctx()
    R = SIREN_R[mode]
    B = pose.shape[0]
    sd = {}
    for i, (W, b) in enumerate(layers):
        sd['layer.%d.weight' % i], sd['layer.%d.bias' % i] = dev(W.float()), dev(b.float())
    if head is not None:
        sd['head.weight'], sd['head.bias'] = dev(head[0].float()), dev(head[1].float())
    keys = list(sd)
    shapes = (ctypes.c_int64 * (4 * len(keys)))()
    ndims = (ctypes.c_int * len(keys))()
    for i, k in enumerate(keys):
        ndims[i] = sd[k].dim()
        for d in range(4):
            shapes[4 * i + d] = sd[k].shape[d] if d < sd[k].dim() else 1
    npad = list(npad) if npad is not None else [(W.shape[0] + 31) // 32 * 32 for W, _ in layers]
    n_gemm = len(layers) - (1 if mode in (0, 3) else 0) + (1 if head is not None else 0)
    if nb is None:
        gemm_npad = npad[1:] if mode in (0, 3) else npad
        nb = [next(w for w in (96, 64, 16) if n % w == 0 and not (mode == 3 and w == 96)) for n in gemm_npad] + ([16] if head is not None else [])
    assert len(nb) == n_gemm, (nb, n_gemm)
    pd, prevd = dev(pose.float()), (dev(prev.half()) if prev is not None else None)
    imaged = dev(image.float()) if image is not None else None
    if head is None:
        outs = [torch.empty(B, R, R, npad[-1], dtype=torch.float16, device='cuda:0')]
    elif mode == 3:
        outs = [torch.empty(B, 4, R, R, device='cuda:0')]
    else:
        dt = torch.float16 if out_f16 else torch.float32
        outs = [torch.empty(B, ch, R, R, dtype=dt, device='cuda:0') for ch in (4, 1, 4, 4, 2)]
    c._call('tha4_test_siren_level', path, mode, len(keys), (ctypes.c_char_p * len(keys))(*[k.encode() for k in keys]),
            _ptr_array([sd[k] for k in keys]), shapes, ndims, len(layers), int(head is not None), pose_dim,
            (ctypes.c_int * len(npad))(*npad), (ctypes.c_int * len(nb))(*nb), _ptr(pd), pose.shape[1], B, _ptr(prevd),
            prev.shape[3] if prev is not None else 0, _ptr(imaged), out_f16, _ptr_array(outs), c._stream())
    torch.cuda.synchronize()
    if head is None:
        return outs[0][..., :layers[-1][0].shape[0]].cpu()
    return outs[0].cpu() if mode == 3 else [o.cpu() for o in outs]


def sine(which, x):
    c = ctx()
    xd = dev(x.float())
    y = torch.empty_like(xd)
    c._call('tha4_test_sine', which, _ptr(xd), ctypes.c_int64(xd.numel()), _ptr(y), c._stream())
    torch.cuda.synchronize()
    return y.cpu()


def grid_sample(img, gc, want_taps=True):
    c = ctx()
    N, C, H, W = img.shape
    out = torch.empty(N, C, H, W, device='cuda:0')
    x0 = torch.empty(N, H, W, dtype=torch.int32, device='cuda:0')
    y0 = torch.empty_like(x0)
    tx = torch.empty(N, H, W, device='cuda:0')
    ty = torch.empty_like(tx)
    i, g = dev(img), dev(gc)
    c._call('tha4_grid_sample', _ptr(i), _ptr(g), N, C, H, W, _ptr(out), _ptr(x0), _ptr(y0), _ptr(tx), _ptr(ty), c._stream())
    torch.cuda.synchronize()
    return out.cpu(), x0.cpu(), y0.cpu(), tx.cpu(), ty.cpu()


def resize(x, ho, wo):
    c = ctx()
    N, C, H, W = x.shape
    out = torch.empty(N, C, ho, wo, device='cuda:0')
    xd = dev(x)
    c._call('tha4_resize_bilinear', _ptr(xd), N, C, H, W, ho, wo, _ptr(out), c._stream())
    torch.cuda.synchronize()
    return out.cpu()


def oracle_grid_sample(clib, img, gc):
    N, C, H, W = img.shape
    out = torch.empty_like(img)
    x0 = torch.empty(N, H, W, dtype=torch.int32)
    y0 = torch.empty_like(x0)
    tx = torch.empty(N, H, W)
    ty = torch.empty_like(tx)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    img, gc = img.contiguous(), gc.contiguous()
    clib.tha4o_grid_sample(p(img), p(gc), N, C, H, W, p(out), p(x0), p(y0), p(tx), p(ty))
    return out, x0, y0, tx, ty


def err(a, b):
    d = (a.double() - b.double()).abs()
    return d.max().item(), d.mean().item()
