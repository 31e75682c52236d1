"""CPU checks of the teacher backward references (tests/teacher_backward_ref.py): each reproduces an independent fp64
statement of its op, and its error bound holds for an fp32 evaluation of the same op while staying far below the size of the
gradient (so that a wrong index, stride or factor cannot hide under it)."""
import pytest
import torch
import torch.nn.functional as F

import teacher_backward_ref as R
from distill_kernel_ref import round_tf32


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _closed_form_norm(x, groups, gamma, beta, dy, act, film0, film1, dy_pool, res, res_mode, add, relu_mask, dtype):
    """dx = K dz - r1 - xhat r2 (+ residual, + add) and d(film1), evaluated in `dtype` (the kernels' formula)."""
    x = x.to(dtype)
    N, C, H, W = x.shape
    cpg = C // groups
    xs = x.view(N, groups, cpg * H * W)
    mean = xs.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((xs - mean) ** 2).mean(-1, keepdim=True) + R.EPS)
    xhat = ((xs - mean) * rstd).view(N, C, H, W)
    s0 = torch.ones(1, C, dtype=dtype) if film0 is None else 1 + film0[:C].to(dtype).view(1, C)
    b0 = torch.zeros(1, C, dtype=dtype) if film0 is None else film0[C:].to(dtype).view(1, C)
    s1 = torch.ones(N, C, dtype=dtype) if film1 is None else 1 + film1[:, :C].to(dtype)
    b1 = torch.zeros(N, C, dtype=dtype) if film1 is None else film1[:, C:].to(dtype)
    g, bt = gamma.to(dtype).view(1, C), beta.to(dtype).view(1, C)
    h2 = xhat * g.view(1, C, 1, 1) + bt.view(1, C, 1, 1)
    h = (h2 * s0.view(1, C, 1, 1) + b0.view(1, C, 1, 1)) * s1.view(N, C, 1, 1) + b1.view(N, C, 1, 1)
    dyu = dy.to(dtype)
    if dy_pool:
        dyu = 0.25 * F.interpolate(dyu, scale_factor=2, mode='nearest')
    if act == 2:
        sg = torch.sigmoid(h)
        dz = dyu * sg * (1 + h * (1 - sg))
    elif act == 1:
        dz = dyu * relu_mask.to(dtype)
    else:
        dz = dyu
    gm = g * s0 * s1
    S1, S2 = dz.sum((2, 3)), (dz * xhat).sum((2, 3))
    m1 = (gm * S1).view(N, groups, cpg).sum(-1).repeat_interleave(cpg, 1) / (cpg * H * W)
    m2 = (gm * S2).view(N, groups, cpg).sum(-1).repeat_interleave(cpg, 1) / (cpg * H * W)
    rs = rstd.view(N, groups).repeat_interleave(cpg, 1)
    dx = (rs * gm).view(N, C, 1, 1) * dz - (rs * m1).view(N, C, 1, 1) - xhat * (rs * m2).view(N, C, 1, 1)
    if res is not None:
        r = res.to(dtype)
        dx = dx + {1: r, 2: F.avg_pool2d(r, 2) * 4, 3: 0.25 * F.interpolate(r, scale_factor=2, mode='nearest')}[res_mode]
    if add is not None:
        dx = dx + add.to(dtype)
    dfilm = torch.cat([(g * S2 + bt * S1) * s0 + b0 * S1, S1], 1) if film1 is not None else None
    return dx, dfilm


@pytest.mark.parametrize('case', ['same_add', 'up2', 'down_pool', 'film', 'attn_none', 'instance_relu', 'instance_none'])
def test_norm_backward_ref(case):
    g = _gen(len(case))
    N, C, H = 2, 96, 8
    groups = C if case.startswith('instance') else 32
    x = (torch.randn(N, C, H, H, generator=g) * 2 + 0.5).half().float()       # f16-exact, as an f16 tape
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.3
    act = {'attn_none': 0, 'instance_none': 0, 'instance_relu': 1}.get(case, 2)
    film0 = torch.randn(2 * C, generator=g) * 0.3 if case == 'film' else None
    film1 = torch.randn(N, 2 * C, generator=g) * 0.3 if case == 'film' else None
    dy_pool = case == 'down_pool'
    dy = torch.randn(N, C, H // 2 if dy_pool else H, H // 2 if dy_pool else H, generator=g)
    res_mode = {'same_add': 1, 'up2': 2, 'down_pool': 3, 'attn_none': 1}.get(case, 0)
    res = None
    if res_mode:
        rh = {1: H, 2: 2 * H, 3: H // 2}[res_mode]
        res = torch.randn(N, C, rh, rh, generator=g)
    add = torch.randn(N, C, H, H, generator=g) if case in ('same_add', 'down_pool') else None
    mask = None
    if act == 1:
        mask, amb = R.relu_mask_and_ambiguous(x, gamma, beta)
        dy = torch.where(amb, torch.zeros_like(dy), dy)
    dx, dfilm, bdx, bdf = R.norm_backward_ref(x, groups, gamma, beta, dy, act, film0, film1, dy_pool, res, res_mode, add, mask)
    args = (x, groups, gamma, beta, dy, act, film0, film1, dy_pool, res, res_mode, add, mask)
    cf64, cf64_film = _closed_form_norm(*args, torch.float64)
    assert (dx - cf64).abs().max().item() <= 1e-10 * dx.abs().max().item()
    cf32, cf32_film = _closed_form_norm(*args, torch.float32)
    ratio = ((cf32.double() - dx).abs() / bdx).max().item()
    print('\n%s: fp32 closed form / bound %.3e, bound / max|dx| %.3e' % (case, ratio, (bdx.max() / dx.abs().max()).item()))
    assert ratio <= 1.0
    assert bdx.max().item() <= 1e-3 * dx.abs().max().item()
    if film1 is not None:
        assert (dfilm - cf64_film).abs().max().item() <= 1e-10 * dfilm.abs().max().item()
        assert ((cf32_film.double() - dfilm).abs() / bdf).max().item() <= 1.0
        assert bdf.max().item() <= 1e-3 * dfilm.abs().max().item()


def test_replicas_add_up():
    s = R.stats_of(torch.randn(3, 64, 8, 8, generator=_gen(1)))
    for rep in (1, 2, 16):
        r = R.split_replicas(s, rep, seed=rep)
        assert r.shape == (rep,) + s.shape
        assert (r.sum(0) - s).abs().max().item() <= 1e-12 * s.abs().max().item()
        if rep > 1:
            assert torch.count_nonzero(r[1]).item() == 0


def test_relu_mask_flags_only_near_zero():
    g = _gen(2)
    x = torch.randn(2, 16, 8, 8, generator=g)
    gamma, beta = torch.rand(16, generator=g) + 0.5, torch.randn(16, generator=g) * 0.3
    mask, amb = R.relu_mask_and_ambiguous(x, gamma, beta)
    z = F.instance_norm(x.double(), weight=gamma.double(), bias=beta.double(), eps=R.EPS)
    assert torch.equal(mask[~amb], (z > 0).double()[~amb])
    assert amb.sum().item() <= 2          # only elements within rounding of the kernel's zero


@pytest.mark.parametrize('kind,strict', [(0, 0), (0, 1), (3, 0), (3, 1)])
def test_conv_dgrad_ref(kind, strict):
    g = _gen(10 + kind + strict)
    N, cin, cout, H = 2, 24, 32, 6
    k = 3 if kind == 0 else 1
    w = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (cin * k * k)) ** 0.5
    dy = torch.randn(N, cout, H, H, generator=g)
    add = torch.randn(N, cin, H, H, generator=g)
    dx, bound = R.conv_dgrad_ref(kind, w, dy, (H, H), add, strict=bool(strict))
    wr = w.double() if strict else round_tf32(w).double()
    # an independent statement: the transposed conv
    ref = F.conv_transpose2d(dy.double(), wr, None, 1, k // 2) + add.double()
    assert (dx - ref).abs().max().item() <= 1e-12
    # fp32 with the activation operand truncated to TF32 (the worst a TF32 read can do) stays inside the bound
    dyt = dy.contiguous().view(torch.int32) & ~0x1FFF
    dyt = dyt.view(torch.float32)
    f32 = F.conv_transpose2d(dyt if not strict else dy, wr.float(), None, 1, k // 2) + add
    assert ((f32.double() - dx).abs() <= bound).all()
    assert bound.max().item() <= 1e-2 * dx.abs().max().item()


@pytest.mark.parametrize('silu', [False, True])
def test_linear_backward_ref(silu):
    g = _gen(20 + silu)
    N, R_, K = 3, 300, 70
    dy, W = torch.randn(N, R_, generator=g), torch.randn(R_, K, generator=g) * 0.05
    pre = torch.randn(N, K, generator=g) * 3 if silu else None
    ref, bound = R.linear_backward_ref(dy, W, pre)
    t = dy.double() @ W.double()
    expect = t * R.silu_grad64(pre) if silu else t
    assert (ref - expect).abs().max().item() <= 1e-12 * expect.abs().max().item()
    # the kernel's arithmetic: fp64 sum rounded once, times an fp32 SiLU'
    k32 = t.float()
    if silu:
        k32 = k32 * R.silu_grad64(pre).float()
    assert ((k32.double() - ref).abs() <= bound).all()
    assert ((t.float().double() - t).abs() <= R.ulp32(t) / 2).all()


@pytest.mark.parametrize('mode', ['moderate', 'peaked', 'uniform'])
def test_attention_backward_ref(mode):
    g = _gen(30 + len(mode))
    N, C, heads = 1, 64, 2
    qkv = torch.randn(N, 3 * C, 16, 16, generator=g)
    if mode == 'peaked':
        qkv[:, :2 * C] *= 4
    if mode == 'uniform':
        qkv[:, C:2 * C] = qkv[:, C:2 * C, :1, :1]
    dout = torch.randn(N, C, 16, 16, generator=g)
    ref, bound = R.attention_backward_ref(qkv, dout, heads)
    q32 = qkv.clone().requires_grad_()
    R.attention_ref(q32, heads).backward(dout)
    ratio = ((q32.grad.double() - ref).abs() / bound).max().item()
    print('\nattention %s: fp32 autograd / bound %.3e' % (mode, ratio))
    assert ratio <= 1.0
    assert bound.max().item() <= 1e-2 * ref.abs().max().item()
