"""Kernel-level parity of the teacher backward (-m gpu) in the layouts the networks run it: f16 tapes with their producers'
statistics replicas, strided gradient views inside wider buffers, the resampled residuals and added terms of the ResBlock
adjoints, FiLM gradients at a block's offset, split-K data gradients with a residual, the fused tail's head adjoint, the pose
MLP and the attention backward at its fragile softmaxes.  Shapes are those of UNetNet(false, 256, 64, {1,2,4,4,4}),
UNetNet(true, 512, 32, {1,2,4,8,8,8}) and the encoder-decoders (S = 128 / 192, pose pads 16 / 32).

Every result is compared elementwise with an fp64 reference and its worst-case bound (tests/teacher_backward_ref.py).  Guard
columns around strided operands are NaN for the elementwise kernels (they have no reason to read them) and finite +-1e4 for
conv operands (zero-padded weights make any legal read contribute exactly 0; a wrong stride does not)."""
import ctypes
import functools

import pytest
import torch

import gpu_util as G
import teacher_backward_ref as R
from tha4_b200._lib import _ptr

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
NAN = float('nan')


def _film1_layout(mc, mults):
    """The U-Net's FiLM table (UNetNet::load): each ResBlock's 2 x cout columns in load order.  Returns ({block name:
    column offset}, {block name: cout}, table width)."""
    ch = [mc * m for m in mults]
    L = len(mults)
    blocks = []
    for i in range(L):
        blocks.append(('down_blocks.%d.res_blocks.0' % i, ch[i]))
        if i < L - 1:
            blocks.append(('down_blocks.%d.downsample' % i, ch[i]))
    blocks += [('middle_blocks.%d' % j, ch[-1]) for j in (0, 2, 4, 6)]
    for bi in range(L):
        blocks += [('up_blocks.%d.resnet_blocks.%d' % (bi, r), ch[L - 1 - bi]) for r in (0, 1)]
        if bi < L - 1:
            blocks.append(('up_blocks.%d.upsample' % bi, ch[L - 1 - bi]))
    off, cout, o = {}, {}, 0
    for name, c in blocks:
        off[name], cout[name] = o, c
        o += 2 * c
    return off, cout, o


BODY_FILM1_OFF, BODY_COUT, BODY_FILM1 = _film1_layout(64, [1, 2, 4, 4, 4])
UPSCALER_FILM1 = _film1_layout(32, [1, 2, 4, 8, 8, 8])[2]
FILM_BLOCK = {64: 'up_blocks.4.resnet_blocks.1', 256: 'up_blocks.1.resnet_blocks.0'}   # body blocks whose norm1 the tests run


def _place(t, ld, c0, guard, dtype=torch.float32):
    """NCHW tensor -> NHWC device buffer [N, H, W, ld] holding it at channels c0.. (guards elsewhere); returns (buffer, the
    operand's view)."""
    N, C, H, W = t.shape
    buf = torch.empty(N, H, W, ld, dtype=dtype, device=DEV)
    if guard == 'sentinel':
        buf.copy_(torch.where(torch.arange(ld, device=DEV) % 2 == 0, 1e4, -1e4).to(dtype).expand(N, H, W, ld))
    else:
        buf.fill_(guard)
    buf[..., c0:c0 + C] = t.permute(0, 2, 3, 1).to(DEV, dtype)
    return buf, buf[..., c0:c0 + C]


def _nchw(v):
    return v.permute(0, 3, 1, 2).double().cpu()


def _check(name, out, ref, bound):
    out = out.double().cpu()
    assert torch.isfinite(out).all(), name
    ratio = ((out - ref).abs() / bound).max().item()
    print('\n%s: max |err| / bound %.3e (max |err| %.3e, max |ref| %.3e)' % (name, ratio, (out - ref).abs().max().item(),
                                                                          ref.abs().max().item()))
    assert ratio <= 1.0, (name, ratio)
    return ratio


def _guards_intact(name, buf, c0, C, fill):
    rest = torch.cat([buf[..., :c0], buf[..., c0 + C:]], -1)
    ok = torch.isnan(rest).all() if fill != fill else (rest == fill).all()
    assert ok, '%s: a guard column was written' % name


def _stats_dev(x, rep, seed):
    """x's per-(n, c) sums spread unevenly over `rep` replicas [rep][N][C][2], on the device."""
    return R.split_replicas(R.stats_of(x), rep, seed).contiguous().to(DEV)


# ------------------------------------------------------------------------------------------ GroupNorm backward
# (C, H, N, role): role = the call in res_bwd / attn_bwd (unet_backward.cu)
GN_CASES = [(32, 512, 1, 'conv0_same_add'), (64, 256, 3, 'norm1_film'), (96, 64, 3, 'skip'), (128, 64, 3, 'down'),
            (192, 32, 3, 'up'), (256, 16, 3, 'attn'), (384, 32, 1, 'skip'), (512, 16, 3, 'conv0_same_add'),
            (256, 32, 1, 'down'), (256, 32, 1, 'norm1_film')]


@pytest.mark.parametrize('C,H,N,role', GN_CASES)
@pytest.mark.parametrize('x_f16', [0, 1])
def test_group_norm_backward(C, H, N, role, x_f16):
    g = torch.Generator().manual_seed(C + H + N + x_f16 + len(role))
    x = torch.randn(N, C, H, H, generator=g) * 2 + 0.5
    if x_f16:
        x = x.half().float()
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.3
    act = 0 if role == 'attn' else 2
    film = role == 'norm1_film'
    film0 = torch.randn(2 * C, generator=g) * 0.3 if film else None
    film1_ld = BODY_FILM1
    off = BODY_FILM1_OFF[FILM_BLOCK[C]] if film else 0
    film1_full = torch.randn(N, film1_ld, generator=g) * 0.3 if film else None
    film1 = film1_full[:, off:off + 2 * C] if film else None
    dy_pool = role == 'down'
    hd = H // 2 if dy_pool else H
    dy = torch.randn(N, C, hd, hd, generator=g)
    res_mode = {'conv0_same_add': 1, 'skip': 1, 'attn': 1, 'up': 2, 'down': 3}.get(role, 0)
    res = None
    if res_mode:
        rh = {1: H, 2: 2 * H, 3: H // 2}[res_mode]
        res = torch.randn(N, C, rh, rh, generator=g)
    add = torch.randn(N, C, H, H, generator=g) if role in ('conv0_same_add', 'down') else None
    ref, dfilm_ref, bound, dfilm_bound = R.norm_backward_ref(x, 32, gamma, beta, dy, act, film0, film1, dy_pool, res, res_mode, add)

    c = G.ctx()
    xb, xv = _place(x, C + 8, 4, NAN, torch.float16 if x_f16 else torch.float32)
    dyb, dyv = _place(dy, C + 32, 0, NAN)                         # dcat[j + 1].slice(0, ch_h)
    rb = rv = None
    if role == 'skip':
        rb, rv = _place(res, C, 0, NAN)                           # dsk: a fresh tensor
    elif res is not None:
        rb, rv = _place(res, C + 48, 16, NAN)                     # a dhs-like slice at a channel offset
    ab, av = _place(add, C + 16, 8, NAN) if add is not None else (None, None)
    if film:
        assert BODY_COUT[FILM_BLOCK[C]] == C
    gd, bd = G.dev(gamma), G.dev(beta)
    f0d = G.dev(film0) if film else None
    f1d = G.dev(film1_full) if film else None
    worst = 0.0
    for rep in (1, 2, 16):
        st = _stats_dev(x, rep, seed=rep + C)
        dxb = torch.full((N, H, H, C + 12), NAN, device=DEV)
        dxv = dxb[..., 4:4 + C]
        dfb = torch.full((N, film1_ld), -7777.0, device=DEV) if film else None
        c._call('tha4_test_group_norm_backward_ex', _ptr(xv), x_f16, xb.shape[-1], N, C, H, H, 32, _ptr(st), rep, C,
                _ptr(gd), _ptr(bd), _ptr(f0d), _ptr(f1d), film1_ld, off, act, _ptr(dyv), dyb.shape[-1], int(dy_pool),
                _ptr(rv), rb.shape[-1] if rb is not None else 0, res_mode, _ptr(av), ab.shape[-1] if ab is not None else 0,
                _ptr(dxv), dxb.shape[-1], _ptr(dfb), film1_ld, c._stream())
        torch.cuda.synchronize()
        name = 'GN bwd C %d %d^2 N %d %s f16 %d rep %d' % (C, H, N, role, x_f16, rep)
        worst = max(worst, _check(name + ' d(x)', _nchw(dxv), ref, bound))
        _guards_intact(name, dxb, 4, C, NAN)
        if film:
            worst = max(worst, _check(name + ' d(film1)', dfb[:, off:off + 2 * C].cpu(), dfilm_ref, dfilm_bound))
            untouched = torch.cat([dfb[:, :off], dfb[:, off + 2 * C:]], 1)
            assert (untouched == -7777.0).all(), 'd(film) written outside the block columns'
    print('worst ratio %.3e' % worst)


# ------------------------------------------------------------------------------------------ InstanceNorm backward
# (C, H, N, act, dy width): the enc-dec norms at 128 / 192 inputs; the bottleneck entry's dy = dbin.slice(0, 512)
IN_CASES = [(64, 192, 1, 1, 64), (128, 64, 2, 1, 128), (256, 48, 2, 1, 256), (256, 32, 2, 0, 256), (512, 16, 2, 1, 528),
            (512, 24, 2, 1, 544), (512, 16, 3, 0, 528)]


@pytest.mark.parametrize('C,H,N,act,dy_w', IN_CASES)
@pytest.mark.parametrize('x_f16', [0, 1])
def test_norm_backward(C, H, N, act, dy_w, x_f16):
    g = torch.Generator().manual_seed(3 * C + H + act + x_f16)
    x = torch.randn(N, C, H, H, generator=g) * 2 + 0.5
    if x_f16:
        x = x.half().float()
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.3
    dy = torch.randn(N, C, H, H, generator=g)
    mask = None
    if act:
        mask, amb = R.relu_mask_and_ambiguous(x, gamma, beta)
        dy = torch.where(amb, torch.zeros_like(dy), dy)
    ref, _, bound, _ = R.norm_backward_ref(x, C, gamma, beta, dy, act, relu_mask=mask)
    c = G.ctx()
    xb, xv = _place(x, C + 8, 4, NAN, torch.float16 if x_f16 else torch.float32)
    dyb, dyv = _place(dy, dy_w + 4, 0, NAN)
    gd, bd = G.dev(gamma), G.dev(beta)
    rep = {64: 16, 128: 2, 256: 1, 512: 16}[C]
    st = _stats_dev(x, rep, seed=C)
    dxb = torch.full((N, H, H, C + 8), NAN, device=DEV)
    dxv = dxb[..., 4:4 + C]
    c._call('tha4_test_norm_backward_ex', _ptr(xv), x_f16, xb.shape[-1], N, C, H, H, _ptr(st), rep, C, _ptr(gd), _ptr(bd), act,
            _ptr(dyv), dyb.shape[-1], _ptr(dxv), dxb.shape[-1], c._stream())
    torch.cuda.synchronize()
    name = 'IN bwd C %d %d^2 N %d act %d f16 %d' % (C, H, N, act, x_f16)
    _check(name, _nchw(dxv), ref, bound)
    _guards_intact(name, dxb, 4, C, NAN)


# ------------------------------------------------------------------------------------------ conv data gradient
@functools.lru_cache(maxsize=8)
def _conv_case(kind, cin, cout, H, N, with_add, strict, seed):
    g = torch.Generator().manual_seed(seed)
    k = 1 if kind == 3 else 3
    w = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (cin * k * k)) ** 0.5
    dy = torch.randn(N, cout, H, H, generator=g)
    add = torch.randn(N, cin, H, H, generator=g) if with_add else None
    dx, bound = R.conv_dgrad_ref(0 if kind != 3 else 3, w, dy, (H, H), add, strict=bool(strict))
    return w, dy, add, dx, bound


def _run_dgrad(kind, w, dy, add, N, cin, cout, H, strict, workspace, dy_ld, dy_c0, add_ld, add_c0, heads=None, head_b=None):
    c = G.ctx()
    dyb, dyv = _place(dy, dy_ld, dy_c0, 'sentinel')
    ab, av = _place(add, add_ld, add_c0, 'sentinel') if add is not None else (None, None)
    cin_k = (cin + 3) // 4 * 4
    dxb = torch.full((N, H, H, cin_k + 8), -5555.0, device=DEV)
    dxv = dxb[..., 4:4 + cin_k]
    wd = G.dev(w.reshape(-1) if heads is None else w)
    hb = G.dev(head_b) if head_b is not None else None
    hc = (ctypes.c_int * len(heads))(*heads) if heads is not None else None
    plan = ctypes.c_int(-1)
    c._call('tha4_test_conv_backward_data_ex', kind, _ptr(wd), _ptr(hb), hc, len(heads) if heads else 0, _ptr(dyv), dy_ld,
            _ptr(av), add_ld, _ptr(dxv), dxb.shape[-1], N, cin, H, H, cout, strict, workspace, ctypes.byref(plan), c._stream())
    torch.cuda.synchronize()
    _guards_intact('dgrad kind %d' % kind, dxb, 4, cin_k, -5555.0)
    return _nchw(dxv)[:, :cin], plan.value


# (B, H): the ResnetBlock adjoint 512 -> 512 at the bottleneck maps.  Default mode on each split-K plan of the tensor-core
# kernel: 'cluster' (run_dgrad as the network calls it), 'workspace' (cluster split-K off), 'atomic' (cluster split-K off and
# no workspace: the partials accumulate with atomics into the output, the residual added by the first K slice only); strict
# mode runs the mma.sync kernel, whose split launches accumulate atomically.
SPLIT_PLAN = {'none': 0, 'cluster': 1, 'workspace': 2, 'atomic': 3}


@pytest.mark.parametrize('B,H', [(1, 16), (2, 24), (4, 16)])
@pytest.mark.parametrize('strict,plan', [(0, 'cluster'), (0, 'workspace'), (0, 'atomic'), (1, 'none')])
def test_resnet_block_adjoint_with_residual(B, H, strict, plan):
    w, dy, add, ref, bound = _conv_case(0, 512, 512, H, B, True, strict, 100 + H)
    c = G.ctx()
    if plan in ('workspace', 'atomic'):
        c.set_option('cluster_splitk', 0)
    try:
        out, ran = _run_dgrad(0, w, dy, add, B, 512, 512, H, strict, 0 if plan == 'atomic' else 1, 512, 0, 512, 0)
    finally:
        c.set_option('cluster_splitk', 1)
    assert ran == SPLIT_PLAN[plan], (plan, ran)
    _check('ResnetBlock dgrad B %d %d^2 strict %d %s' % (B, H, strict, plan), out, ref, bound)


@pytest.mark.parametrize('cin,S', [(4, 128), (8, 128), (4, 192)])
@pytest.mark.parametrize('strict', [0, 1])
def test_first_conv_adjoint_adds_image_term(cin, S, strict):
    w, dy, add, ref, bound = _conv_case(0, cin, 64, S, 2, True, strict, 200 + cin)
    out, _ = _run_dgrad(0, w, dy, add, 2, cin, 64, S, strict, 1, 64, 0, cin + 4, 4)
    _check('first conv dgrad 64 -> %d %d^2 strict %d' % (cin, S, strict), out, ref, bound)


# the U-Net's skip 1x1 (kind 3) and conv1 3x3 (kind 5) adjoints: dy = dcat slice, add = dhs-like slice
@pytest.mark.parametrize('kind,cin,cout,H', [(3, 512, 256, 16), (3, 192, 64, 64), (5, 256, 256, 16), (5, 64, 64, 64)])
@pytest.mark.parametrize('strict', [0, 1])
def test_unet_adjoints_on_strided_views(kind, cin, cout, H, strict):
    w, dy, add, ref, bound = _conv_case(kind, cin, cout, H, 2, True, strict, 300 + kind + cin)
    out, _ = _run_dgrad(kind, w, dy, add, 2, cin, cout, H, strict, 1, cout + 64, 0, cin + 96, 32)
    _check('U-Net dgrad kind %d %d -> %d %d^2 strict %d' % (kind, cout, cin, H, strict), out, ref, bound)


HEADS = {0: [7], 1: [1, 4, 1, 4], 2: [2, 1, 4, 1], 3: [2, 4, 1, 4, 1]}      # head convs in tail.cu order per tail kind


@pytest.mark.parametrize('tail_kind,C', [(0, 64), (0, 32), (1, 64), (2, 64), (3, 64)])
@pytest.mark.parametrize('strict', [0, 1])
def test_head_adjoint(tail_kind, C, strict):
    g = torch.Generator().manual_seed(400 + tail_kind + C)
    ws = [torch.randn(co, C, 3, 3, generator=g) * (2.0 / (C * 9)) ** 0.5 for co in HEADS[tail_kind]]
    bs = [torch.randn(co, generator=g) for co in HEADS[tail_kind]]
    wcat = torch.cat(ws, 0)
    CO, N, S = wcat.shape[0], 2, 32
    dh = torch.randn(N, CO, S, S, generator=g)
    ref, bound = R.conv_dgrad_ref(0, wcat, dh, (S, S), strict=bool(strict))
    dh16 = torch.cat([dh, torch.zeros(N, 16 - CO, S, S)], 1)       # channels CO..15 carry the +-1e4 sentinels below
    dhb, dhv = _place(dh16, 16, 0, 'sentinel')
    dhb[..., CO:] = torch.where(torch.arange(16 - CO, device=DEV) % 2 == 0, 1e4, -1e4)
    c = G.ctx()
    dxb = torch.full((N, S, S, C + 8), -5555.0, device=DEV)
    dxv = dxb[..., 4:4 + C]
    wd, bd = G.dev(torch.cat([w.reshape(-1) for w in ws])), G.dev(torch.cat(bs))
    hc = (ctypes.c_int * len(ws))(*HEADS[tail_kind])
    c._call('tha4_test_conv_backward_data_ex', 6, _ptr(wd), _ptr(bd), hc, len(ws), _ptr(dhv), 16, _ptr(None), 0, _ptr(dxv),
            dxb.shape[-1], N, C, S, S, 16, strict, 1, None, c._stream())
    torch.cuda.synchronize()
    _guards_intact('head adjoint', dxb, 4, C, -5555.0)
    _check('head adjoint tail %d C %d strict %d' % (tail_kind, C, strict), _nchw(dxv), ref, bound)


# ------------------------------------------------------------------------------------------ pose MLP
@pytest.mark.parametrize('R_total', [BODY_FILM1, UPSCALER_FILM1])
@pytest.mark.parametrize('N', [1, 5])
def test_linear_backward(R_total, N):
    """d(film1) -> FiLM projection (SiLU' at c2) -> cond_embed.2 (SiLU' at c1) -> cond_embed.0, stage by stage."""
    g = torch.Generator().manual_seed(R_total + N)
    c = G.ctx()
    for R_, K, silu in ((R_total, 256, True), (256, 256, True), (256, 6, False)):
        dy = torch.randn(N, R_, generator=g)
        W = torch.randn(R_, K, generator=g) * (1.0 / R_) ** 0.5
        pre = torch.randn(N, K, generator=g) * 2 if silu else None
        ref, bound = R.linear_backward_ref(dy, W, pre)
        dyb = torch.full((N, R_ + 4), NAN, device=DEV)
        dyb[:, :R_] = dy.to(DEV)
        preb = None
        if silu:
            preb = torch.full((N, K + 4), NAN, device=DEV)
            preb[:, :K] = pre.to(DEV)
        dxb = torch.full((N, K + 3), -5555.0, device=DEV)
        Wd = G.dev(W)
        c._call('tha4_test_linear_backward', _ptr(dyb), R_ + 4, N, R_, _ptr(Wd), K, _ptr(preb), K + 4, _ptr(dxb), K + 3, c._stream())
        torch.cuda.synchronize()
        _check('linear bwd %d -> %d N %d silu %d' % (R_, K, N, silu), dxb[:, :K].cpu(), ref, bound)
        assert (dxb[:, K:] == -5555.0).all()


# ------------------------------------------------------------------------------------------ attention backward
@pytest.mark.parametrize('N', [1, 3])
@pytest.mark.parametrize('mode', ['peaked', 'uniform'])
def test_attention_backward(N, mode):
    g = torch.Generator().manual_seed(500 + N + len(mode))
    C, heads = 256, 8
    qkv = torch.randn(N, 3 * C, 16, 16, generator=g)
    if mode == 'peaked':        # logits of tens: a near-one-hot softmax (m, 1/l and D_i carry the whole row)
        qkv[:, :2 * C] *= 3.0
    else:                       # every key equal: P exactly uniform
        qkv[:, C:2 * C] = qkv[:, C:2 * C, :1, :1].expand(N, C, 16, 16)
    dout = torch.randn(N, C, 16, 16, generator=g)
    ref, bound = R.attention_backward_ref(qkv, dout, heads)
    c = G.ctx()
    out = torch.empty(N, 3 * C, 16, 16, device=DEV)
    qd, dd = G.dev(qkv), G.dev(dout)
    c._call('tha4_test_attention_backward', _ptr(qd), _ptr(dd), N, C, heads, _ptr(out), c._stream())
    torch.cuda.synchronize()
    for k, name in enumerate(('dQ', 'dK', 'dV')):
        sl = slice(k * C, (k + 1) * C)
        _check('attention bwd N %d %s %s' % (N, mode, name), out[:, sl], ref[:, sl], bound[:, sl])
