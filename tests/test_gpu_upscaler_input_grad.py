"""The upscaler U-Net (Upscaler02) and the full poser (mode_07) under torch.autograd on the H100 (-m gpu): gradients w.r.t. the
rest image, the coarse posed image, the coarse grid change and the pose.

Kernel level: the prologue's adjoint (image warp, grid gradient, bilinear x2), the GroupNorm backward at the upscaler's 32 and
64 channels per full-resolution level, and the 32 -> 16 data gradient of the fused first conv against CPU autograd.  Module
level: the four input gradients against CPU autograd through the fp32 oracle (oracle/tha4_oracle.py) on the teacher_sds
weights, with the coarse inputs at 256 (the fused x2) and 512, and the invariants of the autograd path.  Poser level: mode_07's
d(pose) and d(image), its plain path and eyebrow cache, and a fit of all 45 pose parameters.  The bounds are those of the body
morpher's backward (test_gpu_body_morpher_input_grad.py)."""
import pytest
import torch
import torch.nn.functional as F

import gpu_util as G
from oracle import synth, tha4_oracle as O
from tha4_b200._lib import Tha4Error, _ptr
from tha4_b200.nn.upscaler.upscaler_02 import Upscaler02
from tha4_b200.poser.modes import mode_07

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
DEFAULT_REL, DEFAULT_COS = 0.2, 0.98
STRICT_REL, STRICT_COS = 1e-2, 0.9999
INPUTS = ('d(rest)', 'd(coarse_posed)', 'd(coarse_grid)', 'd(pose)')


def _rel(a, b):
    a, b = a.double().cpu().reshape(-1), b.double().cpu().reshape(-1)
    return ((a - b).norm() / b.norm()).item()


def _rel_cos(name, g, ref):
    g, ref = g.double().cpu().reshape(-1), ref.double().cpu().reshape(-1)
    rel = ((g - ref).norm() / ref.norm()).item()
    cos = F.cosine_similarity(g, ref, dim=0).item()
    print('\n%s: rel L2 %.3e cosine %.6f' % (name, rel, cos))
    return rel, cos


def _up512(t):
    return t if t.shape[-1] == 512 else F.interpolate(t, size=(512, 512), mode='bilinear', align_corners=False)


# ------------------------------------------------------------------------------------------ kernel level
def _warp(clib, grid_change, image):
    import ctypes
    n, _, S, _ = image.shape
    b = torch.empty(S)
    clib.tha4o_base_grid(S, ctypes.c_void_p(b.data_ptr()))
    base = torch.stack([b.view(1, 1, S).expand(n, S, S), b.view(1, S, 1).expand(n, S, S)], dim=-1)
    return F.grid_sample(image, base + grid_change.permute(0, 2, 3, 1), mode='bilinear', padding_mode='border', align_corners=False)


def _lerp_up(t):
    """interpolate(size=512, bilinear, align_corners=False) in the kernels' order of rounded operations (gridsample.cuh lerp2):
    the warp's grid gradient jumps where a sample crosses a pixel, so the reference must sample at the same coordinates."""
    Sh = t.shape[-1]
    if Sh == 512:
        return t
    f = ((torch.arange(512, dtype=torch.float32) + 0.5) * (Sh / 512.0) - 0.5).clamp(min=0.0)
    i0 = f.long()
    i1 = (i0 + 1).clamp(max=Sh - 1)
    l1 = f - i0.float()
    l0 = 1.0 - l1
    ly0, ly1, lx0, lx1 = l0.view(-1, 1), l1.view(-1, 1), l0.view(1, -1), l1.view(1, -1)
    r0, r1 = t[:, :, i0], t[:, :, i1]
    return ly0 * (lx0 * r0[..., i0] + lx1 * r0[..., i1]) + ly1 * (lx0 * r1[..., i0] + lx1 * r1[..., i1])


@pytest.mark.parametrize('grid', ['zero', 'half', 'border', 'mix'])
@pytest.mark.parametrize('size', [256, 512])
def test_upscaler_prologue_backward(oracle_clib, size, grid):
    g = torch.Generator().manual_seed(60 + size // 256 + 3 * len(grid))
    N = 2
    if grid == 'zero':
        gc = torch.zeros(N, 2, size, size)
    elif grid == 'half':       # source coordinates on exact half-integers of the 512x512 image (where the grid is not interpolated)
        gc = torch.randint(-3, 4, (N, 2, size, size), generator=g).float() / 512
    elif grid == 'border':     # one sign per sample and axis, |g| >= 3: every fine sample, interpolated or not, is clamped
        sign = torch.where(torch.rand(N, 2, 1, 1, generator=g) < 0.5, -1.0, 1.0)
        gc = sign * (3 + 2 * torch.rand(N, 2, size, size, generator=g))
    else:
        gc = (torch.rand(N, 2, size, size, generator=g) - 0.5) * 2.4
    rest = synth.synthetic_image(3, N) * 2 - 1
    posed = torch.randn(N, 4, size, size, generator=g)
    dx0 = torch.randn(N, 16, 512, 512, generator=g)
    if grid == 'border':
        dx0[:, 12:14] = 0          # no direct grid term: the grid gradient must then be exactly 0
    rr, pr, gr = rest.clone().requires_grad_(), posed.clone().requires_grad_(), gc.clone().requires_grad_()
    fine_grid = _lerp_up(gr)
    x0 = torch.cat([rr, _lerp_up(pr), _warp(oracle_clib, fine_grid, rr), fine_grid], dim=1)
    x0.backward(dx0[:, :14])
    c = G.ctx()
    d_rest = torch.empty(N, 4, 512, 512, device=DEV)
    d_posed = torch.empty(N, 4, size, size, device=DEV)
    d_grid = torch.empty(N, 2, size, size, device=DEV)
    rd, gd, dd = G.dev(rest), G.dev(gc), G.dev(dx0)
    c._call('tha4_test_upscaler_prologue_backward', _ptr(rd), _ptr(gd), size, N, _ptr(dd), _ptr(d_rest), _ptr(d_posed), _ptr(d_grid),
            c._stream())
    torch.cuda.synchronize()
    r_rest, r_posed = _rel(d_rest, rr.grad), _rel(d_posed, pr.grad)
    print('\nprologue backward %d grid %s: d(rest) %.3e d(posed) %.3e' % (size, grid, r_rest, r_posed))
    assert r_rest <= 1e-5 and r_posed <= 1e-5, (r_rest, r_posed)
    if grid == 'border':
        assert torch.count_nonzero(d_grid).item() == 0
    else:
        r_grid = _rel(d_grid, gr.grad)
        print('d(grid) %.3e' % r_grid)
        assert r_grid <= 1e-5, r_grid
    # each output alone is the same
    d_grid2 = torch.empty_like(d_grid)
    c._call('tha4_test_upscaler_prologue_backward', _ptr(rd), _ptr(gd), size, N, _ptr(dd), _ptr(None), _ptr(None), _ptr(d_grid2),
            c._stream())
    torch.cuda.synchronize()
    assert torch.equal(d_grid, d_grid2)


@pytest.mark.parametrize('C,H', [(32, 256), (64, 128)])
def test_group_norm_backward_full_resolution(C, H):
    g = torch.Generator().manual_seed(C + H)
    N = 2
    x = torch.randn(N, C, H, H, generator=g) * 2 + 0.5
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.3
    f0, f1 = torch.randn(2 * C, generator=g) * 0.3, torch.randn(N, 2 * C, generator=g) * 0.3
    dy = torch.randn(N, C, H, H, generator=g)
    xr, f1r = x.clone().requires_grad_(), f1.clone().requires_grad_()
    y = F.group_norm(xr, 32, gamma, beta, eps=1e-5)
    y = y * (1 + f0[:C].view(1, C, 1, 1)) + f0[C:].view(1, C, 1, 1)
    y = y * (1 + f1r[:, :C].view(N, C, 1, 1)) + f1r[:, C:].view(N, C, 1, 1)
    F.silu(y).backward(dy)
    c = G.ctx()
    dx = torch.empty(N, C, H, H, device=DEV)
    dfilm = torch.empty(N, 2 * C, device=DEV)
    t = [G.dev(v) for v in (x, gamma, beta, f0, f1, dy)]
    c._call('tha4_test_group_norm_backward', _ptr(t[0]), N, C, H, H, 32, _ptr(t[1]), _ptr(t[2]), _ptr(t[3]), _ptr(t[4]), 2,
            _ptr(t[5]), _ptr(dx), _ptr(dfilm), c._stream())
    torch.cuda.synchronize()
    rx, rf = _rel(dx, xr.grad), _rel(dfilm, f1r.grad)
    print('\ngroup norm backward C %d H %d: d(x) %.3e d(film) %.3e' % (C, H, rx, rf))
    assert rx <= 1e-5 and rf <= 1e-5, (rx, rf)


@pytest.mark.parametrize('strict', [1, 0])
def test_first_conv_backward_data(strict):
    """The upscaler's fused first conv: 14 input channels packed as 16, its adjoint from the packed weights (kind 5)."""
    g = torch.Generator().manual_seed(77)
    N, cin, cout, h = 2, 14, 32, 128
    w = torch.randn(cout, cin, 3, 3, generator=g) * (2.0 / (cin * 9)) ** 0.5
    dy = torch.randn(N, cout, h, h, generator=g) * 1e-3
    x = torch.zeros(N, cin, h, h, requires_grad=True)
    F.conv2d(x, w, None, 1, 1).backward(dy)
    c = G.ctx()
    out = torch.empty(N, cin, h, h, device=DEV)
    dyd, wd = G.dev(dy), G.dev(w)
    c._call('tha4_test_conv_backward_data', 5, _ptr(dyd), _ptr(wd), _ptr(out), N, cin, h, h, cout, strict, c._stream())
    torch.cuda.synchronize()
    rel = _rel(out, x.grad)
    print('\nfirst conv dgrad %d->%d strict %d: rel L2 %.3e' % (cout, cin, strict, rel))
    assert rel <= (1e-5 if strict else 3e-3), rel


# ------------------------------------------------------------------------------------------ module level
def _load(sd):
    m = Upscaler02()
    m.load_state_dict(sd)
    return m.to(DEV)


def _inputs(B, size, seed=0):
    """rest image, coarse posed image and grid change at `size`, the six body parameters."""
    g = torch.Generator().manual_seed(seed)
    rest = synth.synthetic_image(seed, B)
    posed = F.interpolate(synth.synthetic_image(seed + 1, B), size=(size, size), mode='bilinear', align_corners=False)
    grid = torch.randn(B, 2, size, size, generator=g) * 0.02
    return [rest, posed.contiguous(), grid, synth.random_poses(B, seed=seed + 3)[:, 39:45].contiguous()]


def _ups(B, seed):
    """Upstream gradients on merged / alpha / grid_change / direct (none on warped)."""
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(B, c, s, s, generator=g) * 1e-3 if k != 2 else None
            for k, (c, s) in enumerate([(4, 512), (1, 512), (4, 512), (2, 512), (4, 512)])]


def _backward(outs, ups):
    pairs = [(o, u) for o, u in zip(outs, ups) if u is not None]
    torch.autograd.backward([o for o, _ in pairs], [u.to(o.device) for o, u in pairs])


def _gpu_grads(m, inputs, ups, want=(0, 1, 2, 3)):
    ts = [t.to(DEV).clone().requires_grad_(k in want) for k, t in enumerate(inputs)]
    outs = m(*ts)
    _backward(outs, ups)
    return [t.grad for t in ts], outs


def _cpu_grads(sd, inputs, ups):
    ts = [t.clone().requires_grad_() for t in inputs]
    _backward(O.upscaler_02(sd, ts[0], _up512(ts[1]), _up512(ts[2]), ts[3]), ups)
    return [t.grad for t in ts]


@pytest.fixture(scope='module', params=[256, 512])
def cpu_ref(request, teacher_sds):
    """CPU autograd through the fp32 oracle at B = 1, shared by both precision modes."""
    inputs = _inputs(1, request.param)
    ups = _ups(1, 11)
    return inputs, ups, _cpu_grads(teacher_sds['upscaler'], inputs, ups)


@pytest.mark.parametrize('strict', [0, 1])
def test_module_input_grads(teacher_sds, cpu_ref, strict):
    inputs, ups, cpu = cpu_ref
    size = inputs[1].shape[-1]
    m = _load(teacher_sds['upscaler'])
    m.context().set_option('strict', strict)
    try:
        with torch.no_grad():
            ref_out = m(*[t.to(DEV) for t in inputs])
        grads, outs = _gpu_grads(m, inputs, ups)
        for a, b in zip(outs, ref_out):
            # strict mode's mma.sync convs split K with float atomics: its forward is not bit-reproducible run to run
            assert a.grad_fn is not None and (torch.equal(a, b) if not strict else _rel(a, b) <= 1e-5)
        assert all(p.grad is None for p in m.parameters())
        for k, (gg, rr) in enumerate(zip(grads, cpu)):
            rel, cos = _rel_cos('Upscaler02 coarse %d strict=%d %s' % (size, strict, INPUTS[k]), gg, rr)
            if strict:
                assert rel <= STRICT_REL and cos >= STRICT_COS, (k, rel, cos)
            else:
                assert rel <= DEFAULT_REL and cos >= DEFAULT_COS, (k, rel, cos)
        # one gradient alone equals the same gradient requested with the others
        for k in range(4):
            alone, _ = _gpu_grads(m, inputs, ups, want=(k,))
            r = _rel(alone[k], grads[k])
            print('strict=%d %s alone vs all: rel %.3e' % (strict, INPUTS[k], r))
            assert r <= (1e-2 if strict else 1e-6), (k, r)       # strict: each call recomputes a non-reproducible forward
        # scaled upstream gradients scale the result exactly: no f16 staging of gradients
        for sc in (2.0 ** -24, 2.0 ** 24):
            scaled, _ = _gpu_grads(m, inputs, [u * sc if u is not None else None for u in ups])
            for a, b in zip(scaled, grads):
                r = _rel(a / sc, b)
                print('scale %g: rel %.3e' % (sc, r))
                assert r <= (1e-2 if strict else 1e-5), (sc, r)
    finally:
        m.context().set_option('strict', 0)


def test_batching_matches_single_samples(teacher_sds):
    m = _load(teacher_sds['upscaler'])
    B = 3
    inputs = _inputs(B, 256, seed=4)
    ups = _ups(B, 5)
    m.context().set_option('strict', 1)
    m.context().set_option('microbatch', 2)
    try:
        batched, _ = _gpu_grads(m, inputs, ups)
        m.context().set_option('microbatch', 32)
        alone = [_gpu_grads(m, [t[n:n + 1] for t in inputs], [u[n:n + 1] if u is not None else None for u in ups])[0]
                 for n in range(B)]
    finally:
        m.context().set_option('microbatch', 32)
        m.context().set_option('strict', 0)
    for n in range(B):
        for k, (a, b) in enumerate(zip(alone[n], batched)):
            r = _rel(a[0], b[n])
            print('batching sample %d %s: rel %.3e' % (n, INPUTS[k], r))
            assert r <= 1e-2, (n, k, r)


def test_double_backward_raises(teacher_sds):
    m = _load(teacher_sds['upscaler'])
    inputs = _inputs(1, 256)
    p = inputs[3].to(DEV).clone().requires_grad_()
    outs = m(*[t.to(DEV) for t in inputs[:3]], p)
    with pytest.raises(Tha4Error):
        torch.autograd.grad(outs[0].sum(), p, create_graph=True)


def test_two_upscalers_on_one_context(teacher_sds):
    sd = teacher_sds['upscaler']
    sd_b = {k: (v * 0.9 if k.endswith('weight') else v) for k, v in sd.items()}
    a = _load(sd)
    b = _load(sd_b)
    b.attach_context(a.context())
    inputs = _inputs(1, 256, seed=2)
    ups = _ups(1, 9)
    res = {}
    for m, name in ((a, 'a'), (b, 'b'), (a, 'a2')):
        res[name], _ = _gpu_grads(m, inputs, ups, want=(3,))
    assert _rel(res['a'][3], res['a2'][3]) <= 1e-6
    assert _rel(res['a'][3], res['b'][3]) > 1e-3
    rel, cos = _rel_cos('second module d(pose)', res['b'][3], _cpu_grads(sd_b, inputs, ups)[3])
    assert rel <= DEFAULT_REL and cos >= DEFAULT_COS


# ------------------------------------------------------------------------------------------ poser level
NETS = ('eyebrow_decomposer', 'eyebrow_morphing_combiner', 'face_morpher', 'body_morpher', 'upscaler')


def _poser(teacher_sds):
    return mode_07.create_poser(DEV, state_dicts={k: teacher_sds[k] for k in NETS})


def _poser_ups():
    """Upstream gradients on the upscaler's merged output (0) and the face morpher's output 0 (11)."""
    ups = [None] * 33
    g = torch.Generator().manual_seed(3)
    ups[0] = torch.randn(1, 4, 512, 512, generator=g) * 1e-3
    ups[11] = torch.randn(1, 4, 192, 192, generator=g) * 1e-3
    return ups


def test_mode_07_pose_and_image_grads(teacher_sds):
    poser = _poser(teacher_sds)
    image, pose = synth.synthetic_image(2, 1), synth.random_poses(1, seed=8)
    ups = _poser_ups()
    im, po = image.to(DEV).clone().requires_grad_(), pose.to(DEV).clone().requires_grad_()
    _backward(poser.get_posing_outputs(im, po), ups)
    imr, por = image.clone().requires_grad_(), pose.clone().requires_grad_()
    _backward(O.mode_07_outputs({k: teacher_sds[k] for k in NETS}, imr, por), ups)
    for name, gg, rr in (('mode_07 d(pose[:45])', po.grad, por.grad), ('mode_07 d(image)', im.grad, imr.grad)):
        rel, cos = _rel_cos(name, gg, rr)
        assert rel <= DEFAULT_REL and cos >= DEFAULT_COS, (name, rel, cos)


def test_mode_07_plain_path_and_cache_unchanged(teacher_sds):
    poser = _poser(teacher_sds)
    image, pose = synth.synthetic_image(2, 1).to(DEV), synth.random_poses(1, seed=8).to(DEV)
    a = poser.get_posing_outputs(image, pose)
    b = poser.get_posing_outputs(image, pose)
    assert all(x is y for x, y in zip(a[27:], b[27:]))          # eyebrow cache hit: the cached tensor objects
    with torch.no_grad():
        c = poser.get_posing_outputs(image, pose.clone().requires_grad_())
    assert all(torch.equal(x, y) for x, y in zip(a, c)) and all(x is y for x, y in zip(a[27:], c[27:]))
    d = poser.get_posing_outputs(image, pose.clone().requires_grad_())       # pose grad: the cached decomposer outputs are constants
    assert all(x is y for x, y in zip(a[27:], d[27:]))
    assert all(x.grad_fn is not None for x in d[:27])
    assert all(torch.equal(x, y) for x, y in zip(a, d))                   # the composed modules compute the single call's values
    e = poser.get_posing_outputs(image.clone().requires_grad_(), pose)       # image grad: the decomposer runs, same values
    assert all(torch.equal(x, y) for x, y in zip(a, e))


def test_mode_07_pose_fit(teacher_sds):
    """30 Adam steps on all 45 pose parameters towards a frame rendered at another pose."""
    poser = _poser(teacher_sds)
    image = synth.synthetic_image(2, 1).to(DEV)
    target_pose = synth.random_poses(1, seed=21).to(DEV)
    with torch.no_grad():
        target = poser.get_posing_outputs(image, target_pose)[0].clone()
    p45 = torch.zeros(1, 45, device=DEV, requires_grad=True)
    opt = torch.optim.Adam([p45], lr=5e-2)
    losses = []
    for _ in range(30):
        loss = (poser.get_posing_outputs(image, p45)[0] - target).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    print('\nmode_07 pose fit: L1 %.4e -> %.4e' % (losses[0], losses[-1]))
    assert losses[-1] <= 0.5 * losses[0], losses
