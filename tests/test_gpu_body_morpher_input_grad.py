"""The body morpher U-Net (Morpher00) under torch.autograd on the H100 (-m gpu): gradients w.r.t. image and pose.

Kernel level: the GroupNorm(+FiLM)(+SiLU) backward, the attention backward, the U-Net tail backward and the 1x1 / up-sampling
conv data gradients against CPU autograd.  Module level: d(image) and d(pose) against CPU autograd through the fp32 oracle
(oracle/tha4_oracle.py) on the teacher_sds weights, the invariants of the autograd path, and a body-pose fit.  The module
bounds are those of the face teachers' backward (DESIGN.md section 4): the gradient is that of the forward the context
computes, and the default mode's forward runs on f16 / TF32 operands."""
import math

import pytest
import torch
import torch.nn.functional as F

import gpu_util as G
from oracle import synth, tha4_oracle as O
from tha4_b200._lib import Tha4Error, _ptr, _ptr_array
from tha4_b200.nn.morpher.morpher_00 import Morpher00

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
DEFAULT_REL, DEFAULT_COS = 0.2, 0.98
STRICT_REL, STRICT_COS = 1e-2, 0.9999


def _rel(a, b):
    a, b = a.double().cpu().reshape(-1), b.double().cpu().reshape(-1)
    return ((a - b).norm() / b.norm()).item()


def _rel_cos(name, g, ref):
    g, ref = g.double().cpu().reshape(-1), ref.double().cpu().reshape(-1)
    rel = ((g - ref).norm() / ref.norm()).item()
    cos = F.cosine_similarity(g, ref, dim=0).item()
    print('\n%s: rel L2 %.3e cosine %.6f' % (name, rel, cos))
    return rel, cos


# ------------------------------------------------------------------------------------------ kernel level
@pytest.mark.parametrize('film', [False, True])
@pytest.mark.parametrize('act', [0, 2])
def test_group_norm_backward(film, act):
    g = torch.Generator().manual_seed(3 + 2 * act + film)
    N, C, H = 2, 128, 16
    x = torch.randn(N, C, H, H, generator=g) * 2 + 0.5
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.3
    f0 = torch.randn(2 * C, generator=g) * 0.3 if film else None
    f1 = torch.randn(N, 2 * C, generator=g) * 0.3 if film else None
    dy = torch.randn(N, C, H, H, generator=g)
    xr = x.clone().requires_grad_()
    f1r = f1.clone().requires_grad_() if film else None
    y = F.group_norm(xr, 32, gamma, beta, eps=1e-5)
    if film:
        y = y * (1 + f0[:C].view(1, C, 1, 1)) + f0[C:].view(1, C, 1, 1)
        y = y * (1 + f1r[:, :C].view(N, C, 1, 1)) + f1r[:, C:].view(N, C, 1, 1)
    (F.silu(y) if act else y).backward(dy)
    c = G.ctx()
    dx = torch.empty(N, C, H, H, device=DEV)
    dfilm = torch.empty(N, 2 * C, device=DEV) if film else None
    t = [G.dev(v) if v is not None else None for v in (x, gamma, beta, f0, f1, dy)]
    c._call('tha4_test_group_norm_backward', _ptr(t[0]), N, C, H, H, 32, _ptr(t[1]), _ptr(t[2]), _ptr(t[3]), _ptr(t[4]), act,
            _ptr(t[5]), _ptr(dx), _ptr(dfilm), c._stream())
    torch.cuda.synchronize()
    rel = _rel(dx, xr.grad)
    print('\ngroup norm backward film %d act %d: d(x) rel L2 %.3e' % (film, act, rel))
    assert rel <= 1e-5, rel
    if film:
        rf = _rel(dfilm, f1r.grad)
        print('d(film) rel L2 %.3e' % rf)
        assert rf <= 1e-5, rf


def _attention_ref(qkv, heads):
    """qkv_attention, 'new order' (oracle/tha4_oracle.py _attention_block)."""
    b, c3, hh, ww = qkv.shape
    c, L = c3 // 3, hh * ww
    ch = c // heads
    q, k, v = qkv.reshape(b, c3, L).chunk(3, dim=1)
    scale = 1.0 / math.sqrt(math.sqrt(ch))
    w = torch.einsum('bct,bcs->bts', (q * scale).reshape(b * heads, ch, L), (k * scale).reshape(b * heads, ch, L))
    w = torch.softmax(w, dim=-1)
    return torch.einsum('bts,bcs->bct', w, v.reshape(b * heads, ch, L)).reshape(b, c, hh, ww)


def test_attention_backward():
    g = torch.Generator().manual_seed(5)
    N, C, heads = 2, 256, 8
    qkv = torch.randn(N, 3 * C, 16, 16, generator=g) * 1.5
    dout = torch.randn(N, C, 16, 16, generator=g)
    qr = qkv.clone().requires_grad_()
    _attention_ref(qr, heads).backward(dout)
    c = G.ctx()
    out = torch.empty(N, 3 * C, 16, 16, device=DEV)
    qd, dd = G.dev(qkv), G.dev(dout)
    c._call('tha4_test_attention_backward', _ptr(qd), _ptr(dd), N, C, heads, _ptr(out), c._stream())
    torch.cuda.synchronize()
    for k, name in enumerate(('dQ', 'dK', 'dV')):
        rel = _rel(out[:, k * C:(k + 1) * C], qr.grad[:, k * C:(k + 1) * C])
        print('\nattention backward %s: rel L2 %.3e' % (name, rel))
        assert rel <= 1e-5, (name, rel)


def _warp(clib, grid_change, image):
    import ctypes
    n, _, S, _ = image.shape
    b = torch.empty(S)
    clib.tha4o_base_grid(S, ctypes.c_void_p(b.data_ptr()))
    base = torch.stack([b.view(1, 1, S).expand(n, S, S), b.view(1, S, 1).expand(n, S, S)], dim=-1)
    return F.grid_sample(image, base + grid_change.permute(0, 2, 3, 1), mode='bilinear', padding_mode='border', align_corners=False)


@pytest.mark.parametrize('grid', ['zero', 'half', 'border', 'mix'])
def test_unet_tail_backward(oracle_clib, grid):
    g = torch.Generator().manual_seed(40 + len(grid))
    N, S = 2, 32
    h = torch.randn(N, 7, S, S, generator=g)
    if grid == 'zero':
        h[:, 4:6] = 0
    elif grid == 'half':       # source coordinates on exact half-integers
        h[:, 4:6] = torch.randint(-3, 4, (N, 2, S, S), generator=g).float() / S
    elif grid == 'border':     # every sample clamped to the border
        h[:, 4:6] = torch.where(torch.rand(N, 2, S, S, generator=g) < 0.5, -3.0, 3.0)
    else:
        h[:, 4:6] = (torch.rand(N, 2, S, S, generator=g) - 0.5) * 2.4
    image = synth.synthetic_image(2, N)[:, :, :S, :S].contiguous() * 2 - 1
    hr, ir = h.clone().requires_grad_(), image.clone().requires_grad_()
    direct, gc, alpha = hr[:, 0:4], hr[:, 4:6], torch.sigmoid(hr[:, 6:7])
    warped = _warp(oracle_clib, gc, ir)
    outs = [O.apply_color_change(alpha, direct, warped), alpha, warped, gc, direct]
    # the grid_change output gets no upstream gradient on the border grid: there the grid gradient must then be exactly 0
    ups = [torch.randn(o.shape, generator=g) if not (grid == 'border' and k == 3) else None for k, o in enumerate(outs)]
    torch.autograd.backward([o for o, u in zip(outs, ups) if u is not None], [u for u in ups if u is not None])
    c = G.ctx()
    outs_d = [G.dev(o.detach().contiguous()) for o in outs]
    ups_d = [G.dev(u) if u is not None else None for u in ups]
    d_head = torch.empty(N, 12, S, S, device=DEV)
    d0 = torch.empty(N, 4, S, S, device=DEV)
    i0d = G.dev(image)
    c._call('tha4_test_tail_backward', 0, _ptr_array(outs_d), N, S, _ptr(i0d), _ptr(None), _ptr_array(ups_d), _ptr(d_head), _ptr(d0),
            _ptr(None), c._stream())
    torch.cuda.synchronize()
    rh, ri = _rel(d_head[:, :7], hr.grad), _rel(d0, ir.grad)
    print('\nU-Net tail backward grid %s: d(head) %.3e d(image) %.3e' % (grid, rh, ri))
    assert rh <= 1e-5 and ri <= 1e-5, (rh, ri)
    if grid == 'border':
        assert torch.count_nonzero(d_head[:, 4:6]).item() == 0


@pytest.mark.parametrize('kind,cin,cout,h', [(3, 256, 768, 16), (3, 512, 256, 16), (3, 128, 64, 32),
                                             (4, 256, 256, 16), (4, 128, 128, 32), (4, 256, 128, 32)])
@pytest.mark.parametrize('strict', [1, 0])
def test_unet_conv_backward_data(kind, cin, cout, h, strict):
    g = torch.Generator().manual_seed(kind * 1000 + cin + cout)
    N = 2
    k = 1 if kind == 3 else 3
    w = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (cin * k * k)) ** 0.5
    if kind == 3:
        ho, fwd = h, lambda t: F.conv2d(t, w)
    else:
        ho, fwd = 2 * h, lambda t: F.conv2d(F.interpolate(t, scale_factor=2, mode='nearest'), w, None, 1, 1)
    dy = torch.randn(N, cout, ho, ho, generator=g) * 1e-3
    x = torch.zeros(N, cin, h, h, requires_grad=True)
    fwd(x).backward(dy)
    c = G.ctx()
    out = torch.empty(N, cin, h, h, device=DEV)
    dyd, wd = G.dev(dy), G.dev(w)
    c._call('tha4_test_conv_backward_data', kind, _ptr(dyd), _ptr(wd), _ptr(out), N, cin, h, h, cout, strict, c._stream())
    torch.cuda.synchronize()
    rel = _rel(out, x.grad)
    print('\nU-Net conv dgrad kind %d %d->%d strict %d: rel L2 %.3e' % (kind, cout, cin, strict, rel))
    assert rel <= (1e-5 if strict else 3e-3), rel


# ------------------------------------------------------------------------------------------ module level
def _load(sd):
    m = Morpher00()
    m.load_state_dict(sd)
    return m.to(DEV)


def _inputs(B, seed=0):
    img = F.interpolate(synth.synthetic_image(seed, B), size=(256, 256), mode='bilinear', align_corners=False).contiguous()
    return img, synth.random_poses(B, seed=seed + 3)[:, 39:45].contiguous()


def _ups(B, seed):
    """Upstream gradients on merged / alpha / grid_change / direct (none on warped)."""
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(B, c, s, s, generator=g) * 1e-3 if k != 2 else None
            for k, (c, s) in enumerate([(4, 256), (1, 256), (4, 256), (2, 256), (4, 256)])]


def _backward(outs, ups):
    pairs = [(o, u) for o, u in zip(outs, ups) if u is not None]
    torch.autograd.backward([o for o, _ in pairs], [u.to(o.device) for o, u in pairs])


def _gpu_grads(m, img, pose, ups, want=(0, 1)):
    i = img.to(DEV).clone().requires_grad_(0 in want)
    p = pose.to(DEV).clone().requires_grad_(1 in want)
    outs = m(i, p)
    _backward(outs, ups)
    return [i.grad, p.grad], outs


@pytest.fixture(scope='module')
def cpu_ref(teacher_sds):
    """CPU autograd through the fp32 oracle at B = 2 (about 20 s on the CPU, shared by both precision modes)."""
    img, pose = _inputs(2)
    ups = _ups(2, 11)
    i, p = img.clone().requires_grad_(), pose.clone().requires_grad_()
    _backward(O.morpher_00(teacher_sds['body_morpher'], i, p), ups)
    return img, pose, ups, [i.grad, p.grad]


@pytest.mark.parametrize('strict', [0, 1])
def test_module_input_grads(teacher_sds, cpu_ref, strict):
    img, pose, ups, cpu = cpu_ref
    m = _load(teacher_sds['body_morpher'])
    m.context().set_option('strict', strict)
    try:
        with torch.no_grad():
            ref_out = m(img.to(DEV), pose.to(DEV))
        grads, outs = _gpu_grads(m, img, pose, ups)
        for a, b in zip(outs, ref_out):
            # strict mode's mma.sync convs split K with float atomics: its forward is not bit-reproducible run to run
            assert a.grad_fn is not None and (torch.equal(a, b) if not strict else _rel(a, b) <= 1e-5)
        assert all(p.grad is None for p in m.parameters())
        for k, (gg, rr) in enumerate(zip(grads, cpu)):
            rel, cos = _rel_cos('Morpher00 strict=%d %s' % (strict, ('d(image)', 'd(pose)')[k]), gg, rr)
            if strict:
                assert rel <= STRICT_REL and cos >= STRICT_COS, (k, rel, cos)
            else:
                assert rel <= DEFAULT_REL and cos >= DEFAULT_COS, (k, rel, cos)
        # one gradient alone equals the same gradient requested with the other
        for k in range(2):
            alone, _ = _gpu_grads(m, img, pose, ups, want=(k,))
            r = _rel(alone[k], grads[k])
            print('strict=%d input %d alone vs both: rel %.3e' % (strict, k, r))
            assert r <= (1e-2 if strict else 1e-6), (k, r)       # strict: each call recomputes a non-reproducible forward
        # scaled upstream gradients scale the result exactly: no f16 staging of gradients
        for sc in (2.0 ** -24, 2.0 ** 24):
            scaled, _ = _gpu_grads(m, img, pose, [u * sc if u is not None else None for u in ups])
            for a, b in zip(scaled, grads):
                r = _rel(a / sc, b)
                print('scale %g: rel %.3e' % (sc, r))
                assert r <= (1e-2 if strict else 1e-5), (sc, r)
    finally:
        m.context().set_option('strict', 0)


def test_batching_matches_single_samples(teacher_sds):
    m = _load(teacher_sds['body_morpher'])
    B = 5
    img, pose = _inputs(B, seed=4)
    ups = _ups(B, 5)
    m.context().set_option('strict', 1)
    m.context().set_option('microbatch', 2)
    try:
        batched, _ = _gpu_grads(m, img, pose, ups)
        m.context().set_option('microbatch', 32)
        alone = [_gpu_grads(m, img[n:n + 1], pose[n:n + 1], [u[n:n + 1] if u is not None else None for u in ups])[0] for n in range(B)]
    finally:
        m.context().set_option('microbatch', 32)
        m.context().set_option('strict', 0)
    for n in range(B):
        for k, (a, b) in enumerate(zip(alone[n], batched)):
            r = _rel(a[0], b[n])
            print('batching sample %d input %d: rel %.3e' % (n, k, r))
            assert r <= 1e-2, (n, k, r)


def test_double_backward_raises(teacher_sds):
    m = _load(teacher_sds['body_morpher'])
    img, pose = _inputs(1)
    p = pose.to(DEV).clone().requires_grad_()
    outs = m(img.to(DEV), p)
    with pytest.raises(Tha4Error):
        torch.autograd.grad(outs[0].sum(), p, create_graph=True)


def test_two_morphers_on_one_context(teacher_sds):
    sd = teacher_sds['body_morpher']
    sd_b = {k: (v * 0.9 if k.endswith('weight') else v) for k, v in sd.items()}
    a = _load(sd)
    b = _load(sd_b)
    b.attach_context(a.context())
    img, pose = _inputs(1, seed=2)
    ups = _ups(1, 9)
    res = {}
    for m, name in ((a, 'a'), (b, 'b'), (a, 'a2')):
        res[name], _ = _gpu_grads(m, img, pose, ups)
    assert _rel(res['a'][1], res['a2'][1]) <= 1e-6
    assert _rel(res['a'][1], res['b'][1]) > 1e-3
    i, p = img.clone().requires_grad_(), pose.clone().requires_grad_()
    _backward(O.morpher_00(sd_b, i, p), ups)
    rel, cos = _rel_cos('second module d(pose)', res['b'][1], p.grad)
    assert rel <= DEFAULT_REL and cos >= DEFAULT_COS


def test_body_pose_fit(teacher_sds):
    """30 Adam steps on the six body parameters (mode_07's pose[:, 39:45]) towards a frame rendered at another pose."""
    m = _load(teacher_sds['body_morpher'])
    img, _ = _inputs(1, seed=6)
    img = img.to(DEV)
    target_pose = synth.random_poses(1, seed=23)[:, 39:45].to(DEV)
    with torch.no_grad():
        target = m(img, target_pose)[0].clone()
    p6 = torch.zeros(1, 6, device=DEV, requires_grad=True)
    opt = torch.optim.Adam([p6], lr=5e-2)
    losses = []
    for _ in range(30):
        loss = (m(img, p6)[0] - target).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    print('\nbody pose fit: L1 %.4e -> %.4e, pose error %.3e -> %.3e' % (losses[0], losses[-1], target_pose.abs().mean().item(),
                                                                         (p6 - target_pose).abs().mean().item()))
    assert losses[-1] <= 0.25 * losses[0], losses       # measured on an H100: 4.1e-3 -> 3.9e-4
