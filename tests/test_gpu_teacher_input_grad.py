"""The encoder-decoder teacher networks under torch.autograd on the H100 (-m gpu): gradients w.r.t. image, layers and pose.

Kernel level: the conv data gradients, the InstanceNorm(+ReLU) backward and the tail backward against CPU autograd.  Module
and poser level: d(image), d(layers) and d(pose) against CPU autograd through the fp32 oracle (oracle/tha4_oracle.py) on the
teacher_sds weights.  Warps are compared on the C oracle's base coordinates, which the library samples with.

The module-level bounds are the measured ones with margin (DESIGN.md section 4): the gradient is that of the forward the
context computes, and on these seeded networks it moves far more than the forward does -- the default mode's TF32 / f16
forward (mean output error ~2e-3) gives a gradient 7e-2 - 1.3e-1 (relative L2) from the fp32 one, strict mode 1.7e-3 - 6.4e-3,
and the same data gradients run in 3xTF32 on a default-mode recompute change nothing measurable."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import gpu_util as G
from oracle import synth, tha4_oracle as O
from tha4_b200._lib import Tha4Error, _ptr, _ptr_array
from tha4_b200.nn.eyebrow_decomposer.eyebrow_decomposer_00 import EyebrowDecomposer00
from tha4_b200.nn.eyebrow_morphing_combiner.eyebrow_morphing_combiner_00 import EyebrowMorphingCombiner00
from tha4_b200.nn.face_morpher.face_morpher_08 import FaceMorpher08
from tha4_b200.poser.modes import mode_12

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
DEFAULT_REL, DEFAULT_COS = 0.2, 0.98         # default mode vs the fp32 oracle (see the module docstring)


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
@pytest.mark.parametrize('kind,cin,cout,h', [(0, 4, 64, 16), (0, 8, 64, 16), (0, 64, 16, 16), (0, 524, 512, 8), (0, 539, 512, 8),
                                             (0, 512, 512, 8), (1, 64, 128, 32), (1, 256, 512, 16), (2, 512, 256, 8), (2, 128, 64, 32)])
@pytest.mark.parametrize('strict', [1, 0])
def test_conv_backward_data(kind, cin, cout, h, strict):
    g = torch.Generator().manual_seed(kind * 1000 + cin + cout)
    N = 2
    k = 3 if kind == 0 else 4
    w = torch.randn((cin, cout, 4, 4) if kind == 2 else (cout, cin, k, k), generator=g) * (2.0 / (cin * k * k)) ** 0.5
    x = torch.zeros(N, cin, h, h)
    if kind == 0:
        ho, fwd = h, lambda t: F.conv2d(t, w, None, 1, 1)
    elif kind == 1:
        ho, fwd = h // 2, lambda t: F.conv2d(t, w, None, 2, 1)
    else:
        ho, fwd = 2 * h, lambda t: F.conv_transpose2d(t, w, None, 2, 1)
    dy = torch.randn(N, cout, ho, ho, generator=g) * 1e-3
    x.requires_grad_()
    fwd(x).backward(dy)
    ref = x.grad
    c = G.ctx()
    out = torch.empty(N, cin, h, h, device=DEV)
    dyd, wd = G.dev(dy), G.dev(w)          # kept alive across the call
    c._call('tha4_test_conv_backward_data', kind, _ptr(dyd), _ptr(wd), _ptr(out), N, cin, h, h, cout, strict, c._stream())
    torch.cuda.synchronize()
    rel = _rel(out, ref)
    print('\nconv dgrad kind %d %d->%d strict %d: rel L2 %.3e' % (kind, cout, cin, strict, rel))
    assert rel <= (1e-5 if strict else 3e-3), rel


@pytest.mark.parametrize('act', [0, 1])
def test_norm_backward(act):
    g = torch.Generator().manual_seed(7 + act)
    N, C, H = 2, 64, 16
    x = torch.randn(N, C, H, H, generator=g) * 2 + 0.5
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.3
    dy = torch.randn(N, C, H, H, generator=g)
    xr = x.clone().requires_grad_()
    y = F.instance_norm(xr, weight=gamma, bias=beta, eps=1e-5)
    (F.relu(y) if act else y).backward(dy)
    c = G.ctx()
    dx = torch.empty(N, C, H, H, device=DEV)
    t = [G.dev(v) for v in (x, gamma, beta, dy)]
    c._call('tha4_test_norm_backward', _ptr(t[0]), N, C, H, H, _ptr(t[1]), _ptr(t[2]), act, _ptr(t[3]), _ptr(dx), c._stream())
    torch.cuda.synchronize()
    rel = _rel(dx, xr.grad)
    print('\nnorm backward act %d: rel L2 %.3e' % (act, rel))
    assert rel <= 1e-5, rel


def _base(clib, n, S):
    b = torch.empty(S)
    clib.tha4o_base_grid(S, ctypes.c_void_p(b.data_ptr()))
    return torch.stack([b.view(1, 1, S).expand(n, S, S), b.view(1, S, 1).expand(n, S, S)], dim=-1)


def _warp(clib, grid_change, image):
    grid = _base(clib, image.shape[0], image.shape[2]) + grid_change.permute(0, 2, 3, 1)
    return F.grid_sample(image, grid, mode='bilinear', padding_mode='border', align_corners=False)


def _tail_ref(clib, kind, h, image0, image1):
    """The oracle's tails (tha4_oracle.py) from the head pre-activations h in the library's channel order."""
    if kind == 1:
        bg_a, bg_c, eb_a, eb_c = torch.sigmoid(h[:, 0:1]), torch.tanh(h[:, 1:5]), torch.sigmoid(h[:, 5:6]), torch.tanh(h[:, 6:10])
        return [O.apply_color_change(eb_a, image0, eb_c), eb_a, eb_c, O.apply_color_change(bg_a, bg_c, image0), bg_a, bg_c]
    grid = h[:, 0:2]
    warped = _warp(clib, grid, image0)
    if kind == 2:
        alpha, color, ca = torch.sigmoid(h[:, 2:3]), torch.tanh(h[:, 3:7]), torch.sigmoid(h[:, 7:8])
        morphed = O.apply_color_change(alpha, color, warped)
        return [O.apply_rgb_change(ca, morphed, image1), ca, O.apply_rgb_change((morphed[:, 3:4] + 1.0) / 2.0, morphed, image1),
                morphed, alpha, color, warped, grid]
    imc, ima, eyc, eya = torch.tanh(h[:, 2:6]), torch.sigmoid(h[:, 6:7]), torch.tanh(h[:, 7:11]), torch.sigmoid(h[:, 11:12])
    im1 = O.apply_color_change(ima, imc, warped)
    return [O.apply_color_change(eya, eyc, im1), eya, eyc, im1, ima, imc, warped, grid]


@pytest.mark.parametrize('kind', [1, 2, 3])
@pytest.mark.parametrize('grid', ['zero', 'half', 'border', 'mix'])
def test_tail_backward(oracle_clib, kind, grid):
    if kind == 1 and grid != 'mix':
        pytest.skip('the decomposer does not warp')
    g = torch.Generator().manual_seed(kind * 10 + len(grid))
    N, S, CO = 2, 32, {1: 10, 2: 8, 3: 12}[kind]
    h = torch.randn(N, CO, S, S, generator=g)
    if kind != 1:
        if grid == 'zero':
            h[:, 0:2] = 0
        elif grid == 'half':       # source coordinates on exact half-integers
            h[:, 0:2] = torch.randint(-3, 4, (N, 2, S, S), generator=g).float() / S
        elif grid == 'border':     # every sample clamped to the border
            h[:, 0:2] = torch.where(torch.rand(N, 2, S, S, generator=g) < 0.5, -3.0, 3.0)
        else:
            h[:, 0:2] = (torch.rand(N, 2, S, S, generator=g) - 0.5) * 2.4
    image0 = synth.synthetic_image(kind, N)[:, :, :S, :S].contiguous() * 2 - 1
    image1 = (synth.synthetic_image(kind + 5, N)[:, :, :S, :S].contiguous() * 2 - 1) if kind == 2 else None
    hr, i0r = h.clone().requires_grad_(), image0.clone().requires_grad_()
    i1r = image1.clone().requires_grad_() if image1 is not None else None
    outs = _tail_ref(oracle_clib, kind, hr, i0r, i1r)
    ups = [torch.randn(o.shape, generator=g) if k % 3 != 1 else None for k, o in enumerate(outs)]
    torch.autograd.backward([o for o, u in zip(outs, ups) if u is not None], [u for u in ups if u is not None])
    c = G.ctx()
    outs_d = [G.dev(o.detach()) for o in outs]
    ups_d = [G.dev(u) if u is not None else None for u in ups]
    d_head = torch.empty(N, 12, S, S, device=DEV)
    d0 = torch.empty(N, 4, S, S, device=DEV)
    d1 = torch.empty(N, 4, S, S, device=DEV) if kind == 2 else None
    i0d, i1d = G.dev(image0), (G.dev(image1) if image1 is not None else None)
    c._call('tha4_test_tail_backward', kind, _ptr_array(outs_d), N, S, _ptr(i0d), _ptr(i1d), _ptr_array(ups_d), _ptr(d_head), _ptr(d0),
            _ptr(d1), c._stream())
    torch.cuda.synchronize()
    rh, ri = _rel(d_head[:, :CO], hr.grad), _rel(d0, i0r.grad)
    print('\ntail backward kind %d grid %s: d(head) %.3e d(image0) %.3e' % (kind, grid, rh, ri))
    assert rh <= 1e-5 and ri <= 1e-5, (rh, ri)
    if kind == 2:
        assert _rel(d1, i1r.grad) <= 1e-5
    if grid == 'border':
        assert torch.count_nonzero(d_head[:, 0:2]).item() == 0


# ------------------------------------------------------------------------------------------ module level
def _load(cls, sd):
    m = cls()
    m.load_state_dict(sd)
    return m.to(DEV)


NETS = {
    'eyebrow_decomposer': (EyebrowDecomposer00, 128, 0, 6),
    'eyebrow_morphing_combiner': (EyebrowMorphingCombiner00, 128, 12, 8),
    'face_morpher': (FaceMorpher08, 192, 27, 8),
}


def _inputs(name, B, seed=0):
    _, S, P, _ = NETS[name]
    img = synth.synthetic_image(seed, B)
    if name == 'face_morpher':
        imgs = [img[:, :, 32:224, 160:352].contiguous()]
    else:
        imgs = [img[:, :, 64:192, 192:320].contiguous()]
        if name == 'eyebrow_morphing_combiner':
            imgs = [imgs[0], synth.synthetic_image(seed + 1, B)[:, :, 64:192, 192:320].contiguous()]   # background, eyebrow
    pose = synth.random_poses(B, seed=seed + 3)[:, 12:39].contiguous() if P == 27 else synth.random_poses(B, seed=seed + 3)[:, :P].contiguous()
    return imgs, (pose if P else None)


def _oracle(name, sd, imgs, pose):
    if name == 'eyebrow_decomposer':
        return O.eyebrow_decomposer(sd, imgs[0])
    if name == 'eyebrow_morphing_combiner':
        return O.eyebrow_morphing_combiner(sd, imgs[0], imgs[1], pose)
    return O.face_morpher(sd, imgs[0], pose)


def _ups(outs, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(o.shape, generator=g) * 1e-3 if k in (0, 1, 3, len(outs) - 1) else None for k, o in enumerate(outs)]


def _backward(outs, ups):
    pairs = [(o, u) for o, u in zip(outs, ups) if u is not None]
    torch.autograd.backward([o for o, _ in pairs], [u.to(o.device) for o, u in pairs])


def _cpu_grads(name, sd, imgs, pose, ups):
    imgs = [i.clone().requires_grad_() for i in imgs]
    pose = pose.clone().requires_grad_() if pose is not None else None
    _backward(_oracle(name, sd, imgs, pose), ups)
    return [i.grad for i in imgs] + ([pose.grad] if pose is not None else [])


def _gpu_grads(m, imgs, pose, ups, want=None):
    ins = [i.to(DEV).clone().requires_grad_(want is None or k in want) for k, i in enumerate(imgs)]
    pin = pose.to(DEV).clone().requires_grad_(want is None or len(imgs) in want) if pose is not None else None
    outs = m(*ins, *([pin] if pin is not None else []))
    _backward(outs, ups)
    return [t.grad for t in ins] + ([pin.grad] if pin is not None else []), outs


@pytest.mark.parametrize('strict', [0, 1])
@pytest.mark.parametrize('name', list(NETS))
def test_module_input_grads(teacher_sds, name, strict):
    cls = NETS[name][0]
    m = _load(cls, teacher_sds[name])
    m.context().set_option('strict', strict)
    try:
        B = 2
        imgs, pose = _inputs(name, B)
        with torch.no_grad():
            ref_out = m(*[i.to(DEV) for i in imgs], *([pose.to(DEV)] if pose is not None else []))
        ups = _ups(ref_out, 11)
        grads, outs = _gpu_grads(m, imgs, pose, ups)
        for a, b in zip(outs, ref_out):
            # strict mode's mma.sync convs split K with float atomics: its forward is not bit-reproducible run to run
            assert a.grad_fn is not None and (torch.equal(a, b) if not strict else _rel(a, b) <= 1e-5)
        assert all(p.grad is None for p in m.parameters())
        cpu = _cpu_grads(name, teacher_sds[name], imgs, pose, ups)
        for k, (gg, rr) in enumerate(zip(grads, cpu)):
            rel, cos = _rel_cos('%s strict=%d input %d' % (name, strict, k), gg, rr)
            if strict:
                assert rel <= 1e-2 and cos >= 0.9999, (k, rel, cos)
            else:
                assert rel <= DEFAULT_REL and cos >= DEFAULT_COS, (k, rel, cos)
        # one gradient alone equals the same gradient requested with the others
        n_in = len(grads)
        for k in range(n_in):
            alone, _ = _gpu_grads(m, imgs, pose, ups, want={k})
            print('%s strict=%d input %d alone vs all: rel %.3e' % (name, strict, k, _rel(alone[k], grads[k])))
            # strict mode's forward is not bit-reproducible (split-K float atomics) and each call recomputes it
            assert _rel(alone[k], grads[k]) <= (1e-2 if strict else 1e-6), k
        # scaled upstream gradients scale the result: no f16 staging of gradients
        for sc in (2.0 ** -24, 2.0 ** 24):
            scaled, _ = _gpu_grads(m, imgs, pose, [u * sc if u is not None else None for u in ups])
            for a, b in zip(scaled, grads):
                print('scale %g: rel %.3e' % (sc, _rel(a / sc, b)))
                assert _rel(a / sc, b) <= (1e-2 if strict else 1e-5)      # strict: each call recomputes a non-reproducible forward
    finally:
        m.context().set_option('strict', 0)


def test_batching_matches_single_samples(teacher_sds):
    m = _load(FaceMorpher08, teacher_sds['face_morpher'])
    B = 5
    imgs, pose = _inputs('face_morpher', B, seed=4)
    with torch.no_grad():
        outs = m(imgs[0].to(DEV), pose.to(DEV))
    ups = _ups(outs, 5)
    # strict mode: in the default mode the TF32 split-K plans, which depend on the batch, move the gradient by ~5e-2; strict
    # mode's own run-to-run variation (split-K float atomics in the recomputed forward) is ~1e-3 - 7e-3
    m.context().set_option('strict', 1)
    m.context().set_option('microbatch', 2)
    try:
        batched, _ = _gpu_grads(m, imgs, pose, ups)
        m.context().set_option('microbatch', 32)
        alone_all = [_gpu_grads(m, [imgs[0][n:n + 1]], pose[n:n + 1], [u[n:n + 1] if u is not None else None for u in ups])[0]
                     for n in range(B)]
    finally:
        m.context().set_option('microbatch', 32)
        m.context().set_option('strict', 0)
    for n in range(B):
        for a, b in zip(alone_all[n], batched):
            print('batching sample %d: rel %.3e' % (n, _rel(a[0], b[n])))
            assert _rel(a[0], b[n]) <= 1e-2, n


# ------------------------------------------------------------------------------------------ poser level
def _poser(teacher_sds):
    return mode_12.create_poser(DEV, state_dicts={k: teacher_sds[k] for k in NETS})


def test_mode_12_pose_and_image_grads(teacher_sds):
    poser = _poser(teacher_sds)
    image, pose = synth.synthetic_image(2, 1), synth.random_poses(1, seed=8)
    ups = [None] * 22
    g = torch.Generator().manual_seed(3)
    ups[0] = torch.randn(1, 4, 192, 192, generator=g) * 1e-3
    ups[10] = torch.randn(1, 4, 128, 128, generator=g) * 1e-3
    for which in ('pose', 'image'):
        im = image.to(DEV).clone().requires_grad_(which == 'image')
        po = pose.to(DEV).clone().requires_grad_(which == 'pose')
        outs = poser.get_posing_outputs(im, po)
        _backward(outs, ups)
        imr, por = image.clone().requires_grad_(which == 'image'), pose.clone().requires_grad_(which == 'pose')
        _backward(O.mode_12_outputs({k: teacher_sds[k] for k in NETS}, imr, por), ups)
        if which == 'pose':
            rel, cos = _rel_cos('mode_12 d(pose[:39])', po.grad[:, :39], por.grad[:, :39])
            assert torch.count_nonzero(po.grad[:, 39:]).item() == 0
        else:
            rel, cos = _rel_cos('mode_12 d(image)', im.grad, imr.grad)
        assert rel <= DEFAULT_REL and cos >= DEFAULT_COS, (which, rel, cos)


def test_mode_12_plain_path_and_cache_unchanged(teacher_sds):
    poser = _poser(teacher_sds)
    image, pose = synth.synthetic_image(2, 1).to(DEV), synth.random_poses(1, seed=8).to(DEV)
    a = poser.get_posing_outputs(image, pose)
    b = poser.get_posing_outputs(image, pose)
    assert all(x is y for x, y in zip(a[16:], b[16:]))          # eyebrow cache hit: the cached tensor objects
    with torch.no_grad():
        c = poser.get_posing_outputs(image, pose.clone().requires_grad_())
    assert all(torch.equal(x, y) for x, y in zip(a, c)) and all(x is y for x, y in zip(a[16:], c[16:]))
    d = poser.get_posing_outputs(image, pose.clone().requires_grad_())       # pose grad: the cached decomposer outputs are constants
    assert all(x is y for x, y in zip(a[16:], d[16:]))
    assert all(torch.equal(x, y) for x, y in zip(a, d))


def test_mode_12_pose_fit(teacher_sds):
    poser = _poser(teacher_sds)
    image = synth.synthetic_image(2, 1).to(DEV)
    target_pose = synth.random_poses(1, seed=21).to(DEV)
    with torch.no_grad():
        target = poser.get_posing_outputs(image, target_pose)[0].clone()
    p39 = torch.zeros(1, 39, device=DEV, requires_grad=True)
    opt = torch.optim.Adam([p39], lr=5e-2)
    losses = []
    for _ in range(30):
        pose = torch.cat([p39, torch.zeros(1, 6, device=DEV)], dim=1)
        loss = (poser.get_posing_outputs(image, pose)[0] - target).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    print('\nmode_12 pose fit: L1 %.4e -> %.4e' % (losses[0], losses[-1]))
    assert losses[-1] <= 0.5 * losses[0], losses


# ------------------------------------------------------------------------------------------ hygiene
def test_double_backward_and_inplace_pose_raise(teacher_sds):
    m = _load(FaceMorpher08, teacher_sds['face_morpher'])
    imgs, pose = _inputs('face_morpher', 1)
    p = pose.to(DEV).clone().requires_grad_()
    outs = m(imgs[0].to(DEV), p)
    with pytest.raises(Tha4Error):
        torch.autograd.grad(outs[0].sum(), p, create_graph=True)
    p2 = pose.to(DEV).clone().requires_grad_()
    q = p2 * 1.0
    outs = m(imgs[0].to(DEV), q)
    with torch.no_grad():
        q.add_(1.0)
    with pytest.raises(RuntimeError, match='inplace'):
        outs[0].sum().backward()


def test_two_face_morphers_on_one_context(teacher_sds):
    sd = teacher_sds['face_morpher']
    a = _load(FaceMorpher08, sd)
    b = _load(FaceMorpher08, {k: (v * 0.9 if k.endswith('weight') else v) for k, v in sd.items()})
    b.attach_context(a.context())
    imgs, pose = _inputs('face_morpher', 1, seed=2)
    ups = None
    res = {}
    for m, name in ((a, 'a'), (b, 'b'), (a, 'a2')):
        with torch.no_grad():
            outs = m(imgs[0].to(DEV), pose.to(DEV))
        ups = ups or _ups(outs, 9)
        res[name], _ = _gpu_grads(m, imgs, pose, ups)
    assert _rel(res['a'][1], res['a2'][1]) <= 1e-6
    assert _rel(res['a'][1], res['b'][1]) > 1e-3
    cpu_b = _cpu_grads('face_morpher', {k: (v * 0.9 if k.endswith('weight') else v) for k, v in sd.items()}, imgs, pose, ups)
    rel, cos = _rel_cos('second module d(pose)', res['b'][1], cpu_b[1])
    assert rel <= DEFAULT_REL and cos >= DEFAULT_COS
