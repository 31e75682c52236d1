"""Frozen SIREN students under torch.autograd on the H100 (-m gpu): gradients w.r.t. image and pose.

d(image) is the exact adjoint of the warp the forward returned: held to relative L2 <= 1e-5 against CPU autograd through
apply_grid_change + blend at the module's own returned grid_change / alpha, on the base coordinates the library samples
with (oracle/gridsample_ref.c; torch's affine_grid differs from them by up to one ulp, which alone moves d(image) by ~1e-5).  d(pose) is the gradient of the TF32 recompute, held
to the parameter gradients' bounds against CPU autograd on the fp32 oracle: relative L2 <= 3e-2, cosine >= 0.999."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import gpu_util as G
from oracle import synth, tha4_oracle as O
from tha4_b200.poser.modes import mode_14

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
BODY_CH = (4, 1, 4, 4, 2)


def _smooth(seed, n, c, amp=1.0):
    return ((synth.synthetic_image(seed, n)[:, :c] - 0.5) * amp).contiguous()


def _body(sd):
    return mode_14.load_body_morpher(None, {k: v.clone() for k, v in sd.items()}).to(DEV).requires_grad_(False)


def _face(sd):
    return mode_14.load_face_morpher(None, {k: v.clone() for k, v in sd.items()}).to(DEV).requires_grad_(False)


def _rel_cos(name, g, ref):
    g, ref = g.double().cpu().reshape(-1), ref.double().reshape(-1)
    rel = ((g - ref).norm() / ref.norm()).item()
    cos = torch.nn.functional.cosine_similarity(g, ref, dim=0).item()
    print('\n%s: rel L2 %.3e cosine %.6f |ref| %.3e' % (name, rel, cos, ref.norm().item()))
    return rel, cos


def _assert_pose_bounds(name, g, ref):
    rel, cos = _rel_cos(name, g, ref)
    assert rel <= 3e-2 and cos >= 0.999, (name, rel, cos)


def _backward(outs, ups):
    pairs = [(o, u) for o, u in zip(outs, ups) if u is not None]
    torch.autograd.backward([o for o, _ in pairs], [u.to(o.device) for o, u in pairs])


def _cpu_body_input_grads(sd, image, pose, ups):
    image, pose = image.clone().requires_grad_(), pose.clone().requires_grad_()
    _backward(O.siren_morpher_03(sd, image, pose), ups)
    return image.grad, pose.grad


def _apply_grid_change(oracle_clib, grid_change, image):
    """O.apply_grid_change on the C oracle's base coordinates (bit-identical to the library's table, test_abi.py)."""
    n, _, h, w = image.shape
    bx, by = torch.empty(w), torch.empty(h)
    oracle_clib.tha4o_base_grid(w, ctypes.c_void_p(bx.data_ptr()))
    oracle_clib.tha4o_base_grid(h, ctypes.c_void_p(by.data_ptr()))
    base = torch.stack([bx.view(1, 1, w).expand(n, h, w), by.view(1, h, 1).expand(n, h, w)], dim=-1)
    grid = base + grid_change.permute(0, 2, 3, 1)
    return F.grid_sample(image, grid, mode='bilinear', padding_mode='border', align_corners=False)


def _cpu_warp_adjoint(oracle_clib, grid_change, alpha, color, image, g_bl, g_wp):
    """d image of (blended, warped) = ((1 - alpha) warped + alpha colour, apply_grid_change(grid_change, image)) at the
    given (returned) grid_change / alpha, by CPU autograd."""
    image = image.clone().requires_grad_()
    warped = _apply_grid_change(oracle_clib, grid_change, image)
    blended = (1 - alpha) * warped + alpha * color
    torch.autograd.backward([blended, warped], [g_bl, g_wp])
    return image.grad


# ------------------------------------------------------------------------------------------ forward values
def test_forward_equals_no_grad_and_parameters_get_no_grad(student_sds):
    body, face = _body(student_sds['body_morpher']), _face(student_sds['face_morpher'])
    img, pose = synth.synthetic_image(3, 2).to(DEV), synth.random_poses(2, seed=6).to(DEV)
    with torch.no_grad():
        ref = body(img, pose)
        fref = face(pose[:, :39].contiguous())
    for im, po in ((img.clone().requires_grad_(), pose), (img, pose.clone().requires_grad_()),
                   (img.clone().requires_grad_(), pose.clone().requires_grad_())):
        outs = body(im, po)
        assert len(outs) == 5
        for a, b in zip(outs, ref):
            assert a.grad_fn is not None and torch.equal(a, b)
        assert len({o.data_ptr() for o in outs}) == 5
        sum(o.sum() for o in outs).backward()
    p39 = pose[:, :39].clone().requires_grad_()
    f = face(p39)
    assert f.grad_fn is not None and torch.equal(f, fref)
    f.sum().backward()
    assert p39.grad is not None and p39.grad.shape == (2, 39)
    assert all(p.grad is None for p in list(body.parameters()) + list(face.parameters()))


# ------------------------------------------------------------------------------------------ exact image adjoint
def _grid_head(sd, dx, dy):
    """Body weights whose grid_change output is the constant (dx, dy): zero grid rows of the head, bias = offset."""
    sd = {k: v.clone() for k, v in sd.items()}
    sd['last_linear.weight'][0:2].zero_()
    sd['last_linear.bias'][0], sd['last_linear.bias'][1] = dx, dy
    return sd


# base + dx puts every sample at ix = x + 256 dx: dx = 0 is the identity grid (integer positions), 1 / 512 exact
# half-integers, +-1.5 the border clamp on every pixel, (0.25, -0.3125) clamps the last 64 columns and the first 80 rows
# (all offsets are exact in fp16 and fp32)
@pytest.mark.parametrize('grid', ['siren', 'zero', 'half_integer', 'border_clamp', 'mixed_clamp'])
def test_image_gradient_is_exact_adjoint_of_returned_warp(student_sds, oracle_clib, grid):
    sd = student_sds['body_morpher']
    sd = {'siren': sd, 'zero': _grid_head(sd, 0.0, 0.0), 'half_integer': _grid_head(sd, 1.0 / 512, -3.0 / 512),
          'border_clamp': _grid_head(sd, 1.5, -1.5), 'mixed_clamp': _grid_head(sd, 0.25, -0.3125)}[grid]
    n = 2
    img, pose = synth.synthetic_image(7, n), synth.random_poses(n, seed=8)
    g_bl, g_wp = torch.randn(n, 4, 512, 512, generator=torch.Generator().manual_seed(1)), _smooth(22, n, 4)
    body = _body(sd)
    im = img.to(DEV).requires_grad_()
    outs = body(im, pose.to(DEV))
    torch.autograd.backward([outs[0], outs[3]], [g_bl.to(DEV), g_wp.to(DEV)])
    gc, alpha, color = outs[4].detach().cpu(), outs[1].detach().cpu(), outs[2].detach().cpu()
    if grid != 'siren':
        assert torch.all(gc[:, 0] == sd['last_linear.bias'][0]) and torch.all(gc[:, 1] == sd['last_linear.bias'][1])
    ref = _cpu_warp_adjoint(oracle_clib, gc, alpha, color, img, g_bl, g_wp)
    rel, _ = _rel_cos('d image, %s grid' % grid, im.grad, ref)
    assert rel <= 1e-5, rel


def test_image_gradient_subsets_of_upstream(student_sds, oracle_clib):
    """Only g_warped, only g_blended, and none (alpha / colour / grid only: d image = 0)."""
    sd = student_sds['body_morpher']
    img, pose = synth.synthetic_image(9, 1), synth.random_poses(1, seed=10)
    body = _body(sd)
    g = _smooth(23, 1, 4)
    for which in ('warped', 'blended', 'none'):
        im = img.to(DEV).requires_grad_()
        outs = body(im, pose.to(DEV))
        if which == 'none':
            (outs[1].sum() + outs[2].sum() + outs[4].sum()).backward()
            assert torch.count_nonzero(im.grad) == 0
            continue
        outs[3 if which == 'warped' else 0].backward(g.to(DEV))
        z = torch.zeros_like(g)
        ups = (z, g) if which == 'warped' else (g, z)
        ref = _cpu_warp_adjoint(oracle_clib, outs[4].detach().cpu(), outs[1].detach().cpu(), outs[2].detach().cpu(), img, *ups)
        rel, _ = _rel_cos('d image, only %s' % which, im.grad, ref)
        assert rel <= 1e-5, rel


# ------------------------------------------------------------------------------------------ pose gradient parity
@pytest.mark.parametrize('which', ['all', 'subset', 'sum'])
def test_body_pose_gradient_parity(student_sds, which):
    sd = student_sds['body_morpher']
    n = 2
    img, pose = synth.synthetic_image(11, n), synth.random_poses(n, seed=4)
    if which == 'sum':
        ups = [torch.ones(n, c, 512, 512) for c in BODY_CH]
    else:
        ups = [_smooth(20 + i, n, c, 1e-3) for i, c in enumerate(BODY_CH)]
        if which == 'subset':
            ups = [ups[0], None, None, ups[3], None]
    ref_image, ref_pose = _cpu_body_input_grads(sd, img, pose, ups)
    body = _body(sd)
    im, po = img.to(DEV).requires_grad_(), pose.to(DEV).requires_grad_()
    outs = body(im, po)
    if which == 'sum':
        sum(o.sum() for o in outs).backward()
    else:
        _backward(outs, ups)
    assert po.grad.shape == (n, 45)
    _assert_pose_bounds('body d pose, upstream %s' % which, po.grad, ref_pose)
    # d image through the student's own (fp16-operand) warp vs the fp32 oracle's: the grids differ by the forward's rounding
    _rel_cos('body d image vs the fp32 oracle, upstream %s' % which, im.grad, ref_image)


def test_face_pose_gradient_parity(student_sds):
    sd = student_sds['face_morpher']
    n = 3
    pose = synth.random_poses(n, seed=9)[:, :39].contiguous()
    up = _smooth(31, n, 4, 1e-3)[:, :, 100:228, 190:318].contiguous()
    p = pose.clone().requires_grad_()
    O.siren_face_morpher(sd, p).backward(up)
    face = _face(sd)
    po = pose.to(DEV).requires_grad_()
    face(po).backward(up.to(DEV))
    _assert_pose_bounds('face d pose', po.grad, p.grad)


# ------------------------------------------------------------------------------------------ the student DAG of mode_14
def test_composed_student_dag_pose_gradient(student_sds):
    """face(pose[:, :39]) pasted at rows 80:208, cols 192:320 of the image the body student warps: d pose [B,45] vs
    autograd through O.mode_14_outputs.  The face-pose part reaches the pose only through d(image) of the body."""
    n = 2
    img, pose = synth.synthetic_image(13, n), synth.random_poses(n, seed=14)
    ups = [_smooth(50 + i, n, c, 1e-3) for i, c in enumerate(BODY_CH)]
    p = pose.clone().requires_grad_()
    _backward(O.mode_14_outputs(student_sds, img, p)[:5], ups)
    body, face = _body(student_sds['body_morpher']), _face(student_sds['face_morpher'])
    po = pose.to(DEV).requires_grad_()
    body_in = img.to(DEV).clone()
    body_in[:, :, 80:208, 192:320] = face(po[:, :39])
    _backward(body(body_in, po), ups)
    _assert_pose_bounds('student DAG d pose', po.grad, p.grad)
    assert po.grad[:, :39].abs().max().item() > 0 and p.grad[:, :39].abs().max().item() > 0
    _assert_pose_bounds('student DAG d pose, face part', po.grad[:, :39], p.grad[:, :39])


# ------------------------------------------------------------------------------------------ only what is asked for
def test_only_requested_gradients_are_computed(student_sds):
    body = _body(student_sds['body_morpher'])
    ctx = body.sync_weights()
    img, pose = synth.synthetic_image(1, 1).to(DEV), synth.random_poses(1, seed=2).to(DEV)
    up = _smooth(3, 1, 4, 1e-3).to(DEV)
    # image only: the scatter and the layout pass, no SIREN recompute
    im = img.clone().requires_grad_()
    out = body(im, pose)[0]
    l0 = ctx.counter('kernel_launches')
    out.backward(up)
    torch.cuda.synchronize()
    image_only = ctx.counter('kernel_launches') - l0
    # pose only: the recompute and the dgrad chain, without weight gradients
    po = pose.clone().requires_grad_()
    out = body(img, po)[0]
    l0 = ctx.counter('kernel_launches')
    out.backward(up)
    pose_only = ctx.counter('kernel_launches') - l0
    # parameters (the existing path) for comparison
    trainable = mode_14.load_body_morpher(None, {k: v.clone() for k, v in student_sds['body_morpher'].items()}).to(DEV)
    trainable.attach_context(ctx)
    out = trainable(img, pose)[0]
    l0 = ctx.counter('kernel_launches')
    out.backward(up)
    params = ctx.counter('kernel_launches') - l0
    print('\nbackward launches: image only %d, pose only %d, parameters %d' % (image_only, pose_only, params))
    assert image_only <= 3, image_only
    assert im.grad is not None and po.grad is not None
    assert pose_only < params, (pose_only, params)


# ------------------------------------------------------------------------------------------ micro-batching
def test_body_micro_batches(student_sds):
    """B = 10 runs as micro-batches of 8 and 2: d pose bitwise equal to the two separate calls, d image to rounding."""
    sd = student_sds['body_morpher']
    ctx = G.ctx()
    image, pose = synth.synthetic_image(5, 10).to(DEV), synth.random_poses(10, seed=12).to(DEV)
    ups = [_smooth(40 + i, 10, c, 1e-3).to(DEV) for i, c in enumerate(BODY_CH)]
    with torch.no_grad():
        outs = _body(sd)(image, pose)
    flat = torch.cat([v.reshape(-1) for v in sd.values()]).to(DEV)
    res = {}
    for key, sl in (('all', slice(0, 10)), ('8', slice(0, 8)), ('2', slice(8, 10))):
        b = sl.stop - sl.start
        di, dp = torch.empty(b, 4, 512, 512, device=DEV), torch.empty(b, 45, device=DEV)
        ctx.siren_morpher_backward_ex(image[sl], pose[sl], [u[sl] for u in ups], outs[4][sl], outs[1][sl], flat, d_image=di, d_pose=dp)
        res[key] = (di, dp)
    again = torch.empty(10, 45, device=DEV)
    ctx.siren_morpher_backward_ex(image, pose, ups, outs[4], outs[1], flat, d_pose=again)
    torch.cuda.synchronize()
    sep_i, sep_p = torch.cat([res['8'][0], res['2'][0]]), torch.cat([res['8'][1], res['2'][1]])
    assert torch.equal(res['all'][1], sep_p)
    assert torch.equal(again, res['all'][1])                 # no atomics in d pose: reproducible
    assert ((res['all'][0] - sep_i).norm() / sep_i.norm()).item() <= 1e-6


def test_face_micro_batches(student_sds):
    sd = student_sds['face_morpher']
    ctx = G.ctx()
    pose = synth.random_poses(70, seed=13)[:, :39].contiguous().to(DEV)
    up = torch.randn(70, 4, 128, 128, generator=torch.Generator().manual_seed(2)).to(DEV) * 1e-3
    flat = torch.cat([v.reshape(-1) for v in sd.values()]).to(DEV)
    d70, d64, d6 = torch.empty(70, 39, device=DEV), torch.empty(64, 39, device=DEV), torch.empty(6, 39, device=DEV)
    ctx.siren_face_morpher_backward_ex(pose, up, flat, d_pose=d70)
    ctx.siren_face_morpher_backward_ex(pose[:64], up[:64], flat, d_pose=d64)
    ctx.siren_face_morpher_backward_ex(pose[64:], up[64:], flat, d_pose=d6)
    torch.cuda.synchronize()
    assert torch.equal(d70, torch.cat([d64, d6]))


def test_parameter_gradients_unchanged_by_the_extended_entry(student_sds):
    """tha4_siren_morpher_backward_ex with grads (and d pose) gives the parameter gradient of tha4_siren_morpher_backward."""
    sd = student_sds['body_morpher']
    ctx = G.ctx()
    image, pose = synth.synthetic_image(15, 2).to(DEV), synth.random_poses(2, seed=16).to(DEV)
    ups = [_smooth(60 + i, 2, c, 1e-3).to(DEV) for i, c in enumerate(BODY_CH)]
    with torch.no_grad():
        outs = _body(sd)(image, pose)
    flat = torch.cat([v.reshape(-1) for v in sd.values()]).to(DEV)
    g_old, g_new, dp = torch.empty_like(flat), torch.empty_like(flat), torch.empty(2, 45, device=DEV)
    ctx.siren_morpher_backward(image, pose, ups, flat, g_old)
    ctx.siren_morpher_backward_ex(image, pose, ups, outs[4], outs[1], flat, grads=g_new, d_pose=dp)
    torch.cuda.synchronize()
    assert ((g_new - g_old).norm() / g_old.norm()).item() <= 1e-5


# ------------------------------------------------------------------------------------------ hygiene
def test_inplace_pose_write_between_forward_and_backward_raises(student_sds):
    face = _face(student_sds['face_morpher'])
    pose = synth.random_poses(1, seed=3)[:, :39].contiguous().to(DEV).requires_grad_()
    out = face(pose)
    with torch.no_grad():
        pose.add_(1e-3)
    with pytest.raises(RuntimeError, match='inplace'):
        out.sum().backward()
    body = _body(student_sds['body_morpher'])
    img, bpose = synth.synthetic_image(1, 1).to(DEV), synth.random_poses(1, seed=2).to(DEV).requires_grad_()
    outs = body(img, bpose)
    with torch.no_grad():
        bpose.mul_(0.5)
    with pytest.raises(RuntimeError, match='inplace'):
        outs[0].sum().backward()


def test_double_backward_raises(student_sds):
    face = _face(student_sds['face_morpher'])
    pose = synth.random_poses(1, seed=3)[:, :39].contiguous().to(DEV).requires_grad_()
    with pytest.raises(RuntimeError, match='create_graph'):
        torch.autograd.grad(face(pose).sum(), [pose], create_graph=True)
    body = _body(student_sds['body_morpher'])
    img = synth.synthetic_image(1, 1).to(DEV).requires_grad_()
    with pytest.raises(RuntimeError, match='create_graph'):
        torch.autograd.grad(body(img, synth.random_poses(1, seed=2).to(DEV))[3].sum(), [img], create_graph=True)


def test_pose_fitting_reduces_the_loss(student_sds):
    """A few Adam steps on the pose toward a frame rendered at a known pose lower the image loss."""
    face = _face(student_sds['face_morpher'])
    target_pose = synth.random_poses(1, seed=21)[:, :39].contiguous().to(DEV)
    with torch.no_grad():
        target = face(target_pose)
    start = target_pose + 0.05 * torch.randn(target_pose.shape, generator=torch.Generator().manual_seed(4)).to(DEV)
    pose = start.clone().requires_grad_()
    opt = torch.optim.Adam([pose], lr=5e-3)
    losses = []
    for _ in range(30):
        loss = (face(pose) - target).square().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    print('\npose fitting loss: %.4e -> %.4e' % (losses[0], losses[-1]))
    assert losses[-1] < 0.5 * losses[0], losses
