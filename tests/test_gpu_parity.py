"""Network- and poser-level parity on the H100 (-m gpu): the CUDA path, called through the reference-shaped Python
API (which goes through the C ABI), against the CPU oracle on the same seeded weights / inputs, and against the
committed golden fixtures produced by the unmodified reference.

Tolerances (outputs live in [-1, 1]; stated per precision mode).  The seeded teacher weights are conditioned like
trained ones (tha4_b200/synthetic.py), so the fp32 oracle is a well-conditioned yardstick: rounding every conv operand of
the CPU oracle to a 10-bit mantissa moves each mode_07 output by <= 3e-4 mean / 1.4e-2 max
(scripts/dev/cpu_10bit_sensitivity.py).
  strict (3xTF32 products == fp32 convolution): single network: max-abs 2e-3, mean-abs 1e-4 over every output;
      whole poser (up to five chained networks, each warping the previous one's output): max-abs 3e-2, mean-abs 3e-4
      -- the max is set by isolated edge pixels where a ~5e-5 difference of a warp offset moves the sampling point.
  default (the BENCHMARKED mode: wgmma convs on f16 / TF32 operands with a 10-bit mantissa, fp32 accumulation,
      fast-math SiLU -- the class of PyTorch's own CUDA path with TF32 convs): every output of every network and of the
      whole poser: mean-abs <= 2e-3, max-abs <= 5e-2.
  student (fp16 tensor-core products, fp32 accumulation): mean-abs 4e-3 on images, 1e-3 on grid_change.
"""
import os

import numpy
import pytest
import torch

from oracle import image_io, synth, tha4_oracle as O
import gpu_util as G
from tha4_b200.poser.modes import mode_07, mode_12, mode_14

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
STRIDE, OFFSET = 8, 3


def _report(name, outs, refs):
    rows = []
    for i, (a, b) in enumerate(zip(outs, refs)):
        mx, mean = G.err(a.cpu(), b)
        rows.append((i, tuple(b.shape), mx, mean))
    print('\n' + name + '\n' + '\n'.join('  out %2d %-18s max %.3e mean %.3e' % r for r in rows))
    return rows


def _assert_close(name, outs, refs, max_tol, mean_tol):
    assert len(outs) == len(refs)
    rows = _report(name, outs, refs)
    for (i, shape, mx, mean), a in zip(rows, outs):
        assert tuple(a.shape) == shape, (name, i)
        assert mean <= mean_tol, (name, i, 'mean', mean)
        assert mx <= max_tol, (name, i, 'max', mx)


@pytest.fixture(scope='module')
def teacher_poser(teacher_sds):
    poser = mode_07.create_poser(DEV, state_dicts=teacher_sds)
    poser.get_modules()
    return poser


def _set_strict(poser, v):
    poser.get_context().set_option('strict', v)


DEFAULT_MAX_TOL, DEFAULT_MEAN_TOL = 5e-2, 2e-3


# ------------------------------------------------------------------------------------------------ module level
@pytest.mark.parametrize('strict', [1, 0])
def test_module_level_parity(teacher_sds, strict):
    """All five teacher networks stand-alone, in strict mode and in the default (benchmarked) mode."""
    g = torch.Generator().manual_seed(5)
    B = 2
    with torch.no_grad():
        for name, cls in mode_07._CLASSES.items():
            m = cls()
            m.load_state_dict(teacher_sds[name])
            m.to(DEV)
            m.context().set_option('strict', strict)
            sd = teacher_sds[name]
            if name == 'eyebrow_decomposer':
                x = synth.synthetic_image(1, B)[:, :, 64:192, 192:320].contiguous()
                outs, refs = m(x.to(DEV)), O.eyebrow_decomposer(sd, x)
            elif name == 'eyebrow_morphing_combiner':
                a = synth.synthetic_image(2, B)[:, :, 64:192, 192:320].contiguous()
                b = synth.synthetic_image(3, B)[:, :, 64:192, 192:320].contiguous()
                p = torch.rand(B, 12, generator=g)
                outs, refs = m(a.to(DEV), b.to(DEV), p.to(DEV)), O.eyebrow_morphing_combiner(sd, a, b, p)
            elif name == 'face_morpher':
                x = synth.synthetic_image(4, B)[:, :, 32:224, 160:352].contiguous()
                p = torch.rand(B, 27, generator=g)
                outs, refs = m(x.to(DEV), p.to(DEV)), O.face_morpher(sd, x, p)
            elif name == 'body_morpher':
                x = torch.nn.functional.interpolate(synth.synthetic_image(5, B), size=(256, 256), mode='bilinear')
                p = torch.rand(B, 6, generator=g) * 2 - 1
                outs, refs = m(x.to(DEV), p.to(DEV)), O.morpher_00(sd, x, p)
            else:
                x = synth.synthetic_image(6, B)
                cp = synth.synthetic_image(7, B)
                cg = torch.randn(B, 2, 512, 512, generator=g) * 0.02
                p = torch.rand(B, 6, generator=g) * 2 - 1
                outs, refs = m(x.to(DEV), cp.to(DEV), cg.to(DEV), p.to(DEV)), O.upscaler_02(sd, x, cp, cg, p)
            if strict:
                _assert_close(name + ' (strict)', outs, refs, 2e-3, 1e-4)
            else:
                _assert_close(name + ' (default mode)', outs, refs, DEFAULT_MAX_TOL, DEFAULT_MEAN_TOL)
            del m
            torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ teacher poser
def test_mode_07_parity_strict_and_golden(teacher_poser, teacher_sds, golden_dir):
    _set_strict(teacher_poser, 1)
    npz = numpy.load(os.path.join(golden_dir, 'teacher_seed0.npz'))
    poses = torch.from_numpy(npz['poses'])
    img = synth.synthetic_image(0, 1)[0]
    with torch.no_grad():
        for p in range(2):
            outs = teacher_poser.get_posing_outputs(img.to(DEV), poses[p].to(DEV))
            refs = O.mode_07_outputs(teacher_sds, img, poses[p])
            assert len(outs) == 33
            _assert_close('mode_07 strict pose %d' % p, outs, refs, 3e-2, 3e-4)
            for i, t in enumerate(outs):      # the reference's own outputs (golden fixture), sub-sampled
                gold = npz['p%d_o%02d' % (p, i)]
                got = t.cpu()[:, :, OFFSET::STRIDE, OFFSET::STRIDE].numpy()
                assert numpy.abs(got - gold).max() <= 3e-2 and numpy.abs(got - gold).mean() <= 3e-4, (p, i)


def test_mode_07_parity_default_mode(teacher_sds):
    """The mode bench.py times: a fresh poser (cold eyebrow cache, every network in the default precision mode), two
    poses, all 33 outputs against the CPU oracle."""
    poser = mode_07.create_poser(DEV, state_dicts=teacher_sds)
    poser.get_context().set_option('strict', 0)
    img = synth.synthetic_image(0, 1)[0]
    with torch.no_grad():
        for seed in (99, 7):
            pose = synth.random_poses(1, seed=seed)[0]
            outs = poser.get_posing_outputs(img.to(DEV), pose.to(DEV))
            refs = O.mode_07_outputs(teacher_sds, img, pose)
            assert len(outs) == 33
            _assert_close('mode_07 default mode, pose seed %d' % seed, outs, refs, DEFAULT_MAX_TOL, DEFAULT_MEAN_TOL)


def test_mode_07_default_mode_golden(teacher_sds, golden_dir):
    """Default mode against the reference's own outputs (fixture written by oracle/make_golden.py from /root/reference)."""
    poser = mode_07.create_poser(DEV, state_dicts=teacher_sds)
    npz = numpy.load(os.path.join(golden_dir, 'teacher_seed0.npz'))
    poses = torch.from_numpy(npz['poses'])
    img = synth.synthetic_image(0, 1)[0]
    with torch.no_grad():
        for p in range(2):
            outs = poser.get_posing_outputs(img.to(DEV), poses[p].to(DEV))
            for i, t in enumerate(outs):
                gold = npz['p%d_o%02d' % (p, i)]
                got = t.cpu()[:, :, OFFSET::STRIDE, OFFSET::STRIDE].numpy()
                assert numpy.abs(got - gold).max() <= DEFAULT_MAX_TOL and numpy.abs(got - gold).mean() <= DEFAULT_MEAN_TOL, (p, i)


def test_mode_07_batch_promotion_and_microbatch(teacher_poser, teacher_sds):
    """rank-3 image / rank-1 pose are promoted (general_poser_02.py:66-69); B=3 with micro-batch 2 == per-sample runs."""
    _set_strict(teacher_poser, 1)
    ctx = teacher_poser.get_context()
    imgs = synth.synthetic_image(1, 3)
    poses = synth.random_poses(3, seed=7)
    ctx.set_option('microbatch', 2)
    with torch.no_grad():
        outs = teacher_poser.get_posing_outputs(imgs.to(DEV), poses.to(DEV))
        for n in (0, 2):
            single = teacher_poser.get_posing_outputs(imgs[n].to(DEV), poses[n].to(DEV))
            for a, b in zip(outs, single):
                assert b.shape[0] == 1
                assert G.err(a[n:n + 1].cpu(), b.cpu())[1] <= 3e-4       # different split-K plans per batch size + atomics: not bit-reproducible
        ref = O.mode_07_outputs(teacher_sds, imgs[1], poses[1])
        _assert_close('mode_07 batch sample 1', [o[1:2] for o in outs], ref, 3e-2, 3e-4)
    ctx.set_option('microbatch', 32)
    out0 = teacher_poser.pose(imgs[0].to(DEV), poses[0].to(DEV))
    assert out0.shape == (1, 4, 512, 512)


def test_mode_07_eyebrow_cache_semantics(teacher_sds):
    """mode_07.py:56-68: same image -> decomposer outputs are reused (same tensor objects); changed image or batch
    size -> recomputed."""
    poser = mode_07.create_poser(DEV, state_dicts=teacher_sds)
    poser.get_context().set_option('strict', 1)
    img = synth.synthetic_image(0, 1).to(DEV)
    p0, p1 = synth.random_poses(2, seed=3).to(DEV)
    with torch.no_grad():
        o0 = poser.get_posing_outputs(img, p0)
        launches0 = poser.get_context().counter('kernel_launches')
        o1 = poser.get_posing_outputs(img, p1)
        launches1 = poser.get_context().counter('kernel_launches')
        assert all(a is b for a, b in zip(o0[27:], o1[27:])), 'cache hit returns the cached decomposer tensors'
        o1b = poser.get_posing_outputs(img.clone(), p1)          # equal content, different tensor: still a hit
        assert all(a is b for a, b in zip(o0[27:], o1b[27:]))
        for a, b in zip(o1, o1b):
            assert G.err(a.cpu(), b.cpu())[1] <= 1e-5          # atomics make runs differ in the last bits
        img2 = img.clone()
        img2[0, 0, 100, 250] += 0.25
        o2 = poser.get_posing_outputs(img2, p1)
        launches2 = poser.get_context().counter('kernel_launches')
        assert not any(a is b for a, b in zip(o0[27:], o2[27:]))
        assert (launches2 - launches1) > (launches1 - launches0), 'a cache miss runs the decomposer kernels again'
        ref = O.mode_07_outputs(teacher_sds, img2[0].cpu(), p1.cpu())
        _assert_close('mode_07 after cache miss', o2, ref, 3e-2, 3e-4)


def test_mode_07_graph_replay_matches_eager(teacher_sds):
    """Single-chunk teacher forwards whose buffer addresses repeat are replayed as ONE captured CUDA graph (capi.cu): the
    replayed frames must equal the eagerly launched ones (same kernels, same order; statistics use atomics, so equality is
    to 1e-5) and follow the pose that is passed, and the launch counter must keep counting the graph's kernels."""
    import tha4_b200._lib as L
    poser = mode_07.create_poser(DEV, state_dicts=teacher_sds)
    ctx = poser.get_context()
    img = synth.synthetic_image(0, 1).to(DEV)
    poses = synth.random_poses(3, seed=17).to(DEV)
    pose_buf = torch.empty(1, 45, device=DEV)
    with torch.no_grad():
        ctx.set_option('cuda_graphs', 0)
        eager = []
        for i in range(3):
            pose_buf.copy_(poses[i:i + 1])
            eager.append([t.clone() for t in poser.get_posing_outputs(img, pose_buf)])
        ctx.set_option('cuda_graphs', 1)
        # a caller that reuses its buffers: outputs of the previous call are dropped before the next call allocates
        outs = None
        l_prev = ctx.counter('kernel_launches')
        per_call = []
        for rep in range(3):
            for i in range(3):
                pose_buf.copy_(poses[i:i + 1])
                outs = None
                outs = poser.get_posing_outputs(img, pose_buf)
                torch.cuda.synchronize()
                l_now = ctx.counter('kernel_launches')
                per_call.append(l_now - l_prev)
                l_prev = l_now
                for a, b in zip(outs, eager[i]):
                    assert G.err(a.cpu(), b.cpu())[0] <= 1e-4, (rep, i)
        assert min(per_call) > 100, 'replayed graphs must keep counting their kernels: %s' % per_call
        assert ctx.counter('graph_captures') >= 1 and ctx.counter('graph_replays') >= 6, \
            (ctx.counter('graph_captures'), ctx.counter('graph_replays'))
        # the pose is staged into a library buffer ahead of the graph, so a pose living at a new address every call
        # (slices of a pose table) still replays
        r0 = ctx.counter('graph_replays')
        for i in range(3):
            outs = None
            outs = poser.get_posing_outputs(img, poses[i:i + 1])
            for a, b in zip(outs, eager[i]):
                assert G.err(a.cpu(), b.cpu())[0] <= 1e-4, i
        assert ctx.counter('graph_replays') >= r0 + 3


@pytest.mark.parametrize('strict', [1, 0])
def test_mode_12_parity(teacher_sds, strict):
    poser = mode_12.create_poser(DEV, state_dicts={k: teacher_sds[k] for k in ('eyebrow_decomposer', 'eyebrow_morphing_combiner', 'face_morpher')})
    poser.get_context().set_option('strict', strict)
    assert poser.get_output_length() == 18
    img = synth.synthetic_image(2, 1)[0]
    pose = synth.random_poses(1, seed=12)[0]
    with torch.no_grad():
        outs = poser.get_posing_outputs(img.to(DEV), pose.to(DEV))
        refs = O.mode_12_outputs(teacher_sds, img, pose)
    assert len(outs) == 22
    if strict:
        _assert_close('mode_12 strict', outs, refs, 3e-2, 3e-4)
    else:
        _assert_close('mode_12 default mode', outs, refs, DEFAULT_MAX_TOL, DEFAULT_MEAN_TOL)


# ------------------------------------------------------------------------------------------------ student poser
STUDENT_MEAN_TOL = [4e-3, 2e-3, 2e-3, 4e-3, 1e-3, 2e-3]


def _check_student(name, outs, refs):
    rows = _report(name, outs, refs)
    for (i, shape, mx, mean), a in zip(rows, outs):
        assert tuple(a.shape) == shape
        assert mean <= STUDENT_MEAN_TOL[i], (name, i, mean)
    assert rows[4][2] <= 1e-2, 'grid_change max error (normalised coordinates)'
    assert rows[1][2] <= 0.1 and rows[2][2] <= 0.1 and rows[5][2] <= 0.1, 'alpha / colour / face max error'


def test_mode_14_parity_lambda00_and_golden(lambda00_sds, golden_dir):
    poser = mode_14.create_poser(DEV, state_dicts=lambda00_sds)
    npz = numpy.load(os.path.join(golden_dir, 'student_lambda00.npz'))
    poses = torch.from_numpy(npz['poses'])
    img = image_io.load_rgba_png(os.path.join(golden_dir, 'data', 'lambda_00.png'))
    with torch.no_grad():
        for p in range(2):
            outs = poser.get_posing_outputs(img.to(DEV), poses[p].to(DEV))
            refs = O.mode_14_outputs(lambda00_sds, img, poses[p])
            assert len(outs) == 6
            _check_student('mode_14 lambda_00 pose %d' % p, outs, refs)
            gold = npz['p%d_o04' % p]                             # reference's own grid_change, sub-sampled
            got = outs[4].cpu()[:, :, OFFSET::STRIDE, OFFSET::STRIDE].numpy()
            assert numpy.abs(got - gold).max() <= 1e-2


def test_mode_14_parity_synthetic_batch(student_sds):
    poser = mode_14.create_poser(DEV, state_dicts=student_sds)
    imgs = synth.synthetic_image(4, 3)
    poses = synth.random_poses(3, seed=5)
    with torch.no_grad():
        outs = poser.get_posing_outputs(imgs.to(DEV), poses.to(DEV))
        for n in range(3):
            refs = O.mode_14_outputs(student_sds, imgs[n], poses[n])
            _check_student('mode_14 synthetic sample %d' % n, [o[n:n + 1] for o in outs], refs)


def test_student_modules_standalone(student_sds):
    face = mode_14.load_face_morpher(None, student_sds['face_morpher']).to(DEV)
    body = mode_14.load_body_morpher(None, student_sds['body_morpher']).to(DEV)
    pose = synth.random_poses(2, seed=8)
    img = synth.synthetic_image(9, 2)
    with torch.no_grad():
        f = face(pose[:, :39].contiguous().to(DEV))
        fr = O.siren_face_morpher(student_sds['face_morpher'], pose[:, :39])
        assert G.err(f.cpu(), fr)[1] <= 2e-3
        b = body(img.to(DEV), pose.to(DEV))
        br = O.siren_morpher_03(student_sds['body_morpher'], img, pose)
        _check_student('siren body standalone', b + [f], br + [fr])


def test_student_tcgen05_and_mma_paths_agree(lambda00_sds):
    """The student runs on TMA + wgmma by default (siren_tc.cu); the mma.sync kernels (siren.cu, option
    "siren_tc" = 0) are the same math in the same precision class (fp16 operands, fp32 accumulate): both must satisfy the
    student tolerances against the oracle and agree with each other."""
    poser = mode_14.create_poser(DEV, state_dicts=lambda00_sds)
    img = image_io.load_rgba_png(os.path.join(os.path.dirname(__file__), 'golden', 'data', 'lambda_00.png'))
    poses = synth.random_poses(3, seed=31)
    imgs = img.unsqueeze(0).expand(3, -1, -1, -1).contiguous()
    ctx = poser.get_context()
    with torch.no_grad():
        refs = O.mode_14_outputs(lambda00_sds, imgs, poses)
        outs = {}
        for flag in (1, 0):
            ctx.set_option('siren_tc', flag)
            outs[flag] = [t.cpu() for t in poser.get_posing_outputs(imgs.to(DEV), poses.to(DEV))]
            _check_student('mode_14 siren_tc=%d' % flag, outs[flag], refs)
        ctx.set_option('siren_tc', 1)
    for i, (a, b) in enumerate(zip(outs[1], outs[0])):
        assert G.err(a, b)[1] <= 2e-3, (i, G.err(a, b))


def test_student_fp16_io(lambda00_sds):
    """BASELINE configs[2] "fp16 I/O + fp32 accumulate": a float16 image selects tha4_student_forward_io(io_dtype = 1).
    Outputs are float16 and equal the fp32-I/O outputs up to one fp16 rounding of the image and of each result
    (values in [-1, 1]: half an ulp = 2.5e-4; the image rounding moves warped pixels by at most the same)."""
    poser = mode_14.create_poser(DEV, state_dicts=lambda00_sds)
    img = image_io.load_rgba_png(os.path.join(os.path.dirname(__file__), 'golden', 'data', 'lambda_00.png'))
    poses = synth.random_poses(3, seed=32)
    imgs = img.unsqueeze(0).expand(3, -1, -1, -1).contiguous()
    with torch.no_grad():
        refs = O.mode_14_outputs(lambda00_sds, imgs, poses)
        full = [t.cpu() for t in poser.get_posing_outputs(imgs.to(DEV), poses.to(DEV))]
        half = poser.get_posing_outputs(imgs.to(DEV).half(), poses.to(DEV))
    assert all(t.dtype == torch.float16 for t in half)
    half = [t.float().cpu() for t in half]
    _check_student('mode_14 fp16 I/O', half, refs)
    for i, (a, b) in enumerate(zip(half, full)):
        assert a.shape == b.shape
        assert G.err(a, b)[0] <= 1.5e-3 and G.err(a, b)[1] <= 2e-4, (i, G.err(a, b))


def test_default_mode_error_class_vs_torch_cuda_tf32(teacher_poser, teacher_sds):
    """Context for the default-mode tolerance: the reference's own CUDA path (cuDNN convolutions with TF32 allowed, PyTorch's
    default) deviates from the CPU fp32 result by a comparable amount on these random-init (chaotic) networks.  Both
    deviations are printed; ours must stay under the default-mode tolerance and within 3x of torch-CUDA's."""
    _set_strict(teacher_poser, 0)
    img = synth.synthetic_image(0, 1)[0]
    sds_dev = {k: {kk: vv.to(DEV) for kk, vv in v.items()} for k, v in teacher_sds.items()}
    orig_grid, orig_t0 = O.base_grid, O._timestep_embedding_zero
    O.base_grid = lambda n, h, w, dtype=torch.float32: orig_grid(n, h, w, dtype).to(DEV)
    O._timestep_embedding_zero = lambda n, c: orig_t0(n, c).to(DEV)
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    try:
        worst_ours, worst_torch = 0.0, 0.0
        for seed in (99, 7):
            pose = synth.random_poses(1, seed=seed)[0]
            with torch.no_grad():
                ours = teacher_poser.get_posing_outputs(img.to(DEV), pose.to(DEV))
                tcu = O.mode_07_outputs(sds_dev, img.to(DEV).unsqueeze(0), pose.to(DEV).unsqueeze(0))
            O.base_grid, O._timestep_embedding_zero = orig_grid, orig_t0
            with torch.no_grad():
                refs = O.mode_07_outputs(teacher_sds, img, pose)
            O.base_grid = lambda n, h, w, dtype=torch.float32: orig_grid(n, h, w, dtype).to(DEV)
            O._timestep_embedding_zero = lambda n, c: orig_t0(n, c).to(DEV)
            e_ours = max((a.cpu() - b).abs().mean().item() for a, b in zip(ours, refs))
            e_torch = max((a.cpu() - b).abs().mean().item() for a, b in zip(tcu, refs))
            print('\nseed %d: worst mean-abs deviation from CPU fp32: tha4_b200 default %.3e | torch CUDA (TF32 convs) %.3e' % (seed, e_ours, e_torch))
            worst_ours, worst_torch = max(worst_ours, e_ours), max(worst_torch, e_torch)
        assert worst_ours <= DEFAULT_MEAN_TOL and worst_ours <= max(3.0 * worst_torch, 5e-4), (worst_ours, worst_torch)
    finally:
        O.base_grid, O._timestep_embedding_zero = orig_grid, orig_t0
        torch.backends.cudnn.allow_tf32 = prev
        _set_strict(teacher_poser, 1)
