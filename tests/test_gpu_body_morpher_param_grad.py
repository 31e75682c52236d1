"""Parameter gradients of the body morpher (Morpher00) on the H100 (-m gpu): a trainable_(True) module against CPU autograd
through the fp32 oracle (oracle.tha4_oracle.morpher_00, every state_dict tensor a leaf -- the oracle builds the time
embedding and the cond0 FiLM from the state_dict, so they get reference gradients too), the flat d_params layout of the
C ABI, micro-batching, and training through Adam.  Bounds as for the face teachers (DESIGN.md section 4)."""
import pytest
import torch
import torch.nn.functional as F

from oracle import synth, tha4_oracle as O
from test_gpu_body_morpher_input_grad import DEV, _backward, _inputs, _load, _ups
from tha4_b200.poser.modes import mode_07

pytestmark = pytest.mark.gpu
NAN = float('nan')
STRICT_REL, STRICT_COS, STRICT_TENSOR_REL = 1e-2, 0.9999, 5e-2
DEFAULT_REL, DEFAULT_COS = 0.2, 0.98


def _flat(d, keys):
    return torch.cat([d[k].double().reshape(-1) for k in keys])


def _gpu_param_grads(m, img, pose, ups, want_inputs=False):
    m.zero_grad(set_to_none=True)
    i = img.to(DEV).clone().requires_grad_(want_inputs)
    p = pose.to(DEV).clone().requires_grad_(want_inputs)
    _backward(m(i, p), ups)
    return {k: q.grad.detach().cpu().clone() for k, q in m.named_parameters()}, [i.grad, p.grad]


@pytest.fixture(scope='module')
def cpu_param_ref(teacher_sds):
    sd = teacher_sds['body_morpher']
    img, pose = _inputs(2)
    ups = _ups(2, 11)
    leaf = {k: v.clone().requires_grad_() for k, v in sd.items()}
    _backward(O.morpher_00(leaf, img, pose), ups)
    return img, pose, ups, {k: v.grad if v.grad is not None else torch.zeros_like(v) for k, v in leaf.items()}


@pytest.mark.parametrize('strict', [1, 0])
def test_param_grads_match_cpu_autograd(teacher_sds, cpu_param_ref, strict):
    img, pose, ups, ref = cpu_param_ref
    m = _load(teacher_sds['body_morpher']).trainable_(True)
    m.context().set_option('strict', strict)
    try:
        got, _ = _gpu_param_grads(m, img, pose, ups)
        keys = list(m.state_dict().keys())
        assert len(keys) == 398 and set(keys) == set(ref)
        a, b = _flat(got, keys), _flat(ref, keys)
        rel = ((a - b).norm() / b.norm()).item()
        cos = F.cosine_similarity(a, b, dim=0).item()
        worst = max((((got[k].double() - ref[k].double()).norm() / ref[k].double().norm().clamp_min(1e-30)).item(), k) for k in keys)
        print('\nMorpher00 strict=%d: flat rel L2 %.3e cosine %.6f, worst tensor %s rel %.3e' % (strict, rel, cos, worst[1], worst[0]))
        if strict:
            assert rel <= STRICT_REL and cos >= STRICT_COS, (rel, cos)
            assert worst[0] <= STRICT_TENSOR_REL, worst
        else:
            assert rel <= DEFAULT_REL and cos >= DEFAULT_COS, (rel, cos)
            # parameters alone equal parameters requested together with the inputs (one call computes both)
            both, gin = _gpu_param_grads(m, img, pose, ups, want_inputs=True)
            assert all(g is not None for g in gin)
            assert ((_flat(both, keys) - a).norm() / a.norm()).item() <= 1e-6
            # no f16 staging of gradients: they scale exactly with the upstream gradient at 2^+-24
            for sc in (2.0 ** 24, 2.0 ** -24):
                s, _ = _gpu_param_grads(m, img, pose, [u * sc if u is not None else None for u in ups])
                assert torch.equal(_flat(s, keys) / sc, a), sc
    finally:
        m.context().set_option('strict', 0)


def test_flat_buffer_every_slot_written_guard_untouched_and_deterministic(teacher_sds):
    m = _load(teacher_sds['body_morpher'])
    ctx = m.sync_weights()
    n = ctx.param_count('body_morpher')
    assert n == 34682119 == sum(p.numel() for p in m.parameters())
    img, pose = [t.to(DEV) for t in _inputs(2)]
    ups = [u.to(DEV) if u is not None else None for u in _ups(2, 3)]
    buf = torch.full((n + 64,), NAN, device=DEV)
    flat = buf[:n]
    ctx.morpher_backward(img, pose, ups, d_params=flat)
    torch.cuda.synchronize()
    assert not torch.isnan(flat).any().item()
    assert torch.isnan(buf[n:]).all().item()
    again = torch.full_like(flat, NAN)
    ctx.morpher_backward(img, pose, ups, d_params=again)
    assert torch.equal(again, flat)


def test_batching_accumulates_chunks(teacher_sds):
    m = _load(teacher_sds['body_morpher']).trainable_()
    img, pose = _inputs(5, seed=2)
    ups = _ups(5, 9)
    keys = list(m.state_dict().keys())
    m.context().set_option('strict', 1)
    try:
        m.context().set_option('microbatch', 2)
        whole, _ = _gpu_param_grads(m, img, pose, ups)
        m.context().set_option('microbatch', 32)
        acc = None
        for n in range(5):
            g, _ = _gpu_param_grads(m, img[n:n + 1], pose[n:n + 1], [u[n:n + 1] if u is not None else None for u in ups])
            acc = _flat(g, keys) if acc is None else acc + _flat(g, keys)
        rel = ((_flat(whole, keys) - acc).norm() / acc.norm()).item()
        # per tensor, so that a small tensor accumulated wrongly across chunks (time_embed, cond0) cannot hide in the total
        worst, off = (0.0, ""), 0
        for k in keys:
            n = whole[k].numel()
            ref = acc[off:off + n]
            r = ((whole[k].double().reshape(-1) - ref).norm() / ref.norm().clamp_min(1e-30)).item()
            worst = max(worst, (r, k))
            off += n
        print('\nB=5 in chunks of 2 vs the sum of single samples: rel %.3e, worst tensor %s %.3e' % (rel, worst[1], worst[0]))
        assert rel <= 1e-2 and worst[0] <= 2e-2, (rel, worst)
    finally:
        m.context().set_option('microbatch', 32)
        m.context().set_option('strict', 0)


def test_adam_step_equals_a_fresh_module_and_finetune_lowers_the_loss(teacher_sds):
    sd = teacher_sds['body_morpher']
    m = _load(sd).trainable_()
    img, pose = [t.to(DEV) for t in _inputs(2, seed=4)]
    # target: the outputs of a weight-perturbed copy
    g = torch.Generator().manual_seed(7)
    target_sd = {k: v + 0.02 * v.std().clamp_min(1e-3) * torch.randn(v.shape, generator=g) if v.dim() > 1 else v for k, v in sd.items()}
    with torch.no_grad():
        target = [o.clone() for o in _load(target_sd)(img, pose)]
    opt = torch.optim.Adam(m.parameters(), lr=1e-5)

    def loss_of(outs):
        return sum((o - t).abs().mean() for o, t in zip(outs, target))

    losses = []
    for step in range(12):
        opt.zero_grad(set_to_none=True)
        loss = loss_of(m(img, pose))
        loss.backward()
        opt.step()
        losses.append(loss.item())
        if step == 0:       # after one step: a freshly built module from the stepped state_dict computes the same outputs
            fresh = _load({k: v.detach().cpu() for k, v in m.state_dict().items()})
            with torch.no_grad():
                a, b = m(img, pose), fresh(img, pose)
            assert all(torch.equal(x, y) for x, y in zip(a, b))
    print('\nMorpher00 Adam fine-tune L1: %.4e -> %.4e' % (losses[0], losses[-1]))
    assert losses[-1] < 0.9 * losses[0], losses


POSER_NETS = ('eyebrow_decomposer', 'eyebrow_morphing_combiner', 'face_morpher', 'body_morpher', 'upscaler')


def test_mode_07_with_a_trainable_body_morpher(teacher_sds):
    """mode_07 with only its body morpher trainable and plain inputs takes the composed path: the outputs equal the single
    call's bitwise, the loss on the upscaler's output reaches the morpher through the upscaler's input gradients (every
    morpher parameter gets .grad, no other module's does), and after an Adam step the plain call equals a fresh poser built
    from the stepped weights."""
    poser = mode_07.create_poser(DEV, state_dicts={k: teacher_sds[k] for k in POSER_NETS})
    mods = poser.get_modules()
    image, pose = synth.synthetic_image(2, 1).to(DEV), synth.random_poses(1, seed=8).to(DEV)
    for _ in range(2):          # warm the eyebrow cache and the captured graph of the inference call
        with torch.no_grad():
            single = [o.clone() for o in poser.get_posing_outputs(image, pose)]
    body = mods['body_morpher'].trainable_()
    outs = poser.get_posing_outputs(image, pose)
    assert outs[0].grad_fn is not None
    assert all(torch.equal(a, b) for a, b in zip(outs, single))
    opt = torch.optim.Adam(body.parameters(), lr=1e-4)
    outs[0].abs().mean().backward()
    assert all(p.grad is not None for p in body.parameters())
    for k in POSER_NETS:
        if k != 'body_morpher':
            assert all(p.grad is None for p in mods[k].parameters()), k
    opt.step()
    with torch.no_grad():
        after = [o.clone() for o in poser.get_posing_outputs(image, pose)]
    sds = {k: teacher_sds[k] for k in POSER_NETS}
    sds['body_morpher'] = {n: v.detach().cpu() for n, v in body.state_dict().items()}
    fresh = mode_07.create_poser(DEV, state_dicts=sds)
    with torch.no_grad():
        ref = fresh.get_posing_outputs(image, pose)
    assert not all(torch.equal(a, b) for a, b in zip(after, single))
    assert all(torch.equal(a, b) for a, b in zip(after, ref))
