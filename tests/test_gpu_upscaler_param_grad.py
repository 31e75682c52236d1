"""Parameter gradients of the upscaler (Upscaler02) on the H100 (-m gpu): a trainable_(True) module against CPU autograd through
the fp32 oracle (oracle.tha4_oracle.upscaler_02, every state_dict tensor a leaf -- the oracle builds the time embedding and the
cond0 FiLM from the state_dict, so they get reference gradients too) at B = 1 with the coarse inputs at 256 (the CPU side
upsamples with F.interpolate) and 512, the flat d_params layout of the C ABI, micro-batching, training through Adam, and
mode_07 with a trainable upscaler and with all five teachers trainable.  Bounds as for the other trainable teachers
(DESIGN.md section 4)."""
import pytest
import torch
import torch.nn.functional as F

from oracle import synth, tha4_oracle as O
from test_gpu_upscaler_input_grad import DEV, _backward, _inputs, _load, _up512, _ups
from tha4_b200.poser.modes import mode_07

pytestmark = pytest.mark.gpu
NAN = float('nan')
STRICT_REL, STRICT_COS, STRICT_TENSOR_REL = 1e-2, 0.9999, 5e-2
DEFAULT_REL, DEFAULT_COS = 0.2, 0.98
N_PARAMS = 35015655
# Biases whose exact gradient is zero: each is added per channel in front of a GroupNorm(32) on 32 channels (one channel per
# group), whose mean removes it -- conv0 of the 32-channel blocks (norm1 follows) and the last up block's conv1 and skip
# (last.0 follows).  Both sides hold rounding noise there (the CPU's at most 2e-9 of the flat gradient's norm), so these are
# held to an absolute bound instead of a relative one.
ZERO_GRAD = ('body.down_blocks.0.res_blocks.0.conv0.bias', 'body.down_blocks.0.downsample.conv0.bias',
             'body.up_blocks.5.resnet_blocks.0.conv0.bias', 'body.up_blocks.5.resnet_blocks.1.conv0.bias',
             'body.up_blocks.5.resnet_blocks.1.conv1.bias', 'body.up_blocks.5.resnet_blocks.1.skip.bias')
ZERO_ABS = 1e-7              # x the norm of the flat reference gradient
POSER_NETS = ('eyebrow_decomposer', 'eyebrow_morphing_combiner', 'face_morpher', 'body_morpher', 'upscaler')


def _flat(d, keys):
    return torch.cat([d[k].double().reshape(-1) for k in keys])


def _gpu_param_grads(m, inputs, ups, want_inputs=False):
    m.zero_grad(set_to_none=True)
    ts = [t.to(DEV).clone().requires_grad_(want_inputs) for t in inputs]
    _backward(m(*ts), ups)
    return {k: q.grad.detach().cpu().clone() for k, q in m.named_parameters()}, [t.grad for t in ts]


def _cpu_param_grads(sd, inputs, ups):
    leaf = {k: v.clone().requires_grad_() for k, v in sd.items()}
    _backward(O.upscaler_02(leaf, inputs[0], _up512(inputs[1]), _up512(inputs[2]), inputs[3]), ups)
    return {k: v.grad if v.grad is not None else torch.zeros_like(v) for k, v in leaf.items()}


def _per_tensor(got, ref, keys, ref_norm):
    """(worst relative error over the tensors with a nonzero gradient, tensor), and the largest norm on either side among
    the ZERO_GRAD tensors relative to ref_norm"""
    worst = max([(((got[k].double().reshape(-1) - ref[k].double().reshape(-1)).norm() / ref[k].double().norm().clamp_min(1e-30)).item(), k)
                 for k in keys if k not in ZERO_GRAD] + [(0.0, '')])
    zero = max([max(got[k].double().norm().item(), ref[k].double().norm().item()) / ref_norm for k in keys if k in ZERO_GRAD] + [0.0])
    return worst, zero


def _compare(name, got, ref, keys):
    a, b = _flat(got, keys), _flat(ref, keys)
    rel = ((a - b).norm() / b.norm()).item()
    cos = F.cosine_similarity(a, b, dim=0).item()
    worst, zero = _per_tensor(got, ref, keys, b.norm().item())
    print('\n%s: flat rel L2 %.3e cosine %.6f, worst tensor %s rel %.3e, zero-gradient biases %.1e of the flat norm'
          % (name, rel, cos, worst[1], worst[0], zero))
    return a, rel, cos, worst, zero


@pytest.fixture(scope='module', params=[256, 512])
def cpu_param_ref(request, teacher_sds):
    inputs = _inputs(1, request.param)
    ups = _ups(1, 11)
    return inputs, ups, _cpu_param_grads(teacher_sds['upscaler'], inputs, ups)


@pytest.mark.parametrize('strict', [1, 0])
def test_param_grads_match_cpu_autograd(teacher_sds, cpu_param_ref, strict):
    inputs, ups, ref = cpu_param_ref
    size = inputs[1].shape[-1]
    m = _load(teacher_sds['upscaler']).trainable_(True)
    m.context().set_option('strict', strict)
    try:
        got, _ = _gpu_param_grads(m, inputs, ups)
        keys = list(m.state_dict().keys())
        assert len(keys) == 466 and set(keys) == set(ref) and keys[-2:] == ['coarse_image_conv.weight', 'coarse_image_conv.bias']
        a, rel, cos, worst, zero = _compare('Upscaler02 coarse %d strict=%d' % (size, strict), got, ref, keys)
        if strict:
            assert rel <= STRICT_REL and cos >= STRICT_COS, (rel, cos)
            assert worst[0] <= STRICT_TENSOR_REL and zero <= ZERO_ABS, (worst, zero)
        else:
            assert rel <= DEFAULT_REL and cos >= DEFAULT_COS, (rel, cos)
            # parameters alone equal parameters requested together with the inputs (one call computes both)
            both, gin = _gpu_param_grads(m, inputs, ups, want_inputs=True)
            assert all(g is not None for g in gin)
            assert ((_flat(both, keys) - a).norm() / a.norm()).item() <= 1e-6
            # no f16 staging of gradients: they scale exactly with the upstream gradient at 2^+-24
            for sc in (2.0 ** 24, 2.0 ** -24):
                s, _ = _gpu_param_grads(m, inputs, [u * sc if u is not None else None for u in ups])
                assert torch.equal(_flat(s, keys) / sc, a), sc
    finally:
        m.context().set_option('strict', 0)


def test_flat_buffer_every_slot_written_guard_untouched_and_deterministic(teacher_sds):
    m = _load(teacher_sds['upscaler'])
    ctx = m.sync_weights()
    n = ctx.param_count('upscaler')
    assert n == N_PARAMS == sum(p.numel() for p in m.parameters())
    inputs = [t.to(DEV) for t in _inputs(1, 256)]
    ups = [u.to(DEV) if u is not None else None for u in _ups(1, 3)]
    buf = torch.full((n + 64,), NAN, device=DEV)
    flat = buf[:n]
    ctx.upscaler_backward(*inputs, ups, d_params=flat)
    torch.cuda.synchronize()
    assert not torch.isnan(flat).any().item()
    assert torch.isnan(buf[n:]).all().item()
    again = torch.full_like(flat, NAN)
    ctx.upscaler_backward(*inputs, ups, d_params=again)
    assert torch.equal(again, flat)


def test_batching_accumulates_chunks(teacher_sds):
    m = _load(teacher_sds['upscaler']).trainable_()
    B = 3
    inputs = _inputs(B, 256, seed=2)
    ups = _ups(B, 9)
    keys = list(m.state_dict().keys())
    m.context().set_option('strict', 1)
    try:
        m.context().set_option('microbatch', 2)
        whole, _ = _gpu_param_grads(m, inputs, ups)
        m.context().set_option('microbatch', 32)
        acc = None
        for n in range(B):
            g, _ = _gpu_param_grads(m, [t[n:n + 1] for t in inputs], [u[n:n + 1] if u is not None else None for u in ups])
            acc = _flat(g, keys) if acc is None else acc + _flat(g, keys)
        rel = ((_flat(whole, keys) - acc).norm() / acc.norm()).item()
        # per tensor, so that a small tensor accumulated wrongly across chunks (time_embed, cond0) cannot hide in the total
        split = dict(zip(keys, acc.split([whole[k].numel() for k in keys])))
        worst, zero = _per_tensor(whole, split, keys, acc.norm().item())
        print('\nB=3 in chunks of 2 vs the sum of single samples: rel %.3e, worst tensor %s %.3e, zero-gradient biases %.1e'
              % (rel, worst[1], worst[0], zero))
        assert rel <= 1e-2 and worst[0] <= 2e-2 and zero <= ZERO_ABS, (rel, worst, zero)
    finally:
        m.context().set_option('microbatch', 32)
        m.context().set_option('strict', 0)


def test_zero_coarse_image_conv_gets_the_cpu_gradient(teacher_sds):
    """The reference initialises coarse_image_conv to zero; its gradient does not depend on its value, and must arrive."""
    sd = dict(teacher_sds['upscaler'])
    for k in ('coarse_image_conv.weight', 'coarse_image_conv.bias'):
        sd[k] = torch.zeros_like(sd[k])
    inputs = _inputs(1, 256, seed=5)
    ups = _ups(1, 13)
    ref = _cpu_param_grads(sd, inputs, ups)
    m = _load(sd).trainable_()
    m.context().set_option('strict', 1)
    try:
        got, _ = _gpu_param_grads(m, inputs, ups)
    finally:
        m.context().set_option('strict', 0)
    keys = ['coarse_image_conv.weight', 'coarse_image_conv.bias']
    _, rel, cos, worst, _ = _compare('zero coarse_image_conv (strict)', got, ref, keys)
    assert ref['coarse_image_conv.weight'].abs().max() > 0
    assert rel <= STRICT_REL and cos >= STRICT_COS and worst[0] <= STRICT_TENSOR_REL, (rel, cos, worst)


def test_adam_step_equals_a_fresh_module_and_finetune_lowers_the_loss(teacher_sds):
    sd = teacher_sds['upscaler']
    m = _load(sd).trainable_()
    inputs = [t.to(DEV) for t in _inputs(1, 256, seed=4)]
    # target: the outputs of a weight-perturbed copy
    g = torch.Generator().manual_seed(7)
    target_sd = {k: v + 0.02 * v.std().clamp_min(1e-3) * torch.randn(v.shape, generator=g) if v.dim() > 1 else v for k, v in sd.items()}
    with torch.no_grad():
        target = [o.clone() for o in _load(target_sd)(*inputs)]
    opt = torch.optim.Adam(m.parameters(), lr=1e-5)

    def loss_of(outs):
        return sum((o - t).abs().mean() for o, t in zip(outs, target))

    losses = []
    for step in range(12):
        opt.zero_grad(set_to_none=True)
        loss = loss_of(m(*inputs))
        loss.backward()
        opt.step()
        losses.append(loss.item())
        if step == 0:       # after one step: a freshly built module from the stepped state_dict computes the same outputs
            fresh = _load({k: v.detach().cpu() for k, v in m.state_dict().items()})
            with torch.no_grad():
                a, b = m(*inputs), fresh(*inputs)
            assert all(torch.equal(x, y) for x, y in zip(a, b))
    print('\nUpscaler02 Adam fine-tune L1: %.4e -> %.4e' % (losses[0], losses[-1]))
    assert losses[-1] < 0.9 * losses[0], losses


def _poser_and_inputs(teacher_sds):
    poser = mode_07.create_poser(DEV, state_dicts={k: teacher_sds[k] for k in POSER_NETS})
    image, pose = synth.synthetic_image(2, 1).to(DEV), synth.random_poses(1, seed=8).to(DEV)
    for _ in range(2):          # warm the eyebrow cache and the captured graph of the inference call
        with torch.no_grad():
            single = [o.clone() for o in poser.get_posing_outputs(image, pose)]
    return poser, image, pose, single


def test_mode_07_with_a_trainable_upscaler(teacher_sds):
    """mode_07 with only its upscaler trainable and plain inputs takes the composed path: the outputs equal the single call's
    bitwise, and only the upscaler's parameters get .grad."""
    poser, image, pose, single = _poser_and_inputs(teacher_sds)
    mods = poser.get_modules()
    up = mods['upscaler'].trainable_()
    outs = poser.get_posing_outputs(image, pose)
    assert outs[0].grad_fn is not None
    assert all(torch.equal(a, b) for a, b in zip(outs, single))
    outs[0].abs().mean().backward()
    assert all(p.grad is not None for p in up.parameters())
    for k in POSER_NETS:
        if k != 'upscaler':
            assert all(p.grad is None for p in mods[k].parameters()), k


def test_mode_07_with_all_five_teachers_trainable(teacher_sds):
    """Every parameter of every module of mode_07 gets .grad from a loss on the final frame, and after an Adam step over all
    of them the plain call equals a fresh poser built from the stepped state_dicts."""
    poser, image, pose, single = _poser_and_inputs(teacher_sds)
    mods = poser.get_modules()
    for k in POSER_NETS:
        mods[k].trainable_()
    params = [p for k in POSER_NETS for p in mods[k].parameters()]
    opt = torch.optim.Adam(params, lr=1e-4)
    outs = poser.get_posing_outputs(image, pose)
    assert all(torch.equal(a, b) for a, b in zip(outs, single))
    outs[0].abs().mean().backward()
    for k in POSER_NETS:
        missing = [n for n, p in mods[k].named_parameters() if p.grad is None]
        assert not missing, (k, missing[:3])
    opt.step()
    with torch.no_grad():
        after = [o.clone() for o in poser.get_posing_outputs(image, pose)]
    sds = {k: {n: v.detach().cpu() for n, v in mods[k].state_dict().items()} for k in POSER_NETS}
    fresh = mode_07.create_poser(DEV, state_dicts=sds)
    with torch.no_grad():
        ref = fresh.get_posing_outputs(image, pose)
    assert not all(torch.equal(a, b) for a, b in zip(after, single))
    assert all(torch.equal(a, b) for a, b in zip(after, ref))
