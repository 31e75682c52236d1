"""Algebraic identities between the U-Nets' parameter gradients (-m gpu), in both precision modes: the body morpher
(Morpher00) and the upscaler (Upscaler02) at B = 1.

The network checks against CPU autograd hold the default mode only to a flat relative L2 error and a cosine, which the
conv weights dominate; a wrong offset or factor in the glue around the small reductions would not move them.  The
relations below follow from how the backward forms those gradients (unet_backward.cu: gn_bwd_finalize_kernel,
gn_param_fold_kernel, linear_wgrad_kernel, the bias sums) and hold for whatever gradients the backward propagated, so f16
tape noise does not enter them:

  * a conv bias shared by two convs gets the same sum twice: <block>.skip.bias == <block>.conv1.bias, and the upscaler's
    coarse_image_conv.bias == body.first_conv.bias, bitwise;
  * at B = 1 a dense layer's weight gradient is an outer product, W.grad = outer(b.grad, u), u the layer's input as the
    forward applied it: SiLU(c2) for every cond1_layers.1, SiLU(t2) for every cond0_layers.1, SiLU(c1) for cond_embed.2,
    the pose for cond_embed.0, SiLU(t1) for time_embed.3, t0 for time_embed.1;
  * per channel c of a ResBlock's norm1 (C channels) with S1 = cond1_layers.1.bias.grad[C + c] (the sum of dz):
      norm1.bias.grad[c]              = (1 + s0)(1 + s1) S1,
      cond0_layers.1.bias.grad[C + c] = (1 + s1) S1,
      cond0_layers.1.bias.grad[c]     = (1 + s1) (cond1_layers.1.bias.grad[c] - b0 S1) / (1 + s0),
    with (s0, b0) the block's time FiLM at t = 0 and (s1, b1) its pose FiLM.

The FiLM vectors and MLP activations are recomputed here in fp64 from the state_dict and the pose (the arithmetic of
oracle.tha4_oracle.unet), each with a bound on how far the GPU's fp32 values can be from them (see _linear).  The bound of
each relation follows from those and from the fp32 roundings of the gradients involved; it is derived, not fitted."""
import pytest
import torch
import torch.nn.functional as F

import test_gpu_body_morpher_input_grad as BM
import test_gpu_upscaler_input_grad as UP

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
U = 2.0 ** -24
TINY = 2.0 ** -126        # below the smallest normal fp32 the roundings are absolute, not relative


def _silu(x, ex):
    """SiLU in fp64 and the bound on the GPU's fp32 value: |SiLU'| <= 1.1 carries the input's error, and v / (1 + expf(-v))
    adds a few ulps (8 u) of the result."""
    y = F.silu(x)
    return y, 1.1 * ex + 8 * U * y.abs() + TINY


def _linear(sd, key, x, ex, silu_in):
    """y = b + W u(x) in fp64 and the bound on the GPU's fp32 linear_kernel: the input's error through |W|, plus the fp32
    sum of I products and the bias in any order, (I + 2) u of the absolute terms (the standard gamma_n bound)."""
    W, b = sd[key + '.weight'].double(), sd[key + '.bias'].double()
    v, ev = _silu(x, ex) if silu_in else (x, ex)
    y = v @ W.t() + b
    ey = ev @ W.abs().t() + (W.shape[1] + 2) * U * (v.abs() @ W.abs().t() + b.abs()) + TINY
    return y, ey


def _film(sd, pose, mc):
    """fp64 activations of the time and pose MLPs and every ResBlock's FiLM, each as (value, bound on the GPU's error)."""
    p = 'body.'
    z = torch.zeros(1, mc, dtype=torch.float64)
    t0 = torch.cat([torch.ones(1, mc // 2), torch.zeros(1, mc - mc // 2)], 1).double()
    t1 = _linear(sd, p + 'time_embed.1', t0, z, False)
    t2 = _linear(sd, p + 'time_embed.3', *t1, True)
    pz = torch.zeros_like(pose, dtype=torch.float64)
    c1 = _linear(sd, p + 'cond_embed.0', pose.double(), pz, False)
    c2 = _linear(sd, p + 'cond_embed.2', *c1, True)
    blocks = sorted({k[:-len('.cond1_layers.1.weight')] for k in sd if k.endswith('.cond1_layers.1.weight')})
    film = {b: (_linear(sd, b + '.cond0_layers.1', *t2, True), _linear(sd, b + '.cond1_layers.1', *c2, True)) for b in blocks}
    return dict(t0=(t0, z), t1=t1, t2=t2, c1=c1, c2=c2, pose=(pose.double(), pz)), film


def _module_grads(net, sd, strict):
    if net == 'body_morpher':
        m = BM._load(sd)
        img, pose = BM._inputs(1, seed=5)
        inputs, ups = [img, pose], BM._ups(1, 13)
    else:
        m = UP._load(sd)
        inputs, ups = UP._inputs(1, 256, seed=5), UP._ups(1, 13)
        pose = inputs[3]
    m.trainable_(True)
    m.context().set_option('strict', strict)
    try:
        m.zero_grad(set_to_none=True)
        BM._backward(m(*[t.to(DEV) for t in inputs]), ups)
        grads = {k: q.grad.detach().cpu().double() for k, q in m.named_parameters()}
    finally:
        m.context().set_option('strict', 0)
    return grads, pose


def _check(name, got, ref, bound):
    err = (got - ref).abs()
    r = (err / bound).max().item()
    assert torch.isfinite(got).all(), name
    return r


@pytest.mark.parametrize('net', ['body_morpher', 'upscaler'])
@pytest.mark.parametrize('strict', [0, 1])
def test_unet_param_identities(teacher_sds, net, strict):
    sd = teacher_sds[net]
    mc = sd['body.first_conv.weight'].shape[0]
    g, pose = _module_grads(net, sd, strict)
    act, film = _film(sd, pose, mc)
    worst = {}

    def note(group, r, what):
        assert r <= 1.0, (net, strict, group, what, r)
        worst[group] = max(worst.get(group, (0.0, '')), (r, what))

    # shared biases: the same fixed-order sum written to two slots
    pairs = [(k[:-len('.skip.bias')] + '.skip.bias', k[:-len('.skip.bias')] + '.conv1.bias') for k in g if k.endswith('.skip.bias')]
    if net == 'upscaler':
        pairs.append(('coarse_image_conv.bias', 'body.first_conv.bias'))
    assert len(pairs) >= 5
    for a, b in pairs:
        assert torch.equal(g[a], g[b]), (net, strict, a, b)

    # outer products at B = 1: dW = fl(dy u32), db = fl(dy), |u32 - u| <= e_u, so
    # |dW - db u| <= |db| (e_u + 4 u (|u| + e_u)) (the roundings of dW and db, and dy vs db, one u each with slack)
    sites = [('body.cond_embed.2', 'c1', True), ('body.cond_embed.0', 'pose', False),
             ('body.time_embed.3', 't1', True), ('body.time_embed.1', 't0', False)]
    sites += [(b + '.cond1_layers.1', 'c2', True) for b in film] + [(b + '.cond0_layers.1', 't2', True) for b in film]
    for key, src, silu in sites:
        u, eu = _silu(*act[src]) if silu else act[src]
        u, eu = u[0], eu[0]
        db = g[key + '.bias']
        ref = torch.outer(db, u)
        bound = torch.outer(db.abs(), eu + 4 * U * (u.abs() + eu)) + TINY
        note('outer products', _check(key, g[key + '.weight'], ref, bound), key)

    # FiLM folds, per block.  GPU side: S1g = fl(S1); d beta = fl(M S1) with M = (1 + s0)(1 + s1) of the GPU's fp32 FiLM
    # (formed in fp64); d b0 = fl((1 + s1) S1); D1 = cond1_layers.1.bias.grad[c] = fl(X s0f + b0 S1) with s0f = fl32(1 + s0)
    # and d s0 = fl((1 + s1) X).  Each relation's bound: the fp64 FiLM's distance from the GPU's (e_s0, e_s1, e_b0) times
    # the magnitudes it multiplies, plus u per rounding (3 u with slack), doubled to cover the second-order terms.
    for b, ((f0, ef0), (f1, ef1)) in film.items():
        C = f0.shape[1] // 2
        s0, b0, es0, eb0 = 1 + f0[0, :C], f0[0, C:], ef0[0, :C], ef0[0, C:]
        s1, es1 = 1 + f1[0, :C], ef1[0, :C]
        d1 = g[b + '.cond1_layers.1.bias']
        D1, S1 = d1[:C], d1[C:]
        aS1 = S1.abs()
        M = s0 * s1
        bound = 2 * (aS1 * (s1.abs() * es0 + s0.abs() * es1 + es0 * es1) + 3 * U * (M * S1).abs()) + TINY
        note('d beta = (1 + s0)(1 + s1) S1', _check(b, g[b + '.norm1.bias'], M * S1, bound), b)
        d0 = g[b + '.cond0_layers.1.bias']
        bound = 2 * (aS1 * es1 + 3 * U * (s1 * S1).abs()) + TINY
        note('d b0 = (1 + s1) S1', _check(b, d0[C:], s1 * S1, bound), b)
        num = D1 - b0 * S1
        e_num = 2 * U * D1.abs() + (eb0 + 2 * U * b0.abs()) * aS1
        X = num / s0
        eX = e_num / s0.abs() + X.abs() * (es0 + U * s0.abs()) / s0.abs()
        bound = 2 * (s1.abs() * eX + es1 * (X.abs() + eX) + 2 * U * (s1 * X).abs()) + TINY
        note('d s0 = (1 + s1)(D1 - b0 S1) / (1 + s0)', _check(b, d0[:C], s1 * X, bound), b)
    print('\n%s strict %d: worst |err| / bound per relation:' % (net, strict))
    for k, (r, what) in worst.items():
        print('  %-42s %.3e (%s)' % (k, r, what))
