"""Kernel-level parity on the H100 (-m gpu): every CUDA kernel family against a plain fp32 PyTorch reference of the
same op (CPU), and the grid_sample / interpolate index math bit-exactly against the C oracle."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import synth, tha4_oracle as O
import gpu_util as G

pytestmark = pytest.mark.gpu


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ------------------------------------------------------------------------------------------ grid_sample / resize
@pytest.mark.parametrize('size,amp', [(128, 0.05), (192, 0.3), (256, 1.5), (512, 0.02)])
def test_grid_sample_bit_exact_vs_c_oracle(oracle_clib, size, amp):
    n = 2
    img = synth.synthetic_image(size, n)[:, :, :size, :size].contiguous()
    gc = torch.randn(n, 2, size, size, generator=_gen(size)) * amp
    out, x0, y0, tx, ty = G.grid_sample(img, gc)
    ro, rx0, ry0, rtx, rty = G.oracle_grid_sample(oracle_clib, img, gc)
    assert torch.equal(x0, rx0) and torch.equal(y0, ry0), 'integer corner indices must be bit-exact'
    assert torch.equal(tx, rtx) and torch.equal(ty, rty), 'lerp weights must be bit-exact'
    assert torch.equal(out, ro), 'sampled values follow the same op order as the oracle'
    ref = O.apply_grid_change(gc, img)
    assert G.err(out, ref)[0] < 2e-5


def test_grid_sample_adversarial_grids(oracle_clib):
    size, n = 128, 1
    img = synth.synthetic_image(5, n)[:, :, :size, :size].contiguous()
    cases = {
        'zero': torch.zeros(n, 2, size, size),
        'far_positive': torch.full((n, 2, size, size), 5.0),
        'far_negative': torch.full((n, 2, size, size), -5.0),
        'half_pixel': torch.full((n, 2, size, size), 1.0 / size),      # source index lands on .5 boundaries
        'one_pixel': torch.full((n, 2, size, size), 2.0 / size),       # exact integer shift
    }
    for name, gc in cases.items():
        out, x0, y0, tx, ty = G.grid_sample(img, gc)
        ro, rx0, ry0, rtx, rty = G.oracle_grid_sample(oracle_clib, img, gc)
        assert torch.equal(x0, rx0) and torch.equal(y0, ry0) and torch.equal(tx, rtx) and torch.equal(ty, rty), name
        assert torch.equal(out, ro), name
        assert G.err(out, O.apply_grid_change(gc, img))[0] < 2e-5, name
    out = G.grid_sample(img, cases['zero'])[0]
    assert G.err(out, img)[0] < 1e-5
    out = G.grid_sample(img, cases['far_positive'])[0]
    assert torch.equal(out, img[:, :, -1:, -1:].expand_as(out).contiguous())


@pytest.mark.parametrize('hi,ho', [(512, 256), (256, 512), (128, 256)])
def test_resize_bilinear_vs_oracle(oracle_clib, hi, ho):
    a = torch.rand(2, 4, hi, hi, generator=_gen(hi))
    out = G.resize(a, ho, ho)
    ref = torch.empty(2, 4, ho, ho)
    oracle_clib.tha4o_resize_bilinear(ctypes.c_void_p(a.data_ptr()), 2, 4, hi, hi, ho, ho, ctypes.c_void_p(ref.data_ptr()))
    assert torch.equal(out, ref)
    assert G.err(out, F.interpolate(a, size=(ho, ho), mode='bilinear', align_corners=False))[0] < 3e-7


# ------------------------------------------------------------------------------------------ convolution
def _conv_ref(kind, x, w, bias, in_up):
    if in_up:
        x = F.interpolate(x, scale_factor=2, mode='nearest')
    if kind == 0:
        return F.conv2d(x, w, bias, 1, 1)
    if kind == 1:
        return F.conv2d(x, w, bias, 2, 1)
    if kind == 2:
        return F.conv_transpose2d(x, w, bias, 2, 1)
    if kind == 4:
        return F.conv2d(F.interpolate(x, scale_factor=2, mode='nearest'), w, bias, 1, 1)
    return F.conv2d(x, w, bias)


CONV_CASES = [
    # kind, N, Cin, H, Cout, bias, res_mode, in_up, ksplit
    (0, 2, 4, 32, 64, False, 0, 0, 0),
    (0, 1, 8, 48, 64, False, 0, 0, 0),
    (0, 2, 64, 32, 64, True, 1, 0, 0),
    (0, 1, 96, 32, 32, True, 0, 0, 0),
    (0, 1, 524, 16, 512, False, 0, 0, 0),        # pose-concat bottleneck (Cin padded to 544), auto split-K
    (0, 1, 540, 24, 512, False, 0, 0, 3),
    (0, 2, 128, 16, 128, True, 2, 1, 0),         # up-sampling ResBlock: nearest x2 gather + upsampled residual
    (0, 2, 128, 16, 128, True, 3, 0, 0),         # down-sampling ResBlock residual: 2x2 mean
    (0, 1, 16, 64, 32, True, 0, 0, 0),
    (1, 2, 64, 64, 128, False, 0, 0, 0),
    (1, 1, 256, 32, 512, False, 0, 0, 0),
    (2, 1, 512, 16, 256, False, 0, 0, 0),
    (2, 2, 128, 24, 64, False, 0, 0, 0),
    (3, 2, 256, 16, 768, True, 0, 0, 0),
    (3, 1, 384, 32, 128, True, 1, 0, 0),
    (4, 2, 128, 16, 128, True, 2, 0, 0),         # phase-decomposed nearest-x2 + 3x3 (+ upsampled residual)
    (4, 1, 64, 24, 64, True, 0, 0, 0),
    (4, 1, 256, 16, 256, True, 0, 0, 4),
    (0, 1, 32, 64, 32, True, 0, 0, 0),           # f16 operands: 64-byte rows (Cin % 64 == 32)
    (0, 1, 160, 32, 64, True, 1, 0, 0),
    (0, 1, 528, 16, 512, False, 0, 0, 0),        # pose-concat bottleneck as the f16 path sees it (pose padded to 16)
    (0, 1, 544, 24, 512, False, 0, 0, 3),
    (3, 1, 512, 16, 1536, True, 0, 0, 0),        # attention qkv
    (0, 1, 32, 512, 32, True, 1, 0, 0),          # many tiles: several CTAs per SM
    (0, 2, 64, 256, 64, True, 1, 0, 0),
    (0, 3, 128, 200, 128, True, 0, 0, 0),        # streaming kernel with partial tiles in both directions
    (4, 1, 64, 128, 64, True, 2, 0, 0),          # 4 phases x 128 tiles
    (2, 1, 128, 128, 64, False, 0, 0, 0),
    (0, 1, 96, 384, 32, True, 0, 0, 0),
]


@pytest.mark.parametrize('case', CONV_CASES)
@pytest.mark.parametrize('path', ['strict_mma', 'tf32_tcgen05', 'f16_tcgen05', 'tf32_mma'])
def test_conv_vs_torch(case, path):
    """strict_mma: 3xTF32 mma.sync (== fp32); tf32_tcgen05: TMA + wgmma on tf32 operands where the configuration is
    supported (stride-1 taps, no fused upsample), else mma.sync; f16_tcgen05: the same kernel with f16 operands
    (kind::f16, 128- or 64-byte rows) where Cin % 8 == 0, as the networks run it behind a normalisation layer;
    tf32_mma: single-TF32 mma.sync everywhere."""
    strict = 1 if path == 'strict_mma' else 0
    G.ctx().set_option('tcgen05', 0 if path == 'tf32_mma' else 1)
    G.ctx().set_option('half_operands', 1 if path == 'f16_tcgen05' else 0)
    kind, N, Cin, H, Cout, has_bias, res_mode, in_up, ksplit = case
    g = _gen(hash(case) % 10000)
    k = {0: 3, 1: 4, 2: 4, 3: 1, 4: 3}[kind]
    x = torch.randn(N, Cin, H, H, generator=g)
    wshape = (Cin, Cout, k, k) if kind == 2 else (Cout, Cin, k, k)
    w = torch.randn(wshape, generator=g) / math.sqrt(Cin * k * k)
    bias = torch.randn(Cout, generator=g) if has_bias else None
    ref = _conv_ref(kind, x, w, bias, in_up)
    res = None
    if res_mode:
        Ho = ref.shape[2]
        rh = {1: Ho, 2: Ho // 2, 3: Ho * 2}[res_mode]
        res = torch.randn(N, Cout, rh, rh, generator=g)
        ref = ref + {1: res, 2: F.interpolate(res, scale_factor=2, mode='nearest'), 3: F.avg_pool2d(res, 2, 2)}[res_mode]
    out = G.conv(kind, x, w, bias, res, res_mode, in_up, strict, ksplit)
    mx, mean = G.err(out, ref)
    tol = (6e-5 if kind == 4 else 2e-5) if strict else 6e-3     # kind 4 pre-sums weights: (a+b)x vs ax+bx rounding          # 3xTF32 == fp32; single TF32: 2^-11 relative per product
    G.ctx().set_option('tcgen05', 1)
    G.ctx().set_option('half_operands', 1)
    assert mx < tol * max(1.0, ref.abs().max().item()), (case, path, mx, mean)


@pytest.mark.parametrize('wscale', [1e-6, 1e-4, 1.0, 300.0])
def test_conv_f16_weight_range(wscale):
    """The f16 operand copy of a layer's weights is normalised by a power of two (conv_tc.cu, conv_make_half): a layer whose
    weights all sit in f16's subnormal range (|w| < 6.1e-5), or beyond f16's maximum, must still convolve to TF32-class
    accuracy.  Weights span five orders of magnitude below the layer maximum."""
    G.ctx().set_option('tcgen05', 1)
    G.ctx().set_option('half_operands', 1)
    g = _gen(77)
    x = torch.randn(1, 64, 32, 32, generator=g)
    mag = 10.0 ** (-5.0 * torch.rand(64, 64, 3, 3, generator=g))                 # 1e-5 .. 1 of the maximum
    w = torch.randn(64, 64, 3, 3, generator=g).sign() * mag * wscale / math.sqrt(64 * 9)
    ref = F.conv2d(x, w, None, 1, 1)
    out = G.conv(0, x, w, None, None, 0, 0, 0, 0)
    mx, mean = G.err(out, ref)
    assert mx < 6e-3 * ref.abs().max().item(), (wscale, mx, ref.abs().max().item())


CONV_NORM_CASES = [
    # kind, N, Cin, norm_C, H, Cout, groups, act, film, bias, res_mode, ksplit
    (0, 2, 64, 64, 32, 64, 32, 2, True, True, 1, 0),          # U-Net ResBlock conv1: GroupNorm + FiLM + SiLU, residual
    (0, 1, 128, 128, 64, 128, 32, 2, False, True, 0, 0),      # conv0 of a same-resolution ResBlock
    (0, 1, 32, 32, 128, 32, 32, 2, True, True, 1, 0),         # 64-byte operand rows (Cin % 64 == 32), many tiles
    (0, 1, 96, 96, 48, 32, 32, 2, False, True, 0, 0),         # concat-sized input, partial tiles in both directions
    (0, 1, 512, 512, 16, 512, 0, 1, False, False, 0, 0),      # enc-dec bottleneck: InstanceNorm + ReLU, cluster split-K
    (0, 1, 528, 512, 16, 512, 0, 1, False, False, 0, 0),      # pose-concat bottleneck conv: 512 normalised + 16 pass-through channels
    (0, 2, 512, 512, 24, 512, 0, 1, False, False, 0, 3),      # workspace split-K
    (1, 1, 64, 64, 64, 128, 0, 1, False, False, 0, 0),        # 4x4 stride-2 (element-strided TMA boxes)
    (2, 1, 256, 256, 32, 128, 0, 1, False, False, 0, 0),      # transposed 4x4 stride-2 (4 phases)
    (4, 1, 128, 128, 32, 128, 32, 2, True, True, 2, 0),       # up-sampling ResBlock conv0 (phase-decomposed), upsampled residual
    (3, 2, 256, 256, 16, 768, 32, 0, False, True, 0, 0),      # attention: GroupNorm (no activation) -> 1x1 qkv
    (0, 1, 64, 64, 256, 64, 32, 2, True, True, 1, 0),          # single-chunk unsplit variant; residual tile by TMA, one staging slot reused
    (0, 1, 128, 128, 120, 128, 32, 2, True, True, 1, 0),       # 4 column steps over 3 staging slots, residual by TMA, partial tiles in x
]


@pytest.mark.parametrize('case', CONV_NORM_CASES)
@pytest.mark.parametrize('halo', [1, 0])
def test_conv_with_fused_input_norm(case, halo):
    """The default mode's conv: the pending normalisation (+FiLM, +activation) of the RAW f16 input is applied to the
    operand tiles in shared memory between TMA and wgmma.  Reference: conv(act(norm(x))) in fp32.  Tolerance:
    two f16 roundings of O(1) operands (raw value, normalised value) + tanh.approx SiLU, over a K-term dot product:
    6e-3 of the output's scale (same class as the separate-pass f16 path)."""
    kind, N, Cin, nC, H, Cout, groups, act, film, has_bias, res_mode, ksplit = case
    if kind != 0 and not halo:
        pytest.skip('only 3x3 stride-1 convs have two kernels')
    G.ctx().set_option('tcgen05', 1)
    G.ctx().set_option('halo_conv', halo)      # 1: conv_halo.cu (one halo box per chunk, transformed once); 0: conv_tc.cu (one box per tap)
    g = _gen(hash(case) % 10007)
    k = {0: 3, 1: 4, 2: 4, 3: 1, 4: 3}[kind]
    x = torch.randn(N, Cin, H, H, generator=g) * 1.7 + 0.4
    if nC < Cin:
        x[:, nC:] = torch.rand(N, Cin - nC, 1, 1, generator=g).expand(-1, -1, H, H)      # tiled pose planes: constant per channel
    gamma, beta = 1.0 + 0.3 * torch.randn(nC, generator=g), 0.3 * torch.randn(nC, generator=g)
    f0 = torch.randn(2 * nC, generator=g) * 0.3 if film else None
    f1 = torch.randn(N, 2 * nC, generator=g) * 0.3 if film else None
    wshape = (Cin, Cout, k, k) if kind == 2 else (Cout, Cin, k, k)
    w = torch.randn(wshape, generator=g) / math.sqrt(Cin * k * k)
    bias = torch.randn(Cout, generator=g) if has_bias else None
    xn = x[:, :nC]
    h = F.group_norm(xn, groups, gamma, beta, eps=1e-5) if groups else F.instance_norm(xn, weight=gamma, bias=beta, eps=1e-5)
    if film:
        h = O._scaleshift(O._scaleshift(h, f0.unsqueeze(0).expand(N, -1)), f1)
    h = {0: h, 1: F.relu(h), 2: F.silu(h)}[act]
    h = torch.cat([h, x[:, nC:]], dim=1)
    ref = _conv_ref(kind, h, w, bias, 0)
    res = None
    if res_mode:
        Ho = ref.shape[2]
        rh = {1: Ho, 2: Ho // 2, 3: Ho * 2}[res_mode]
        res = torch.randn(N, Cout, rh, rh, generator=g)
        ref = ref + {1: res, 2: F.interpolate(res, scale_factor=2, mode='nearest'), 3: F.avg_pool2d(res, 2, 2)}[res_mode]
    out, out16 = G.conv_norm(kind, x, nC, groups, gamma, beta, f0, f1, act, w, bias, res, res_mode, ksplit)
    G.ctx().set_option('halo_conv', 1)
    scale = max(1.0, ref.abs().max().item())
    mx, mean = G.err(out, ref)
    assert mx < 6e-3 * scale, (case, mx, mean)
    assert G.err(out16, out)[0] <= 1e-3 * scale, 'the f16 copy is the fp32 output rounded once'


# ------------------------------------------------------------------------------------------ normalisation
@pytest.mark.parametrize('C,H,groups,act,pool', [(64, 48, 0, 1, 0), (512, 16, 0, 0, 0), (32, 64, 32, 2, 0), (192, 16, 32, 2, 1), (384, 16, 32, 2, 0)])
def test_norm_default_mode_f16_output(C, H, groups, act, pool):
    """The normalisation variant the default (benchmarked) mode runs: f16 output tensor, fast-math SiLU (ex2.approx /
    rcp.approx).  Tolerance: f16 rounding of an O(1) value (2^-11 relative) + 2 ulp of fast math."""
    g = _gen(C * 3 + H)
    x = torch.randn(2, C, H, H, generator=g) * 2 - 0.5
    gamma, beta = torch.randn(C, generator=g), torch.randn(C, generator=g)
    f0 = f1 = None
    if groups:
        f0, f1 = torch.randn(2 * C, generator=g) * 0.3, torch.randn(2, 2 * C, generator=g) * 0.3
        h = F.group_norm(x, groups, gamma, beta, eps=1e-5)
        h = O._scaleshift(O._scaleshift(h, f0.unsqueeze(0).expand(2, -1)), f1)
    else:
        h = F.instance_norm(x, weight=gamma, bias=beta, eps=1e-5)
    ref = {0: h, 1: F.relu(h), 2: F.silu(h)}[act]
    if pool:
        ref = F.avg_pool2d(ref, 2, 2)
    out = G.norm(x, groups, gamma, beta, f0, f1, act=act, pool=pool, out_f16=1)
    d = (out - ref).abs()
    assert (d <= 6e-4 * ref.abs() + 2e-5).all(), (d.max().item(), (d / (ref.abs() + 1e-3)).max().item())


# ------------------------------------------------------------------------------------------ fused decoder tails
def _tail_reference(kind, feature, gamma, beta, groups, act, ws, bs, image0, image1):
    """The reference's own ops for one tail site (eyebrow_decomposer_00.py:49-64, eyebrow_morphing_combiner_00.py:51-72,
    face_morpher_08.py:170-193, morpher_00.py:53-66), restated on the raw last feature map."""
    h = F.group_norm(feature, groups, gamma, beta, eps=1e-5) if groups else F.instance_norm(feature, weight=gamma, bias=beta, eps=1e-5)
    h = F.relu(h) if act == 1 else F.silu(h)
    heads = [F.conv2d(h, w, b, 1, 1) for w, b in zip(ws, bs)]
    if kind == 0:
        return O._unet_tail(heads[0], image0)
    if kind == 1:
        bga, bgc, eba, ebc = torch.sigmoid(heads[0]), torch.tanh(heads[1]), torch.sigmoid(heads[2]), torch.tanh(heads[3])
        return [O.apply_color_change(eba, image0, ebc), eba, ebc, O.apply_color_change(bga, bgc, image0), bga, bgc]
    if kind == 2:
        gc, alpha, color, ca = heads[0], torch.sigmoid(heads[1]), torch.tanh(heads[2]), torch.sigmoid(heads[3])
        warped = O.apply_grid_change(gc, image0)
        morphed = O.apply_color_change(alpha, color, warped)
        return [O.apply_rgb_change(ca, morphed, image1), ca, O.apply_rgb_change((morphed[:, 3:4] + 1.0) / 2.0, morphed, image1),
                morphed, alpha, color, warped, gc]
    gc, imc, ima, eyc, eya = heads[0], torch.tanh(heads[1]), torch.sigmoid(heads[2]), torch.tanh(heads[3]), torch.sigmoid(heads[4])
    im0 = O.apply_grid_change(gc, image0)
    im1 = O.apply_color_change(ima, imc, im0)
    return [O.apply_color_change(eya, eyc, im1), eya, eyc, im1, ima, imc, im0, gc]


TAIL_SITES = [
    # kind, C, S, groups, act, head couts (tail.cu order), which heads have a bias
    (0, 32, 512, 32, 2, [7], [True]),                              # Upscaler02 (upscaler_02.py:84-96)
    (0, 64, 256, 32, 2, [7], [True]),                              # Morpher00 (morpher_00.py:53-66)
    (1, 64, 128, 0, 1, [1, 4, 1, 4], [True] * 4),                  # EyebrowDecomposer00
    (2, 64, 128, 0, 1, [2, 1, 4, 1], [False, True, True, True]),   # EyebrowMorphingCombiner00
    (3, 64, 192, 0, 1, [2, 4, 1, 4, 1], [False, True, True, True, True]),   # FaceMorpher08
]


@pytest.mark.parametrize('site', TAIL_SITES)
@pytest.mark.parametrize('strict', [0, 1])
def test_tail_site_vs_reference_ops(site, strict):
    """Every fused 'grid_sample + decoder' site in isolation, in the default (benchmarked) mode and in strict mode.
    Head weights have trained-like scales (colour ~0.2, warps of a few pixels) so that the warp of a smooth image is a
    well-conditioned function of the head outputs.  Default-mode tolerance: 10-bit operands of a 9*C-term dot product
    (~2e-4 of the head output scale) seen through sigmoid / tanh / a bilinear warp of a smooth image."""
    kind, C, S, groups, act, couts, has_b = site
    g = _gen(kind * 1000 + C + S)
    N = 2 if S <= 256 else 1
    feature = torch.randn(N, C, S, S, generator=g) * 1.5 + 0.3
    gamma, beta = 1.0 + 0.2 * torch.randn(C, generator=g), 0.2 * torch.randn(C, generator=g)
    ws, bs = [], []
    for co, hb in zip(couts, has_b):
        w = torch.randn(co, C, 3, 3, generator=g) / math.sqrt(9 * C)
        if not hb or (kind == 0):
            w = w * 0.3
        if not hb:
            w = w * 0.1                                               # grid_change heads: offsets of ~0.02 (a few pixels)
        ws.append(w)
        bs.append(0.1 * torch.randn(co, generator=g) if hb else None)
    if kind == 0:
        ws[0][4:6] *= 0.1
    image0 = synth.synthetic_image(kind + 3, N)[:, :, :S, :S].contiguous()
    image1 = synth.synthetic_image(kind + 9, N)[:, :, :S, :S].contiguous() if kind == 2 else None
    with torch.no_grad():
        refs = _tail_reference(kind, feature, gamma, beta, groups, act, ws, bs, image0, image1)
    outs = G.tail(kind, feature, gamma, beta, groups, act, ws, bs, image0, image1, strict=strict)
    max_tol, mean_tol = (2e-4, 1e-5) if strict else (6e-3, 3e-4)
    for i, (a, b) in enumerate(zip(outs, refs)):
        mx, mean = G.err(a, b)
        assert mx <= max_tol and mean <= mean_tol, (site, strict, i, mx, mean)
    if not strict:
        # the default mode's kernel is the persistent pipelined one; the one-tile-per-CTA kernel (option tail_persist = 0) is the
        # same arithmetic in the same order: identical outputs
        G.ctx().set_option('tail_persist', 0)
        try:
            one_tile = G.tail(kind, feature, gamma, beta, groups, act, ws, bs, image0, image1, strict=0)
        finally:
            G.ctx().set_option('tail_persist', 1)
        for i, (a, b) in enumerate(zip(outs, one_tile)):
            assert torch.equal(a, b), (site, i, G.err(a, b))


@pytest.mark.parametrize('C,H', [(64, 48), (512, 16), (128, 24)])
def test_instance_norm_relu(C, H):
    g = _gen(C + H)
    x = torch.randn(2, C, H, H, generator=g) * 3 + 1
    gamma, beta = torch.randn(C, generator=g), torch.randn(C, generator=g)
    ref = F.relu(F.instance_norm(x, weight=gamma, bias=beta, eps=1e-5))
    assert G.err(G.norm(x, 0, gamma, beta, act=1), ref)[0] < 2e-5


@pytest.mark.parametrize('C,H,pool', [(32, 64, 0), (96, 32, 0), (192, 16, 1), (384, 16, 0), (512, 16, 1)])
def test_group_norm_film_silu_pool(C, H, pool):
    g = _gen(C * 7 + H)
    x = torch.randn(2, C, H, H, generator=g) * 2 - 0.5
    gamma, beta = torch.randn(C, generator=g), torch.randn(C, generator=g)
    f0, f1 = torch.randn(2 * C, generator=g) * 0.3, torch.randn(2, 2 * C, generator=g) * 0.3
    h = F.group_norm(x, 32, gamma, beta, eps=1e-5)
    h = O._scaleshift(h, f0.unsqueeze(0).expand(2, -1))
    h = O._scaleshift(h, f1)
    ref = F.silu(h)
    if pool:
        ref = F.avg_pool2d(ref, 2, 2)
    assert G.err(G.norm(x, 32, gamma, beta, f0, f1, act=2, pool=pool), ref)[0] < 5e-5


@pytest.mark.parametrize('strict', [0, 1])
def test_attention_vs_reference(strict):
    """strict: the fp32 kernel; default mode: the mma.sync kernel with f16 operands (10-bit mantissa on q, k, P and v:
    a CPU emulation of exactly that rounding gives max 7.2e-3 / mean 2.9e-4 on this input)."""
    g = _gen(11)
    qkv = torch.randn(2, 768, 16, 16, generator=g)
    qkv[:, :512] *= 2.0                       # logits of a few units: a peaked softmax, not a uniform one
    b, c, L, heads = 2, 256, 256, 8
    q, k, v = qkv.reshape(b, 3 * c, L).chunk(3, dim=1)
    scale = 1.0 / math.sqrt(math.sqrt(c // heads))
    w = torch.einsum('bct,bcs->bts', (q * scale).reshape(b * heads, c // heads, L), (k * scale).reshape(b * heads, c // heads, L))
    w = torch.softmax(w, dim=-1)
    ref = torch.einsum('bts,bcs->bct', w, v.reshape(b * heads, c // heads, L)).reshape(b, c, 16, 16)
    G.ctx().set_option('strict', strict)
    try:
        mx, mean = G.err(G.attention(qkv), ref)
    finally:
        G.ctx().set_option('strict', 0)
    assert (mx < 2e-5) if strict else (mx < 1.5e-2 and mean < 6e-4), (strict, mx, mean)     # CPU emulation of the f16 rounding: 7.2e-3 / 2.9e-4


def test_linear_silu():
    g = _gen(3)
    x, W, b = torch.randn(3, 256, generator=g), torch.randn(640, 256, generator=g) / 16, torch.randn(640, generator=g)
    assert G.err(G.linear(x, W, b, 1), F.linear(F.silu(x), W, b))[0] < 2e-5
    assert G.err(G.linear(x[:, :6].contiguous(), W[:, :6].contiguous(), b, 0), F.linear(x[:, :6], W[:, :6], b))[0] < 1e-5


# ------------------------------------------------------------------------------------------ image I/O (SURVEY 8f-1)
@pytest.mark.parametrize('background', [0, 1, 2, 3, 4])
@pytest.mark.parametrize('rint', [False, True])
def test_frame_to_srgb8_vs_oracle(background, rint):
    """The puppeteers' display conversion on the GPU: within 1 LSB of the op-by-op restatement everywhere (powf differs
    from torch's pow in the last ulp, which can move a value across an integer), exact on >= 99.5 % of the bytes."""
    from oracle import image_io
    frames = synth.synthetic_image(21, 2) * 1.1                    # a little outside [-1, 1]: exercises the clip
    out = G.ctx().frame_to_srgb8(frames.to('cuda:0'), background={0: None, 1: 'green', 2: 'blue', 3: 'black', 4: 'white'}[background], rint=rint)
    torch.cuda.synchronize()
    assert out.shape == (2, 512, 512, 4) and out.dtype == torch.uint8
    for n in range(2):
        ref = image_io.frame_to_srgb8(frames[n], background, rint)
        d = (out[n].cpu().int() - ref.int()).abs()
        assert d.max().item() <= 1, (background, rint, d.max().item())
        assert (d == 0).float().mean().item() >= 0.995


def test_rgba8_to_poser_image_vs_loader(golden_dir):
    """PNG pixels -> poser input tensor on the GPU against the host loader (which is pinned to the reference's
    extract_pytorch_image_from_filelike in tests/test_oracle_pinned.py)."""
    import os
    import numpy
    import PIL.Image
    from oracle import image_io
    path = os.path.join(golden_dir, 'data', 'lambda_00.png')
    rgba = torch.from_numpy(numpy.asarray(PIL.Image.open(path).convert('RGBA')).copy())
    out = G.ctx().rgba8_to_poser_image(rgba.to('cuda:0')).cpu()
    ref = image_io.load_rgba_png(path)
    assert out.shape == ref.shape == (4, 512, 512)
    assert G.err(out, ref)[0] <= 2e-6
