"""CPU checks of the fp64 forward references and their bounds (tests/teacher_forward_ref.py): each reference against an
independent closed form, an fp32 / f16 evaluation of each op inside its bound, and each bound small next to the output (so
that it can catch a wrong value); and the GPU case list of test_gpu_teacher_forward_kernels.py against the U-Nets' own
concatenations, derived from state_dict_spec."""
import torch
import torch.nn.functional as F

import teacher_forward_ref as R
from distill_kernel_ref import round_tf32


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _case(seed, N=2, C=96, H=12, groups=32, film=True):
    g = _gen(seed)
    x16 = (torch.randn(N, C, H, H, generator=g) * 1.5 + 0.4).half().double()
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.3
    film0 = torch.randn(2 * C, generator=g) * 0.3 if film else None
    film1 = torch.randn(N, 2 * C, generator=g) * 0.3 if film else None
    return x16, gamma, beta, film0, film1


def test_normalized_operand_matches_group_norm_closed_form():
    x16, gamma, beta, film0, film1 = _case(1)
    C = x16.shape[1]
    sums = R.split_replicas(R.stats_of(x16), 16, 3).sum(0)
    for act in (0, 1, 2):
        a, _ = R.normalized_operand(x16, sums, C, 32, gamma, beta, act, film0, film1)
        h = F.group_norm(x16, 32, gamma.double(), beta.double(), eps=1e-5)
        h = h * (1 + film0[:C].double().view(1, C, 1, 1)) + film0[C:].double().view(1, C, 1, 1)
        h = h * (1 + film1[:, :C].double().view(-1, C, 1, 1)) + film1[:, C:].double().view(-1, C, 1, 1)
        h = {0: h, 1: F.relu(h), 2: F.silu(h)}[act]
        assert (a - h).abs().max().item() < 1e-9


def test_normalized_operand_passes_the_pose_planes_through():
    x16, gamma, beta, _, _ = _case(2, C=40, groups=0, film=False)
    a, e = R.normalized_operand(x16, R.stats_of(x16[:, :32]), 32, 0, gamma[:32], beta[:32], 1)
    assert torch.equal(a[:, 32:], x16[:, 32:]) and (e[:, 32:] == 0).all()
    ref = F.relu(F.instance_norm(x16[:, :32], weight=gamma[:32].double(), bias=beta[:32].double(), eps=1e-5))
    assert (a[:, :32] - ref).abs().max().item() < 1e-9


def _emulate_operand(x16, sums, C, groups, gamma, beta, act, film0, film1, tanh_err_sign):
    """The kernel's arithmetic: fp32 coefficients from the fp64 sums, rounded to f16, one FMA rounded to f16, SiLU as
    h + h tanh(h) in f16 with tanh off by 0.9 of the assumed worst case."""
    N, _, H, W = x16.shape
    gs, cpg = R._group_sums(sums, groups)
    inv = 1.0 / (H * W * cpg)
    mean = gs[..., 0] * inv
    var = (gs[..., 1] * inv - mean * mean).float().clamp_min(0)
    A = torch.rsqrt(var + 1e-5) * gamma.float().view(1, C)
    B = beta.float().view(1, C) - mean.float() * A
    for film in (film0, film1):
        f = film.float().view(-1, 2 * C)
        A, B = A * (1 + f[:, :C]), B * (1 + f[:, :C]) + f[:, C:]
    if act == 2:
        A, B = A * 0.5, B * 0.5
    A16, B16 = (t.half().double().view(-1, C, 1, 1) for t in (A, B))
    h = (x16 * A16 + B16).half().double()
    if act == 2:
        t = (torch.tanh(h) + tanh_err_sign * 0.9 * R.TANH16_ABS).half().double()
        return (h * t + h).half().double()
    return F.relu(h) if act == 1 else h


def test_operand_emulation_stays_inside_its_bound():
    for seed in range(4):
        x16, gamma, beta, film0, film1 = _case(10 + seed)
        C = x16.shape[1]
        sums = R.stats_of(x16)
        for act in (0, 1, 2):
            a, e = R.normalized_operand(x16, sums, C, 32, gamma, beta, act, film0, film1)
            sign = torch.where(torch.rand(a.shape, generator=_gen(seed)) < 0.5, -1.0, 1.0).double()
            em = _emulate_operand(x16, sums, C, 32, gamma, beta, act, film0, film1, sign)
            ratio = ((em - a).abs() / e).max().item()
            assert ratio <= 1.0, (seed, act, ratio)
            # and the bound is tight enough to see a value that is off by one part in 200 of the operand scale
            assert (e / (a.abs().amax() + 1e-30)).max().item() < 5e-3


def test_up2_phases_match_upsample_then_conv():
    """Dyadic weights sum exactly in fp32: the four-phase form equals nearest x2 followed by the 3x3 conv."""
    g = _gen(5)
    w = torch.randint(-64, 64, (24, 16, 3, 3), generator=g).float() / 256
    a = torch.randn(2, 16, 6, 7, generator=g).double()
    wk = R.up2_phase_weights(w).double()
    ref = F.conv2d(F.interpolate(a, scale_factor=2, mode='nearest'), w.double(), None, 1, 1)
    assert (R._conv(4, a, wk) - ref).abs().max().item() < 1e-12


def test_packed_weights_are_tf32_then_scaled_f16():
    g = _gen(6)
    w = torch.randn(64, 32, 3, 3, generator=g) * 1e-3
    wk = R.kernel_weights(0, w)
    wt = round_tf32(w).double()
    scale = 2.0 ** -torch.frexp(wt.abs().max()).exponent.item()      # max |w| * scale in [0.5, 1)
    err = (wk - wt).abs()
    assert (err <= 2.0 ** -11 * wt.abs() + R.F16_FLOOR / scale).all()     # one f16 rounding of the scaled weight
    assert err.max().item() > 0


def test_conv_ref_matches_conv2d_and_fp32_accumulation_stays_inside_bound():
    g = _gen(7)
    for kind, cin, cout, H, act in ((0, 96, 64, 10, 2), (4, 64, 32, 6, 2), (0, 40, 32, 8, 1)):
        x16, gamma, beta, film0, film1 = _case(20 + kind, C=cin, H=H, film=kind == 0 and cin != 40)
        norm_C = 32 if cin == 40 else cin
        groups = 0 if cin == 40 else 32
        w = torch.randn(cout, cin, 3, 3, generator=g) * (2.0 / (9 * cin)) ** 0.5
        bias = torch.randn(cout, generator=g) * 0.1
        Ho = 2 * H if kind == 4 else H
        res = torch.randn(x16.shape[0], cout, Ho, Ho, generator=g) if kind == 0 else None
        sums = R.stats_of(x16[:, :norm_C])
        a, e = R.normalized_operand(x16, sums, norm_C, groups, gamma[:norm_C], beta[:norm_C], act,
                                    film0[:2 * norm_C] if film0 is not None else None, film1)
        wk = R.kernel_weights(kind, w)
        ref, bound = R.conv_ref(kind, a, e, wk, bias, res, 1 if res is not None else 0)
        # independent closed form of the same sum
        if kind == 4:
            alt = R._conv(4, a, wk)
        else:
            alt = F.conv2d(a, wk, None, 1, 1)
        alt = alt + bias.double().view(1, -1, 1, 1) + (res.double() if res is not None else 0)
        assert (alt - ref).abs().max().item() < 1e-10
        # the kernel's arithmetic in fp32: f16 operand (the rounded reference operand), products summed in fp32
        a32 = a.half().float()
        if kind == 4:
            y32 = torch.zeros(ref.shape, dtype=torch.float32)
            for ph in range(4):
                py, px = ph >> 1, ph & 1
                y32[:, :, py::2, px::2] = F.conv2d(F.pad(a32, (1 - px, px, 1 - py, py)), wk[ph].float())
        else:
            y32 = F.conv2d(a32, wk.float(), None, 1, 1)
        y32 = y32 + bias.view(1, -1, 1, 1) + (res if res is not None else 0)
        ratio = ((y32.double() - ref).abs() / bound).max().item()
        assert ratio <= 1.0, (kind, ratio)
        # small next to the output: a value off by 3 % of the output scale is outside the bound
        assert (bound.max() / ref.abs().max()).item() < 3e-2, (kind, (bound.max() / ref.abs().max()).item())


def test_stats_bounds():
    g = _gen(8)
    y = torch.randn(2, 16, 32, 32, generator=g) * 3
    y16 = y.half()
    s, b = R.stats_ref_from_f16(y16)
    assert ((R.stats_of(y) - s).abs() <= b).all()
    mag = torch.stack([y.double().abs().sum((2, 3)), (y.double() ** 2).sum((2, 3))], -1)
    assert (b / mag).max().item() < 1e-3
    assert ((y16.double() - y.double()).abs() <= R.f16_copy_bound(y)).all()


# ------------------------------------------------------------------------------------------ GPU case list vs the networks
def _unet_concats(mc, mults):
    """(resolution level, width, group size, slice boundary) of every up-ResBlock concatenation cat[j] = (h, hs) of a U-Net
    with one res-block per level, all from the weights state_dict_spec.unet_spec lists: the width is what the block's conv0
    reads, the boundary is the width of h, the output of the block before it in the up path (the last middle block, the
    level's first ResBlock, or the previous level's up-sampler)."""
    from tha4_b200.nn.state_dict_spec import unet_spec
    spec = unet_spec('', mc, mults, [False] * len(mults))
    shapes = {k: s for k, s, _ in spec}
    L = len(mults)
    out = set()
    for bi in range(L):
        for r in range(2):
            key = 'up_blocks.%d.resnet_blocks.%d' % (bi, r)
            cin = shapes[key + '.conv0.weight'][1]        # conv0 reads the whole concatenation
            if r == 1:
                prev = 'up_blocks.%d.resnet_blocks.0' % bi
            else:
                prev = 'middle_blocks.6' if bi == 0 else 'up_blocks.%d.upsample' % (bi - 1)
            ch_h = shapes[prev + '.conv1.weight'][0]
            out.add((L - 1 - bi, cin, cin // 32, ch_h))
    return out


def test_gpu_concat_cases_cover_both_unets():
    import test_gpu_teacher_forward_kernels as T
    covered = {(c[1], c[1] // 32, c[2]) for c in T.CONCAT_CASES}
    for mc, mults in ((64, [1, 2, 4, 4, 4]), (32, [1, 2, 4, 8, 8, 8])):
        table = _unet_concats(mc, mults)
        assert len(table) >= 5
        distinct = {(w, gsz, ch_h) for (_, w, gsz, ch_h) in table}
        missing = distinct - covered
        assert not missing, (mc, sorted(missing))


def test_tail_reference_matches_reference_ops_and_fp32_stays_inside_bound():
    """tail_ref against the reference's own ops (oracle) on the same operand, and an fp32 evaluation of those ops on the
    f16-rounded operand inside the bound, for every tail kind; the bound small next to the outputs."""
    from oracle import tha4_oracle as O
    g = _gen(30)
    heads = {0: [7], 1: [1, 4, 1, 4], 2: [2, 1, 4, 1], 3: [2, 4, 1, 4, 1]}
    for kind in range(4):
        N, C, S = 2, 32, 32
        groups, act = (32, 2) if kind == 0 else (0, 1)
        x16 = (torch.randn(N, C, S, S, generator=g) * 1.5 + 0.3).half().double()
        gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.3
        ws = [torch.randn(co, C, 3, 3, generator=g) / (9 * C) ** 0.5 * (0.01 if (i == 0 and kind != 1) else 0.3)
              for i, co in enumerate(heads[kind])]
        bs = [0.1 * torch.randn(co, generator=g) for co in heads[kind]]
        lo = torch.rand(N, 4, 4, 4, generator=g) * 2 - 1
        img0 = F.interpolate(lo, size=(S, S), mode='bilinear', align_corners=False)
        img1 = F.interpolate(torch.rand(N, 4, 4, 4, generator=g) * 2 - 1, size=(S, S), mode='bilinear', align_corners=False)
        refs = R.tail_ref(kind, x16, R.stats_of(x16), groups, act, gamma, beta, ws, bs, img0, img1 if kind == 2 else None)
        a, _ = R.normalized_operand(x16, R.stats_of(x16), C, groups, gamma, beta, act)
        for dt, op in ((torch.float64, a), (torch.float32, a.half().float())):
            h = F.conv2d(op.to(dt), torch.cat(ws).to(dt), torch.cat(bs).to(dt), 1, 1)
            i0, i1 = img0.to(dt), img1.to(dt)
            if kind == 0:
                outs = O._unet_tail(h, i0)
            elif kind == 1:
                bga, bgc, eba, ebc = torch.sigmoid(h[:, 0:1]), torch.tanh(h[:, 1:5]), torch.sigmoid(h[:, 5:6]), torch.tanh(h[:, 6:10])
                outs = [O.apply_color_change(eba, i0, ebc), eba, ebc, O.apply_color_change(bga, bgc, i0), bga, bgc]
            elif kind == 2:
                gc, al, co, ca = h[:, 0:2], torch.sigmoid(h[:, 2:3]), torch.tanh(h[:, 3:7]), torch.sigmoid(h[:, 7:8])
                warped = O.apply_grid_change(gc, i0)
                morphed = O.apply_color_change(al, co, warped)
                outs = [O.apply_rgb_change(ca, morphed, i1), ca, O.apply_rgb_change((morphed[:, 3:4] + 1.0) / 2.0, morphed, i1),
                        morphed, al, co, warped, gc]
            else:
                gc, imc, ima, eyc, eya = h[:, 0:2], torch.tanh(h[:, 2:6]), torch.sigmoid(h[:, 6:7]), torch.tanh(h[:, 7:11]), torch.sigmoid(h[:, 11:12])
                im0 = O.apply_grid_change(gc, i0)
                im1 = O.apply_color_change(ima, imc, im0)
                outs = [O.apply_color_change(eya, eyc, im1), eya, eyc, im1, ima, imc, im0, gc]
            for i, (o, (ref, bound)) in enumerate(zip(outs, refs)):
                err = (o.double() - ref).abs()
                if dt == torch.float64:
                    assert err.max().item() < 1e-9, (kind, i)
                else:
                    assert (err / (bound + 1e-30)).max().item() <= 1.0, (kind, i, (err / (bound + 1e-30)).max().item())
        for i, (ref, bound) in enumerate(refs):
            assert (bound.max() / ref.abs().max().clamp_min(1e-3)).item() < 3e-2, (kind, i)
