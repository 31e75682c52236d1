"""CPU checks of the SIREN student test machinery (no GPU): the fp16 rounding-point reference (oracle/siren_fp16.py)
restates the same network as the fp32 oracle, the comparisons of tests/test_gpu_siren.py catch the faults they are meant
to catch, and the wgmma plan validator accepts the production plans and names each violation it rejects."""
import ctypes

import pytest
import torch

from oracle import siren_fp16 as S, synth, tha4_oracle as O


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _body_layers(sd, i):
    return [S.layer(sd, 'siren_layers.%d.%d.linear' % (i, j)) for j in range(3)]


def _head(sd, key):
    return S.layer(sd, key)


def test_fp16_reference_matches_fp32_oracle(lambda00_sds, oracle_clib):
    """The body student on the trained lambda_00 weights: the fp16 restatement against the fp32 oracle stays within the
    precision class of fp16 activations (measured with an independent restatement: grid_change mean 1.8e-4 / max 1.35e-3,
    alpha 3.1e-4 / 1.1e-2, colour 3.5e-4 / 2.8e-2)."""
    sd = lambda00_sds['body_morpher']
    pose = synth.random_poses(1, seed=5)
    image = synth.synthetic_image(0, 1)
    with torch.no_grad():
        ref = O.siren_morpher_03(sd, image, pose)
        a0 = S.level_forward(0, _body_layers(sd, 0), pose)
        a1 = S.level_forward(1, _body_layers(sd, 1), pose, prev=a0)
        out = S.level_forward(2, _body_layers(sd, 2), pose, head=_head(sd, 'last_linear'), prev=a1, image=image, clib=oracle_clib)
    errs = {}
    for name, i, mean_class, max_class in (('grid_change', 4, 1.8e-4, 1.35e-3), ('alpha', 1, 3.1e-4, 1.1e-2), ('color', 2, 3.5e-4, 2.8e-2)):
        d = (out[i] - ref[i].double()).abs()
        errs[name] = (d.mean().item(), d.max().item())
        print('fp16 reference vs fp32 oracle, %s: mean %.2e max %.2e' % (name, *errs[name]))
        assert d.mean().item() <= 2 * mean_class and d.max().item() <= 3 * max_class, (name, errs[name])
        assert d.mean().item() >= mean_class / 10, ('the fp16 reference rounds like the fp32 oracle?', name, errs[name])


def _controlled_level1(seed=0, R=32, B=3, feat=90, n=128):
    g = _gen(seed)
    pose = (torch.rand(B, 45, generator=g) * 2 - 1)
    W, b = S.controlled_layer(g, n, feat, extra=2 + 45, bias_max=30.0, l1=20.0)
    prev = S.f16(torch.rand(B, R // 2, R // 2, feat, generator=g).double() * 2 - 1)
    return [(W, b)], pose, prev


def _init_level1(student_sds, R=32, B=2):
    sd = student_sds['body_morpher']
    g = _gen(3)
    pose = synth.random_poses(B, seed=7)
    prev = S.f16(torch.sin(torch.randn(B, R // 2, R // 2, 180, generator=g).double() * 2))
    return _body_layers(sd, 1), pose, prev


@pytest.mark.parametrize('mutation', S.MUTATIONS)
def test_comparisons_catch_mutated_references(student_sds, mutation):
    """Each fault fails both the single-layer ulp comparison (test 1) and the per-level bounds (test 2) by at least 2x."""
    layers, pose, prev = _controlled_level1()
    ref = S.level_forward(1, layers, pose, prev=prev, R=32)
    assert S.ulp_ratio(ref, ref)[0] == 0
    bad = S.level_forward(1, layers, pose, prev=prev, R=32, mutate=mutation, nb=64)
    ratio, mx, mean = S.ulp_ratio(bad, ref)
    print('%s: single layer, ulp ratio %.1f (max %.2e mean %.2e)' % (mutation, ratio, mx, mean))
    assert ratio >= 2, (mutation, ratio)

    layers, pose, prev = _init_level1(student_sds)
    ref = S.level_forward(1, layers, pose, prev=prev, R=32)
    bad = S.level_forward(1, layers, pose, prev=prev, R=32, mutate=mutation, nb=96)
    ratio, mx, mean = S.level_ratio(bad, ref)
    print('%s: init-like level 1, bound ratio %.1f (max %.2e mean %.2e)' % (mutation, ratio, mx, mean))
    assert ratio >= 2, (mutation, ratio)


def test_upsample_variants_round_where_the_kernels_round():
    """wgmma: HMUL2 + 3 HFMA2 (four roundings), mma.sync: fp32 lerp (one rounding); both within 2 fp16 ulp of each other
    and exact where the taps coincide with source pixels (edge clamps)."""
    g = _gen(1)
    prev = S.f16(torch.rand(2, 8, 8, 16, generator=g).double() * 2 - 1)
    a, b = S.upsample(prev, 'wgmma'), S.upsample(prev, 'mma')
    assert (a - b).abs().max().item() <= 2 * 2 ** -10
    assert not torch.equal(a, b)
    ref = torch.nn.functional.interpolate(prev.permute(0, 3, 1, 2), scale_factor=2, mode='bilinear', align_corners=False).permute(0, 2, 3, 1)
    assert (b - ref).abs().max().item() <= 2 ** -11


# ------------------------------------------------------------------------------------------------ plan validator
@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as g
    g.build_cuda()
    from tha4_b200 import _lib
    return _lib.load_library()


def _check(lib, mode, layers, R, e_npad=0, prev_c=0, out_c=None):
    """layers: (kpad, npad, nb, sine, first) per GEMM layer"""
    n = len(layers)
    cols = [(ctypes.c_int * max(n, 1))(*[l[j] for l in layers]) for j in range(5)]
    if out_c is None:
        out_c = layers[-1][1] if layers and layers[-1][3] else 0
    msg = ctypes.create_string_buffer(512)
    rc = lib.tha4_test_siren_plan_check(mode, n, *cols, R, e_npad, prev_c, out_c, msg, 512)
    return rc, msg.value.decode()


PRODUCTION = {
    0: dict(layers=[(384, 384, 96, 1, 0), (384, 192, 96, 1, 0)], R=128, e_npad=384),
    1: dict(layers=[(192, 192, 96, 1, 1), (192, 192, 96, 1, 0), (192, 96, 96, 1, 0)], R=256, prev_c=192),
    2: dict(layers=[(96, 96, 96, 1, 1), (96, 96, 96, 1, 0), (96, 96, 96, 1, 0), (96, 16, 16, 0, 0)], R=512, prev_c=96),
    3: dict(layers=[(128, 128, 64, 1, 0)] * 7 + [(128, 16, 16, 0, 0)], R=128, e_npad=128),
}


def test_plan_validator_accepts_production_plans(lib):
    for mode, p in PRODUCTION.items():
        assert _check(lib, mode, **p) == (0, ''), mode


def _with(p, **kw):
    q = dict(p, layers=list(p['layers']))
    for k, v in kw.items():
        if k != 'layers' and k.startswith('layer'):
            i, field = int(k[5]), k[7:]
            t = list(q['layers'][i])
            t[('kpad', 'npad', 'nb', 'sine', 'first').index(field)] = v
            q['layers'][i] = tuple(t)
        else:
            q[k] = v
    return q


VIOLATIONS = [
    ('layer count', 0, dict(layers=[])),
    ('layer count', 3, dict(layers=[(128, 128, 64, 1, 0)] * 8 + [(128, 16, 16, 0, 0)])),
    ('multiple of 16', 1, dict(layer0_kpad=184, prev_c=184)),
    ('operand buffer', 2, dict(layer0_kpad=192, prev_c=192)),              # prev_c = 192 > 2 x 64 is caught first
    ('operand buffer', 1, dict(layer1_kpad=256, layer0_npad=256, layer0_nb=64)),
    ('its producer wrote', 1, dict(layer1_kpad=192, layer0_npad=96)),
    ('its producer wrote', 0, dict(layer0_kpad=384, e_npad=256)),
    ('its producer wrote', 2, dict(layer0_kpad=96, prev_c=64)),
    ('is not 16, 64 or 96', 1, dict(layer1_nb=32)),
    ('NBMAX', 3, dict(layer2_nb=96, layer2_npad=96, layer3_kpad=96)),
    ('multiple of nb', 1, dict(layer2_npad=64)),
    ('sine layer npad', 2, dict(layer1_npad=192, layer1_nb=96, layer2_kpad=96)),
    ('head must be the last', 2, dict(layer1_sine=0)),
    ('head npad', 2, dict(layer3_npad=32, layer3_nb=16)),
    ('head npad', 3, dict(layer7_nb=64, layer7_npad=64)),
    ('modes 2 / 3 only', 1, dict(layer2_sine=0, layer2_npad=16, layer2_nb=16, out_c=0)),
    ('> 384', 0, dict(e_npad=448)),
    ('> 384', 1, dict(layers=[(192, 480, 96, 1, 1)], out_c=480)),
    ('prev_c', 1, dict(prev_c=100)),
    ('prev_c', 1, dict(prev_c=200)),
    ('out_c', 0, dict(out_c=96)),
    ('out_c', 1, dict(out_c=192)),
    ('multiple of 128', 2, dict(R=320)),
    ('first GEMM layer', 1, dict(layer0_first=0)),
    ('not the first GEMM layer', 0, dict(layer0_first=1)),
]


@pytest.mark.parametrize('needle,mode,change', VIOLATIONS, ids=['%d-%s' % (m, n) for n, m, _ in VIOLATIONS])
def test_plan_validator_names_each_violation(lib, needle, mode, change):
    p = _with(PRODUCTION[mode], **change)
    rc, msg = _check(lib, mode, **p)
    print(mode, change, '->', msg)
    assert rc != 0 and needle in msg, (change, msg)
