"""The 1x1 skip of a U-Net ResBlock folded into the K loop of the block's second conv (-m gpu).

Kernel level (tha4_test_conv_skip_fold): y = conv3x3(GroupNorm + FiLM + SiLU (h0)) + b1 + conv1x1(x) + b_skip as one halo
launch (skip_fold = 1) and as today's pair, the skip conv then conv1 adding it as its residual (skip_fold = 0).  Both form
the same f16 operands and the same products, each weight segment at its own f16 scale; only the fp32 summation order
differs.  Each order's sum of K = 9 Cmid + Cin terms is within K 2^-23 sum |products| of the exact sum, so the two differ
by at most 2 K 2^-23 sum |products| per output element (the bound of test_gpu_halo_split.py).  Module level: Morpher00
and Upscaler02 with skip_fold 1 against skip_fold 0, and the launch log of a whole frame."""
import ctypes
import math
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import gpu_util as G
from oracle import synth, tha4_oracle as O
from tha4_b200._lib import _ptr

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')


def make_inputs(seed, N, Cin, H, W, Cout):
    """A skip block's conv1: h0 [N, Cout, H, W] raw (GroupNorm 32 + FiLM + SiLU pending), x [N, Cin, H, W] the block input."""
    g = torch.Generator().manual_seed(seed)
    Cmid = Cout
    x = torch.randn(N, Cmid, H, W, generator=g) * 1.7 + 0.4
    gamma, beta = 1.0 + 0.3 * torch.randn(Cmid, generator=g), 0.3 * torch.randn(Cmid, generator=g)
    f0, f1 = torch.randn(2 * Cmid, generator=g) * 0.3, torch.randn(N, 2 * Cmid, generator=g) * 0.3
    w = torch.randn(Cout, Cmid, 3, 3, generator=g) / math.sqrt(Cmid * 9)
    b = torch.randn(Cout, generator=g)
    x2 = torch.randn(N, Cin, H, W, generator=g)
    ws = torch.randn(Cout, Cin, 1, 1, generator=g) / math.sqrt(Cin) * 3.0      # a weight scale of its own
    bs = torch.randn(Cout, generator=g)
    return dict(x=x, gamma=gamma, beta=beta, film0=f0, film1=f1, w=w, bias=b, x2=x2, w_skip=ws, b_skip=bs)


def skip_fold(x, gamma, beta, film0, film1, w, bias, x2, w_skip, b_skip, ksplit=0, reps=0):
    """(fp32 output, statistics [N, Cout, 2], folded, mean device microseconds per run or None)."""
    c = G.ctx()
    N, Cmid, H, W = x.shape
    Cout, Cin = w.shape[0], x2.shape[1]
    y = torch.empty(N, Cout, H, W, device=DEV)
    st = torch.empty(N, Cout, 2, dtype=torch.float64, device=DEV)
    folded = ctypes.c_int(-1)
    us = ctypes.c_float(0.0)
    t = [G.dev(v) for v in (x, gamma, beta, film0, film1, w, bias, x2, w_skip, b_skip)]
    c._call('tha4_test_conv_skip_fold', _ptr(t[0]), N, Cmid, H, W, 32, _ptr(t[1]), _ptr(t[2]), _ptr(t[3]), _ptr(t[4]), 2,
            _ptr(t[5]), _ptr(t[6]), _ptr(t[7]), Cin, _ptr(t[8]), _ptr(t[9]), Cout, ksplit, _ptr(y), _ptr(st),
            ctypes.byref(folded), reps, ctypes.byref(us), c._stream())
    torch.cuda.synchronize()
    return y.cpu(), st.cpu(), folded.value, (us.value if reps > 0 else None)


def reference(inp):
    """fp64 output, and the same sum over |products| (the magnitude the reorder bound scales with)."""
    d = torch.device('cuda:0')
    x = inp['x'].to(d, torch.float64)
    h = F.group_norm(x, 32, inp['gamma'].to(d, torch.float64), inp['beta'].to(d, torch.float64), eps=1e-5)
    f0, f1 = inp['film0'].to(d, torch.float64), inp['film1'].to(d, torch.float64)
    h = F.silu(O._scaleshift(O._scaleshift(h, f0.unsqueeze(0).expand(x.shape[0], -1)), f1))
    w, ws, x2 = inp['w'].to(d, torch.float64), inp['w_skip'].to(d, torch.float64), inp['x2'].to(d, torch.float64)
    y = F.conv2d(h, w, inp['bias'].to(d, torch.float64), 1, 1) + F.conv2d(x2, ws, inp['b_skip'].to(d, torch.float64))
    mag = F.conv2d(h.abs(), w.abs(), None, 1, 1) + F.conv2d(x2.abs(), ws.abs())
    return y.cpu(), mag.cpu()


def run_both(inp, ksplit=0):
    c = G.ctx()
    outs = {}
    try:
        for fold in (0, 1):
            c.set_option('skip_fold', fold)
            outs[fold] = skip_fold(**inp, ksplit=ksplit)
            assert outs[fold][2] == fold, 'the hook ran the other path'
    finally:
        c.set_option('skip_fold', 1)
    return outs


def check(outs, inp, case):
    ref, mag = reference(inp)
    (y0, s0, _, _), (y1, s1, _, _) = outs[0], outs[1]
    assert torch.isfinite(y1).all()
    scale = max(1.0, ref.abs().max().item())
    for y in (y0, y1):
        assert (y.double() - ref).abs().max().item() < 6e-3 * scale, ('vs fp64 reference', case)
    K = 9 * inp['x'].shape[1] + inp['x2'].shape[1]
    bound = 2 * K * 2.0 ** -23 * mag * 1.01 + 2.0 ** -23 * ref.abs()      # 1 %: the f16 operands against the fp64 ones; an ulp
    d = (y1.double() - y0.double()).abs()
    assert (d <= bound).all(), ('fp32 reorder bound', case, (d / bound).max().item())
    for y, s in ((y0, s0), (y1, s1)):        # the statistics the next normalisation reads are those of each output
        m = torch.stack([y.double().abs().sum(dim=(2, 3)), y.double().pow(2).sum(dim=(2, 3))], dim=-1)
        st = torch.stack([y.double().sum(dim=(2, 3)), y.double().pow(2).sum(dim=(2, 3))], dim=-1)
        assert ((s - st).abs() <= 1e-5 * m + 1e-6).all(), ('statistics vs output', case)


# (H = W, Cin, Cout): every skip block of Morpher00 (256^2, 64 channels, mults 1 2 4 4 4) and Upscaler02 (512^2, 32 channels,
# mults 1 2 4 8 8 8): down blocks (Cin -> 2 Cin) and up blocks (the concatenation -> Cout)
SHAPES = [
    (16, 512, 256), (32, 512, 256), (64, 512, 256), (64, 384, 256), (64, 128, 256), (128, 384, 128), (128, 192, 128),
    (128, 64, 128), (256, 192, 64), (256, 128, 64), (256, 96, 64), (256, 32, 64), (512, 96, 32), (512, 64, 32),
]


@pytest.mark.parametrize('shape', SHAPES)
def test_network_shapes_batch1(shape):
    H, Cin, Cout = shape
    inp = make_inputs(900 + SHAPES.index(shape), 1, Cin, H, H, Cout)
    check(run_both(inp), inp, shape)


CASES_B2 = [
    # N, H, W, Cin, Cout: batch 2, and partial tiles (H not a multiple of 16 / 32, W not a multiple of 8)
    (2, 16, 16, 512, 256), (2, 64, 64, 384, 256), (2, 128, 128, 192, 128), (2, 256, 256, 96, 64),
    (1, 40, 36, 384, 256), (2, 48, 44, 96, 64), (1, 50, 52, 64, 32),
]


@pytest.mark.parametrize('case', CASES_B2)
def test_batch2_and_partial_tiles(case):
    N, H, W, Cin, Cout = case
    inp = make_inputs(950 + CASES_B2.index(case), N, Cin, H, W, Cout)
    check(run_both(inp), inp, case)


PLANS = [
    # (H, Cin, Cout), options forced: 128- / 256-pixel tiles, one / two CTAs per SM, row-owning pairs, cluster split-K
    ((64, 512, 256), dict(halo_m256=0), 0),
    ((64, 384, 256), dict(halo_m256=1, halo_ctas=1, halo_cs=1), 0),
    ((64, 384, 256), dict(halo_m256=1, halo_ctas=1, halo_cs=2), 0),
    ((128, 192, 128), dict(halo_m256=1, halo_ctas=2), 0),
    ((128, 64, 128), dict(halo_m256=1, halo_ctas=2), 0),
    ((256, 96, 64), dict(halo_m256=1, halo_ctas=1, halo_cs=2), 0),
    ((256, 32, 64), dict(halo_m256=1, halo_ctas=1, halo_cs=1), 0),
    ((512, 96, 32), dict(halo_m256=0), 0),
    ((512, 64, 32), dict(halo_m256=1, halo_cs=2), 0),
    ((32, 512, 256), dict(halo_m256=0), 2),
    ((16, 512, 256), dict(halo_m256=0), 4),
    ((32, 96, 256), dict(halo_m256=0), 8),           # 8 3x3 chunks of 32 channels + 3 skip chunks: eight ranks
]


@pytest.mark.parametrize('plan', PLANS)
def test_plan_variants(plan):
    (H, Cin, Cout), opts, ksplit = plan
    c = G.ctx()
    inp = make_inputs(980 + PLANS.index(plan), 1, Cin, H, H, Cout)
    try:
        for k, v in opts.items():
            c.set_option(k, v)
        outs = run_both(inp, ksplit=ksplit)
    finally:
        for k in opts:
            c.set_option(k, -1)
    check(outs, inp, plan)


_PLAN_CODE = r'''
import sys
sys.path.insert(0, %r)
sys.path.insert(0, %r)
import torch
from oracle import synth
from tha4_b200.poser.modes import mode_07
poser = mode_07.create_poser(torch.device('cuda:0'), state_dicts=synth.teacher_state_dicts(0))
poser.get_context().set_option('cuda_graphs', 0)       # the launch log synchronises after every halo launch
for N in (1, 4):
    image = synth.synthetic_image(0, N).to('cuda:0')
    pose = synth.random_poses(N, seed=1).to('cuda:0')
    poser.get_posing_outputs(image, pose)
    torch.cuda.synchronize()
    sys.stderr.write('BATCH %%d\n' %% N); sys.stderr.flush()
    poser.get_posing_outputs(image, pose)
    torch.cuda.synchronize()
    sys.stderr.write('END\n'); sys.stderr.flush()
'''


def test_frame_runs_every_skip_folded():
    """The launch log (THA4_HALO_DEBUG=2) of a mode_07 frame at batch 1 and 4: the 27 skip blocks of the two U-Nets run
    conv1 with the skip folded in (27 halo launches with a second source)."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = _PLAN_CODE % (os.path.dirname(here), here)
    r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, env=dict(os.environ, THA4_HALO_DEBUG='2'))
    assert r.returncode == 0, r.stderr[-3000:]
    for part in r.stderr.split('BATCH ')[1:]:
        n = int(part.split('\n', 1)[0])
        folded = [line for line in part.split('END\n')[0].splitlines() if line.startswith('halo launch:') and not line.endswith(' cin2 0')]
        assert len(folded) == 27, (n, len(folded))
        assert all((' N %d ' % n) in line for line in folded), folded


def _unet_outputs(module, args):
    with torch.no_grad():
        return [o.detach().cpu().double() for o in module(*[a.to(DEV) for a in args])]


@pytest.mark.parametrize('net', ['body_morpher', 'upscaler'])
def test_module_outputs_match_unfolded(teacher_sds, net):
    from tha4_b200.nn.morpher.morpher_00 import Morpher00
    from tha4_b200.nn.upscaler.upscaler_02 import Upscaler02
    B = 2
    if net == 'body_morpher':
        m = Morpher00()
        args = [F.interpolate(synth.synthetic_image(3, B), size=(256, 256), mode='bilinear', align_corners=False).contiguous(),
                synth.random_poses(B, seed=4)[:, 39:45].contiguous()]
    else:
        m = Upscaler02()
        g = torch.Generator().manual_seed(5)
        args = [synth.synthetic_image(3, B), F.interpolate(synth.synthetic_image(4, B), size=(256, 256), mode='bilinear', align_corners=False).contiguous(),
                torch.randn(B, 2, 256, 256, generator=g) * 0.02, synth.random_poses(B, seed=6)[:, 39:45].contiguous()]
    m.load_state_dict(teacher_sds[net])
    m = m.to(DEV)
    c = m.context()
    try:
        c.set_option('skip_fold', 0)
        ref = _unet_outputs(m, args)
        c.set_option('skip_fold', 1)
        out = _unet_outputs(m, args)
    finally:
        c.set_option('skip_fold', 1)
    for k, (o, r) in enumerate(zip(out, ref)):
        # fp32 reordering inside each folded conv, carried through the f16 activations of the layers that follow
        rel = ((o - r).norm() / max(r.norm().item(), 1e-30)).item()
        print('\n%s output %d: max abs %.3e rel L2 %.3e' % (net, k, (o - r).abs().max().item(), rel))
        assert rel <= 2e-3, (net, k, rel)
