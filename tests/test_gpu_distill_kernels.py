"""Kernel-level parity of the student training step (tha4_b200/csrc/distill.cu) on the H100 (-m gpu).

Each stage runs through its tha4_test_* entry, which calls the host function the training step calls, at the production
shapes of SirenMorpher03 / SirenFaceMorpher00.  The references are fp64 and round only where the kernel rounds
(tests/distill_kernel_ref.py).  Every family has a dyadic case, on which the result must equal the reference bit for bit
whatever the summation order, and a random case held to a worst-case bound computed from the inputs.
"""
import ctypes
import math

import pytest
import torch

import distill_kernel_ref as D
import gpu_util as G
from tha4_b200._lib import _ptr, _ptr_array

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
E23 = 2.0 ** -23

# (nreal, kreal, kpad, npad, R) of every layer in state_dict order (distill.cu body_layers / face_layers)
BODY = [(360, 47, 48, 360, 128), (360, 360, 360, 360, 128), (180, 360, 360, 180, 128),
        (180, 227, 228, 180, 256), (180, 180, 180, 180, 256), (90, 180, 180, 92, 256),
        (90, 137, 140, 92, 512), (90, 90, 92, 92, 512), (90, 90, 92, 92, 512), (7, 90, 92, 8, 512)]
FACE = [(128, 41, 44, 128, 128)] + [(128, 128, 128, 128, 128)] * 7 + [(4, 128, 128, 4, 128)]


def _ctx():
    return G.ctx()


def _call(name, *args):
    c = _ctx()
    c._call(name, *args, c._stream())


def _ints(v):
    return (ctypes.c_int * len(v))(*v)


def _randn(shape, seed, scale=1.0):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)) * scale


def _exceed(name, err, bound, extra=''):
    """assert err <= bound elementwise, naming the worst element"""
    over = err > bound
    if bool(over.any()):
        i = int(torch.argmax((err - bound).reshape(-1)))
        pytest.fail('%s%s: %d elements over the bound, worst at flat index %d: |err| %.3e > bound %.3e'
                    % (name, extra, int(over.sum()), i, err.reshape(-1)[i].item(), bound.reshape(-1)[i].item()))


# ------------------------------------------------------------------------------------------ dense GEMM (1x1 conv)
def _dense_gemm(W, x, Cout, R, transpose, bias=None):
    P, Cin = x.shape
    y = torch.full((P, Cout), float('nan'), device=DEV)
    Wd, xd = W.to(DEV).contiguous(), x.to(DEV).contiguous()
    bd = None if bias is None else bias.to(DEV).contiguous()
    _call('tha4_test_dense_gemm', _ptr(Wd), W.shape[0], W.shape[1], int(transpose), _ptr(bd), _ptr(xd), Cin, _ptr(y), Cout, P // (R * R), R)
    torch.cuda.synchronize()
    return y


def _gemm_cases():
    cases = []
    for i, (n, k, kp, np_, R) in enumerate(BODY):
        if i != 8:                                       # layer 8 has layer 7's shape
            cases.append(('body%d' % i, n, k, kp, np_, R, False))
        if 1 <= i <= 9 and i != 8:
            cases.append(('body%d_T' % i, n, k, kp, np_, R, True))
    for i in (0, 1, 8):
        n, k, kp, np_, R = FACE[i]
        cases.append(('face%d' % i, n, k, kp, np_, R, False))
    for i in (1, 8):
        n, k, kp, np_, R = FACE[i]
        cases.append(('face%d_T' % i, n, k, kp, np_, R, True))
    return cases


@pytest.mark.parametrize('kind', ['dyadic', 'random'])
@pytest.mark.parametrize('name, nreal, kreal, kpad, npad, R, transpose', _gemm_cases(), ids=[c[0] for c in _gemm_cases()])
def test_dense_gemm(kind, name, nreal, kreal, kpad, npad, R, transpose):
    Cin, Cout = (npad, kpad) if transpose else (kpad, npad)
    Kr = nreal if transpose else kreal                # real reduction length
    P = R * R
    seed = sum(map(ord, name))
    if kind == 'dyadic':
        x = D.dyadic((P, Cin), 4, 4, seed)
        W = D.dyadic((nreal, kreal), 6, 6, seed + 1)
        xm, xu = D.dyadic_unit(4, 4)
        wm, wu = D.dyadic_unit(6, 6)
        bias = None if transpose else D.dyadic((nreal,), 10, 10, seed + 2)
        D.assert_exact_sums(Kr, xm * wm, xu * wu, start=0.0 if transpose else D.dyadic_unit(10, 10)[0])
    else:
        x = _randn((P, Cin), seed)
        W = _randn((nreal, kreal), seed + 1, 1.0 / math.sqrt(Kr))
        bias = None if transpose else _randn((nreal,), seed + 2, 0.1)
    bias_pad = None if bias is None else torch.cat([bias, torch.zeros(Cout - nreal)])
    y = _dense_gemm(W, x, Cout, R, transpose, bias_pad)
    Wt = D.round_tf32(W).double().to(DEV)             # what pack_dense_kernel hands the conv
    xd = x.double().to(DEV)
    A = Wt if transpose else Wt.t()                   # [Kr][nout]
    xr = xd[:, :Kr]
    ref = xr @ A
    nout = A.shape[1]
    if bias is not None:
        ref = ref + bias.double().to(DEV)
    pad = y[:, nout:]
    assert bool((pad == 0).all()), '%s: pad output channels %d..%d are not exactly 0' % (name, nout, Cout - 1)
    got = y[:, :nout].double()
    if kind == 'dyadic':
        assert torch.equal(got, ref), '%s: dyadic GEMM not bit-exact, max |err| %.3e' % (name, (got - ref).abs().max().item())
        return
    S = xr.abs() @ A.abs()
    bound = (2.0 ** -10 + Kr * E23) * S + D.ulp32(ref.abs() + (0 if bias is None else bias.double().abs().to(DEV)))
    err = (got - ref).abs()
    print('\n%s: max |err| / bound %.3e' % (name, (err / bound).max().item()))
    _exceed(name, err, bound)


# ------------------------------------------------------------------------------------------ weight and bias gradients
WGRAD = [(360, 48, 360, 47, 128), (360, 360, 360, 360, 128), (180, 360, 180, 360, 128), (180, 228, 180, 227, 256),
         (180, 180, 180, 180, 256), (92, 180, 90, 180, 256), (92, 140, 90, 137, 512), (92, 92, 90, 90, 512), (8, 92, 7, 90, 512),
         (128, 44, 128, 41, 128), (128, 128, 128, 128, 128), (4, 128, 4, 128, 128)]


def _psplit(P):
    return max(1, min(64, P // 4096))


def _wgrad_cases():
    cases = [(nc, kc, nr, kr, R * R, 'layer') for nc, kc, nr, kr, R in WGRAD]               # psplit 4, 16, 64
    for nc, kc, nr, kr, _ in (WGRAD[0], WGRAD[5], WGRAD[8], WGRAD[11]):
        cases.append((nc, kc, nr, kr, 4096, 'psplit1'))
        cases.append((nc, kc, nr, kr, 70001, 'partial'))                                  # 4118 pixels per split, not % 32
    for nc, kc, nr, kr, _ in (WGRAD[6], WGRAD[8]):
        cases.append((nc, kc, nr, kr, 8 * 512 * 512, 'batch8'))                             # 32768 pixels per split
    return cases


@pytest.mark.parametrize('kind', ['dyadic', 'random'])
@pytest.mark.parametrize('Nc, Kc, nreal, kreal, P, tag', _wgrad_cases(),
                         ids=['%dx%d_P%d' % (c[0], c[1], c[4]) for c in _wgrad_cases()])
def test_dense_wgrad_accumulates(kind, Nc, Kc, nreal, kreal, P, tag):
    seed = Nc * 7 + Kc * 3 + P % 997
    gen = torch.Generator(device=DEV).manual_seed(seed)
    if kind == 'dyadic':
        a, b = (3, 4) if P <= 70001 else ((2, 3) if P <= 512 * 512 else (1, 2))
        dz = D.dyadic((P, Nc), a, a, seed, device=DEV)
        x = D.dyadic((P, Kc), b, b, seed + 1, device=DEV)
        (dm, du), (xm, xu) = D.dyadic_unit(a, a), D.dyadic_unit(b, b)
        w0 = D.dyadic((nreal, kreal), 3, a + b, seed + 2).to(DEV)
        b0 = D.dyadic((nreal,), 3, a, seed + 3).to(DEV)
        D.assert_exact_sums(P, dm * xm, du * xu, start=D.dyadic_unit(3, a + b)[0])
        D.assert_exact_sums(P, dm, du, start=D.dyadic_unit(3, a)[0])
    else:
        dz = torch.randn((P, Nc), generator=gen, device=DEV)
        x = torch.randn((P, Kc), generator=gen, device=DEV)
        w0 = torch.randn((nreal, kreal), generator=gen, device=DEV)
        b0 = torch.randn((nreal,), generator=gen, device=DEV)
    GUARD = 1024
    SENT = -12345.678
    buf = torch.full((nreal * kreal + GUARD,), SENT, device=DEV)
    bbuf = torch.full((nreal + GUARD,), SENT, device=DEV)
    buf[:nreal * kreal] = w0.reshape(-1)
    bbuf[:nreal] = b0
    _call('tha4_test_dense_wgrad', _ptr(dz), Nc, _ptr(x), Kc, P, nreal, kreal, _ptr(buf), _ptr(bbuf))
    torch.cuda.synchronize()
    assert bool((buf[nreal * kreal:] == SENT).all()), 'dW guard region written'
    assert bool((bbuf[nreal:] == SENT).all()), 'db guard region written'
    dW, db = buf[:nreal * kreal].view(nreal, kreal).double(), bbuf[:nreal].double()
    dzr = D.round_tf32(dz[:, :nreal]).double()
    xr = D.round_tf32(x[:, :kreal]).double()
    refW = w0.double() + dzr.t() @ xr
    refb = b0.double() + dz[:, :nreal].double().sum(0)
    del x
    if kind == 'dyadic':
        assert torch.equal(dW, refW), 'dW not bit-exact (start + sum): max |err| %.3e' % (dW - refW).abs().max().item()
        assert torch.equal(db, refb), 'db not bit-exact (start + sum): max |err| %.3e' % (db - refb).abs().max().item()
        return
    ps = _psplit(P)
    per = -(-P // ps)
    SW = dzr.abs().t() @ xr.abs() + w0.double().abs()
    boundW = (per / 8 + ps + 8 + 1) * E23 * SW
    cq = Nc // 4
    PL = 256 // cq
    grid = min(148, max(1, P // 512))
    rows = -(-P // (grid * PL))
    Sb = dz[:, :nreal].double().abs().sum(0) + b0.double().abs()
    boundb = (rows + PL + grid + 1) * E23 * Sb
    print('\nP %d psplit %d: dW err/bound %.3e, db err/bound %.3e' % (P, ps, ((dW - refW).abs() / boundW).max().item(),
                                                                      ((db - refb).abs() / boundb).max().item()))
    _exceed('dW', (dW - refW).abs(), boundW)
    _exceed('db', (db - refb).abs(), boundb)


# ------------------------------------------------------------------------------------------ level input and its adjoint
def _level_input(prev, Cprev, pose, npose, R, N, C):
    out = torch.full((N, R, R, C), float('nan'), device=DEV)
    pd = pose.to(DEV).contiguous()
    prevd = None if prev is None else prev.to(DEV).contiguous()
    _call('tha4_test_level_input', 0, _ptr(prevd), Cprev, 0 if prev is None else prev.shape[-1], _ptr(pd), pose.shape[1], npose,
          R, N, C, _ptr(None), 0, _ptr(out))
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.parametrize('R, Cprev, prev_ld, C, npose', [(128, 0, 0, 48, 45), (256, 180, 180, 228, 45), (512, 90, 92, 140, 45),
                                                          (128, 0, 0, 44, 39)])
def test_level_input_is_bit_exact(oracle_clib, R, Cprev, prev_ld, C, npose):
    N, pose_ld = 2, 64
    pose = _randn((N, pose_ld), R + C)
    pose[:, npose:] = 1e30                           # junk past the pose entries must not be read
    prev = None
    if Cprev:
        prev = _randn((N, R // 2, R // 2, prev_ld), R + 1)
        prev[..., Cprev:] = float('nan')             # pad channels of the previous level are not read either
    out = _level_input(prev, Cprev, pose, npose, R, N, C)
    base = D.base_grid(oracle_clib, R)
    if Cprev:
        up = D.upsample2(oracle_clib, prev[..., :Cprev].permute(0, 3, 1, 2)).permute(0, 2, 3, 1)
        assert torch.equal(out[..., :Cprev], up), 'upsampled channels: max |err| %.3e' % (out[..., :Cprev] - up).abs().max().item()
    assert torch.equal(out[..., Cprev], base.view(1, 1, R).expand(N, R, R)), 'x coordinate channel'
    assert torch.equal(out[..., Cprev + 1], base.view(1, R, 1).expand(N, R, R)), 'y coordinate channel'
    assert torch.equal(out[..., Cprev + 2:Cprev + 2 + npose], pose[:, None, None, :npose].expand(N, R, R, npose)), 'pose channels'
    assert bool((out[..., Cprev + 2 + npose:] == 0).all()), 'pad channels are not exactly 0'


def test_level_input_dyadic(oracle_clib):
    """Dyadic previous level: the bilinear weights (multiples of 1/16) make every value exact, so fp64 agrees too."""
    N, R, Cprev, C = 2, 256, 180, 228
    prev = D.dyadic((N, R // 2, R // 2, 180), 8, 8, 3)
    pose = D.dyadic((N, 45), 8, 8, 4)
    out = _level_input(prev, Cprev, pose, 45, R, N, C)
    ref = torch.nn.functional.interpolate(prev.permute(0, 3, 1, 2).double(), scale_factor=2, mode='bilinear', align_corners=False)
    assert torch.equal(out[..., :Cprev].double(), ref.permute(0, 2, 3, 1))


@pytest.mark.parametrize('kind', ['dyadic', 'random'])
@pytest.mark.parametrize('R, Cprev, up_ld, prev_ld', [(256, 180, 228, 180), (512, 90, 140, 92)])
def test_upsample_backward(kind, R, Cprev, up_ld, prev_ld):
    N, Rh = 2, R // 2
    if kind == 'dyadic':
        dup = D.dyadic((N, R, R, up_ld), 8, 8, R)
        m, u = D.dyadic_unit(8, 8)
        D.assert_exact_sums(16, m, u / 16)                  # <= 4 x 4 taps, weights multiples of 1/16
    else:
        dup = _randn((N, R, R, up_ld), R)
    SENT = 777.0
    dprev = torch.full((N, Rh, Rh, prev_ld), SENT, device=DEV)
    dd = dup.to(DEV)
    _call('tha4_test_level_input', 1, _ptr(None), Cprev, prev_ld, _ptr(None), 0, 0, R, N, 0, _ptr(dd), up_ld, _ptr(dprev))
    torch.cuda.synchronize()
    dprev = dprev.cpu()
    if prev_ld > Cprev:
        assert bool((dprev[..., Cprev:] == SENT).all()), 'pad channels %d..%d of dprev were written' % (Cprev, prev_ld - 1)
    d = dup[..., :Cprev].permute(0, 3, 1, 2)
    ref = D.upsample2_adjoint(d).permute(0, 2, 3, 1)
    got = dprev[..., :Cprev].double()
    border = torch.zeros(Rh, Rh, dtype=torch.bool)
    border[0, :] = border[-1, :] = border[:, 0] = border[:, -1] = True
    if kind == 'dyadic':
        for name, sel in (('border', border), ('interior', ~border)):
            e = (got - ref)[:, sel]
            assert bool((e == 0).all()), '%s source pixels not bit-exact: max |err| %.3e' % (name, e.abs().max().item())
        return
    bound = 16 * E23 * D.upsample2_weights_abs(d).permute(0, 2, 3, 1)
    err = (got - ref).abs()
    for name, sel in (('border', border), ('interior', ~border)):
        _exceed('dprev', err[:, sel], bound[:, sel], ' (%s source pixels)' % name)


# ------------------------------------------------------------------------------------------ sine
def _sine_inputs(n, seed):
    g = torch.Generator().manual_seed(seed)
    z = (torch.rand(n, generator=g) * 2 - 1) * 40.0          # |30 z| <= 1200
    z[:n // 8] = 0.0                                          # pad channels: z = 0 exactly
    z[n // 8:n // 4] = (torch.rand(n // 8, generator=g) * 2 - 1) * 0.1
    da = torch.randn(n, generator=g)
    da[n // 4:n // 4 + n // 16] = 0.0
    return z, da


def test_sine_forward_and_backward():
    n = 1 << 20
    z, da = _sine_inputs(n, 5)
    zd, dad = z.to(DEV), da.to(DEV)
    a, dz = torch.empty(n, device=DEV), torch.empty(n, device=DEV)
    _call('tha4_test_distill_sine', 0, _ptr(zd), _ptr(None), n, _ptr(a))
    _call('tha4_test_distill_sine', 1, _ptr(zd), _ptr(dad), n, _ptr(dz))
    torch.cuda.synchronize()
    assert torch.equal(dad.cpu(), da), 'the backward must not modify da'
    a, dz = a.cpu().double(), dz.cpu().double()
    arg = (z * 30.0).double()                                  # fl32(30 z), as the kernel forms it
    ref_a = torch.sin(arg)
    ref_dz = 30.0 * da.double() * torch.cos(arg)
    zero = z == 0
    assert bool((a[zero] == 0).all()), 'sin(30 * 0) must be exactly 0'
    assert torch.equal(dz[zero], (da[zero] * 30.0).double()), 'dz at z = 0 must be exactly 30 da'
    assert bool((dz[da == 0] == 0).all())
    _exceed('sin(30 z)', (a - ref_a).abs(), 2 * D.ulp32(ref_a))
    _exceed('30 da cos(30 z)', (dz - ref_dz).abs(), 30 * da.double().abs() * 2.0 ** -21 + 2 * D.ulp32(ref_dz))


# ------------------------------------------------------------------------------------------ pose gradient
BODY_POSE = [(128 * 128, 360, 360, 47, 2), (256 * 256, 180, 180, 227, 182), (512 * 512, 92, 90, 137, 92)]
FACE_POSE = [(128 * 128, 128, 128, 41, 2)]


def _pose_grad(levels, dzs, Ws, N, npose):
    dzd = [d.to(DEV).contiguous() for d in dzs]
    Wd = [w.to(DEV).contiguous() for w in Ws]
    out = torch.full((N, npose), float('nan'), device=DEV)
    _call('tha4_test_pose_grad', len(levels), _ptr_array(dzd), _ints([l[1] for l in levels]), _ints([l[0] for l in levels]),
          _ptr_array(Wd), _ints([l[2] for l in levels]), _ints([l[3] for l in levels]), _ints([l[4] for l in levels]), N, npose,
          _ptr(out))
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.parametrize('kind', ['dyadic', 'random'])
@pytest.mark.parametrize('which', ['body', 'face'])
def test_pose_gradient(kind, which):
    levels, npose = (BODY_POSE, 45) if which == 'body' else (FACE_POSE, 39)
    N = 3
    dzs, Ws = [], []
    for i, (hw, C, nr, kr, col0) in enumerate(levels):
        if kind == 'dyadic':
            dz = D.dyadic((N, hw, C), 3, 3, 10 + i)
            D.assert_exact_sums(256, D.dyadic_unit(3, 3)[0], D.dyadic_unit(3, 3)[1])      # one fp32 chunk sum
            W = D.dyadic((nr, kr), 6, 6, 20 + i)
        else:
            dz = _randn((N, hw, C), 10 + i)
            W = _randn((nr, kr), 20 + i, 0.05)
        dz[..., nr:] = float('nan')                  # pad channels of dz are not read
        dzs.append(dz)
        Ws.append(W)
    got = _pose_grad(levels, dzs, Ws, N, npose).double()
    ref = torch.zeros(N, npose, dtype=torch.float64)
    bound = torch.zeros(N, npose, dtype=torch.float64)
    for (hw, C, nr, kr, col0), dz, W in zip(levels, dzs, Ws):
        Wp = W[:, col0:col0 + npose].double()
        ref += dz[..., :nr].double().sum(1) @ Wp
        PL = 256 // (C // 4)
        bound += (-(-256 // PL) + PL) * E23 * (dz[..., :nr].double().abs().sum(1) @ Wp.abs())
    if kind == 'dyadic':
        assert torch.equal(got, ref.float().double()), 'dyadic d(pose) not bit-exact: max |err| %.3e' % (got - ref).abs().max().item()
    else:
        bound += D.ulp32(ref) / 2
        print('\n%s d(pose) err/bound %.3e' % (which, ((got - ref).abs() / bound).max().item()))
        _exceed('d(pose)', (got - ref).abs(), bound)
    # each sample's value is bit-reproducible and independent of the batch
    one = _pose_grad(levels, [d[1:2] for d in dzs], Ws, 1, npose)
    assert torch.equal(one[0], got[1].float()), 'sample 1 differs between N = 1 and N = 3'


# ------------------------------------------------------------------------------------------ loss and gradient tails
GRIDS = {'random': None, 'zero': (0.0, 0.0), 'half_integer': (1.0 / 512, -3.0 / 512), 'border_clamp': (1.5, -1.5),
         'mixed_clamp': (0.25, -0.3125)}


def _out7(grid, N, seed):
    R = 512
    g = torch.Generator().manual_seed(seed)
    out7 = torch.zeros(N, R, R, 8)
    if GRIDS[grid] is None:
        out7[..., 0:2] = (torch.rand(N, R, R, 2, generator=g) * 2 - 1) * 0.05
    else:
        out7[..., 0], out7[..., 1] = GRIDS[grid]
    a = torch.rand(N, R, R, generator=g) * 1.5 - 0.25
    sel = torch.randint(0, 8, (N, R, R), generator=g)
    a[sel == 0] = 0.0
    a[sel == 1] = 1.0
    out7[..., 2] = a
    out7[..., 3:7] = torch.rand(N, R, R, 4, generator=g) * 2 - 1
    out7[..., 7] = float('nan')                      # pad slot: not read
    return out7


def _clamped(oracle_clib, gc):
    R = gc.shape[-1]
    b = D.base_grid(oracle_clib, R)
    ix = (((b.view(1, 1, R) + gc[:, 0]) + 1) * R - 1) / 2
    iy = (((b.view(1, R, 1) + gc[:, 1]) + 1) * R - 1) / 2
    return (ix <= 0) | (ix >= R - 1), (iy <= 0) | (iy >= R - 1)


def _away(ref, seed, lo=1e-3, hi=0.1):
    """a target at least `lo` away from ref"""
    g = torch.Generator().manual_seed(seed)
    s = torch.where(torch.rand(ref.shape, generator=g) < 0.5, -1.0, 1.0)
    return (ref + s * (lo + (hi - lo) * torch.rand(ref.shape, generator=g))).float()


def _tail(kind, out, image, N, t=(None, None, None), g=None, w=None):
    od = out.to(DEV).contiguous()
    imd = None if image is None else image.to(DEV).contiguous()
    td = [None if x is None else x.to(DEV).contiguous() for x in t]
    gd = None if g is None else [None if x is None else x.to(DEV).contiguous() for x in g]
    d_out = torch.full(out.shape, float('nan'), device=DEV)
    sums = torch.full((4,), float('nan'), dtype=torch.float64, device=DEV)
    wts = None if w is None else (ctypes.c_float * len(w))(*w)
    _call('tha4_test_distill_tail', kind, _ptr(od), _ptr(imd), N, _ptr(td[0]), _ptr(td[1]), _ptr(td[2]),
          None if gd is None else _ptr_array(gd), wts, _ptr(d_out), _ptr(sums))
    torch.cuda.synchronize()
    return d_out.cpu().double(), sums.cpu()


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


@pytest.mark.parametrize('grid', list(GRIDS))
def test_body_loss_tail(oracle_clib, grid):
    N, R = 2, 512
    out7 = _out7(grid, N, 31)
    gi = torch.Generator().manual_seed(32)
    image = torch.rand(N, 4, R, R, generator=gi) * 2 - 1
    tie = (torch.arange(R * R).view(R, R) % 7 == 0).expand(N, R, R)
    _, (bl, _, _, wp, _) = D.body_outputs64(oracle_clib, out7, image)
    # colour ties: colour = T0 (and the blend 0.5 away from it); grid ties: grid_change = T3
    col = out7[..., 3:7].clone()
    col[tie] = (wp.detach().permute(0, 2, 3, 1)[tie] + 0.5).float()
    out7[..., 3:7] = col
    a = out7[..., 2]
    a[tie] = 0.5
    _, (bl, _, colv, wp, gc) = D.body_outputs64(oracle_clib, out7, image)
    T0 = _away(bl.detach(), 33)
    T0 = torch.where(tie[:, None], colv.detach().float(), T0)
    T2 = _away(wp.detach(), 34)
    T3 = _away(gc.detach(), 35)
    T3 = torch.where(tie[:, None], out7[..., 0:2].permute(0, 3, 1, 2), T3)
    w = [1.0, 2.0, 3.0, 4.0]
    d, sums = _tail(0, out7, image, N, (T0, T2, T3), w=w)
    rsums, rd = D.body_loss_ref(oracle_clib, out7, image, T0, T2, T3, w)
    for i in range(4):
        assert abs(sums[i].item() - rsums[i].item()) <= 1e-6 * rsums[i].item(), ('loss term %d' % i, sums[i].item(), rsums[i].item())
    assert bool((d[..., 7] == 0).all()), 'slot 7 of d_out7 must be exactly 0'
    rel = _rel(d[..., :7], rd[..., :7])
    print('\nbody loss tail, %s grid: rel L2 %.3e' % (grid, rel))
    assert rel <= 1e-6, rel
    nb, ng = N * 4 * R * R, N * 2 * R * R
    wx, wy, wz, ww = w[0] / nb, w[1] / nb, w[2] / ng, w[3] / nb
    al = out7[..., 2].double()
    amax = image.abs().amax(dim=(2, 3)).double()                     # [N, 4]
    dwp = (wx * (1 - al).abs() + wy)                                  # per pixel, per channel
    Mg = R / 2 * dwp * 2 * amax.sum(1).view(N, 1, 1) + wz
    Ma = (wx * (out7[..., 3:7].double().abs() + amax.view(N, 1, 1, 4))).sum(-1)
    Mc = wx * al.abs().unsqueeze(-1) + ww
    bound = 32 * D.U32 * torch.cat([Mg.unsqueeze(-1).expand(N, R, R, 2), Ma.unsqueeze(-1), Mc.expand(N, R, R, 4)], -1)
    _exceed('d out7', (d[..., :7] - rd[..., :7]).abs(), bound, ' (%s grid)' % grid)
    # exact ties give sgn(0) = 0: at a colour tie only the blend term remains (alpha = 1/2 there, so it is exact)
    dcol_tie = wx * 0.5 * torch.sign(bl.detach() - T0.double()).permute(0, 2, 3, 1)[tie]
    assert torch.equal(d[..., 3:7][tie], dcol_tie.float().double()), 'colour ties: d colour must be the blend term alone'
    cx, cy = _clamped(oracle_clib, out7[..., 0:2].permute(0, 3, 1, 2))
    assert bool((d[..., 0][cx & tie] == 0).all()) and bool((d[..., 1][cy & tie] == 0).all()), \
        'clamped samples at grid ties must have a zero grid gradient'


BODY_CH = (4, 1, 4, 4, 2)


@pytest.mark.parametrize('which', ['blended', 'alpha', 'color', 'warped', 'grid', 'all', 'none'])
@pytest.mark.parametrize('grid', ['random', 'mixed_clamp'])
def test_body_grad_tail(oracle_clib, which, grid):
    N, R = 2, 512
    out7 = _out7(grid, N, 41)
    image = torch.rand(N, 4, R, R, generator=torch.Generator().manual_seed(42)) * 2 - 1
    names = ['blended', 'alpha', 'color', 'warped', 'grid']
    g = [_randn((N, c, R, R), 43 + i, 1e-3) if which in (n, 'all') else None for i, (n, c) in enumerate(zip(names, BODY_CH))]
    d, _ = _tail(1, out7, image, N, g=None if which == 'none' else g)
    assert bool((d[..., 7] == 0).all()), 'slot 7 of d_out7 must be exactly 0'
    if which == 'none':
        assert bool((d == 0).all())
        return
    rd = D.body_grad_ref(oracle_clib, out7, image, g)
    rel = _rel(d[..., :7], rd[..., :7])
    print('\ngrad tail, %s upstream, %s grid: rel L2 %.3e' % (which, grid, rel))
    assert rel <= 1e-6, rel
    z = lambda t, c: torch.zeros(N, c, R, R, dtype=torch.float64) if t is None else t.double().abs()
    gbl, gal, gcol, gwp, ggr = [z(t, c) for t, c in zip(g, BODY_CH)]
    al = out7[..., 2].double().unsqueeze(1)
    amax = image.abs().amax(dim=(2, 3)).double().view(N, 4, 1, 1)
    dwp = gbl * (1 - al).abs() + gwp
    Mg = R / 2 * (dwp * 2 * amax).sum(1, keepdim=True) + ggr
    Ma = gal + (gbl * (out7[..., 3:7].permute(0, 3, 1, 2).double().abs() + amax)).sum(1, keepdim=True)
    Mc = gbl * al.abs() + gcol
    bound = 32 * D.U32 * torch.cat([Mg.expand(N, 2, R, R), Ma, Mc], 1).permute(0, 2, 3, 1)
    _exceed('d out7', (d[..., :7] - rd[..., :7]).abs(), bound, ' (%s upstream, %s grid)' % (which, grid))
    if g[4] is None:
        cx, cy = _clamped(oracle_clib, out7[..., 0:2].permute(0, 3, 1, 2))
        assert bool((d[..., 0][cx] == 0).all()) and bool((d[..., 1][cy] == 0).all()), 'clamped samples: grid gradient must be 0'


def test_face_loss_tail():
    N, R = 3, 128
    g = torch.Generator().manual_seed(51)
    out4 = torch.rand(N, R, R, 4, generator=g) * 2 - 1
    o = out4.permute(0, 3, 1, 2)
    target = _away(o.double(), 52)
    tie = torch.rand(N, 4, R, R, generator=g) < 0.1
    target[tie] = o[tie]                             # face output equal to the target
    mask = (torch.rand(N, 4, R, R, generator=g) < 0.5).float()
    mask[:, :, R // 2:] = torch.rand(N, 4, R // 2, R, generator=g)     # binary top half, fractional bottom half
    w = [1.0, 20.0]
    d, sums = _tail(2, out4, None, N, (target, mask, None), w=w)
    rsums, rd = D.face_loss_ref(out4, target, mask, w)
    for i in range(2):
        assert abs(sums[i].item() - rsums[i].item()) <= 1e-6 * rsums[i].item(), ('loss term %d' % i, sums[i].item(), rsums[i].item())
    rel = _rel(d, rd)
    print('\nface loss tail: rel L2 %.3e' % rel)
    assert rel <= 1e-6, rel
    nel = N * 4 * R * R
    bound = 4 * D.U32 * (w[0] / nel + w[1] / nel * mask.double().permute(0, 2, 3, 1))
    _exceed('d out4', (d - rd).abs(), bound)
    assert bool((d.permute(0, 3, 1, 2)[tie] == 0).all()), 'exact ties must give sgn(0) = 0'


# ------------------------------------------------------------------------------------------ Adam
def _adam_grads(n, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    mag = torch.pow(10.0, torch.rand(n, generator=g, device=DEV) * 15 - 12)      # 1e-12 .. 1e3 per entry
    return mag, g


def _cancel_term(opt, pt, m_old, grad, t, lr):
    """What the rounding of m = b1 m + (1 - b1) g can move an update by when the two terms cancel (the update's relative
    error is unbounded there): (lr / bc1) 2u (b1 |m| + (1 - b1) |g|) / (sqrt(v_hat) + eps), from torch's new state."""
    v = opt.state[pt]['exp_avg_sq'].double()
    denom = v.sqrt() / math.sqrt(1 - 0.999 ** t) + 1e-8
    return lr / (1 - 0.9 ** t) * 2 * D.U32 * (0.9 * m_old.double().abs() + 0.1 * grad.double().abs()) / denom


def test_adam_matches_torch():
    n = 2 * 148 * 8 * 256 + 12345                 # past two grid strides, not a multiple of one
    steps, lr = 2000, 1e-3
    mag, gen = _adam_grads(n, 61)
    zero = torch.zeros(n, dtype=torch.bool, device=DEV)
    zero[::97] = True
    p0 = torch.randn(n, generator=gen, device=DEV)
    ctx = _ctx()
    # (a) one step at a time from torch's state: |p - p_torch| <= 2e-5 |update| + 2 ulp(p)
    pt = torch.nn.Parameter(p0.clone())
    opt = torch.optim.Adam([pt], lr=lr, betas=(0.9, 0.999), eps=1e-8)
    pk, mk, vk = torch.empty(n, device=DEV), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    worst = 0.0
    for t in range(1, steps + 1):
        grad = torch.where(zero, 0.0, mag * torch.randn(n, generator=gen, device=DEV))
        st = opt.state.get(pt)
        pk.copy_(pt.data)
        if st:
            mk.copy_(st['exp_avg']); vk.copy_(st['exp_avg_sq'])
        m_old = mk.clone()
        before = pt.data.double()
        ctx.adam_step(pk, 2 * grad, mk, vk, lr, t, grad_scale=0.5)
        pt.grad = grad.clone()
        opt.step()
        upd = (pt.data.double() - before).abs()
        err = (pk.double() - pt.data.double()).abs()
        bound = 2e-5 * upd + 2 * D.ulp32(pt.data) + 2 * _cancel_term(opt, pt, m_old, grad, t, lr)
        r = (err / bound).max().item()
        worst = max(worst, r)
        if r > 1:
            _exceed('Adam step %d' % t, err, bound)
    print('\nAdam, one step from torch\'s state: worst err / bound %.3e over %d steps' % (worst, steps))
    # (b) a free-running trajectory: the per-step bound summed, plus one ulp per step for the two roundings of p; a rounding
    # of m decays by b1 per step, so it reaches at most 1 / (1 - b1) = 10 updates
    pt = torch.nn.Parameter(p0.clone())
    opt = torch.optim.Adam([pt], lr=lr, betas=(0.9, 0.999), eps=1e-8)
    pk, mk, vk = p0.clone(), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    gen.manual_seed(62)
    acc_upd = torch.zeros(n, dtype=torch.float64, device=DEV)
    acc_ulp = torch.zeros(n, dtype=torch.float64, device=DEV)
    acc_cancel = torch.zeros(n, dtype=torch.float64, device=DEV)
    for t in range(1, steps + 1):
        grad = torch.where(zero, 0.0, mag * torch.randn(n, generator=gen, device=DEV))
        st = opt.state.get(pt)
        m_old = st['exp_avg'].clone() if st else torch.zeros(n, device=DEV)
        before = pt.data.double()
        ctx.adam_step(pk, 2 * grad, mk, vk, lr, t, grad_scale=0.5)
        pt.grad = grad.clone()
        opt.step()
        acc_upd += (pt.data.double() - before).abs()
        acc_ulp += D.ulp32(pt.data)
        acc_cancel += _cancel_term(opt, pt, m_old, grad, t, lr)
    torch.cuda.synchronize()
    assert torch.equal(pk[zero], p0[zero]), 'entries with zero gradient moved'
    assert bool((mk[zero] == 0).all()) and bool((vk[zero] == 0).all())
    err = (pk.double() - pt.data.double()).abs()
    bound = 2e-5 * acc_upd + acc_ulp + 2 * D.ulp32(pt.data) + 2 * 10 * acc_cancel
    print('Adam trajectory: worst err / bound %.3e, err / accumulated update %.3e' % ((err / bound).max().item(),
                                                                                        (err / acc_upd.clamp_min(1e-30))[~zero].max().item()))
    _exceed('Adam after %d steps' % steps, err, bound)
