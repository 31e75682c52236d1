"""Options belong to the context they are set on (-m gpu): a switch set on one context changes neither the kernels nor the
plans another context runs, the retired switches are unknown options, out-of-range values are rejected, and an option
reaches a call made on another thread (the library binds the context's options per call, not per thread)."""
import ctypes
import threading

import pytest
import torch

from oracle import synth
from tha4_b200._lib import Context, Tha4Error, _ptr
from tha4_b200.charmodel import CharacterBank

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
# the retired switches, each with the value it had by default (a library that still knows a name keeps its behaviour)
RETIRED = {'side_stream': 1, 'tc_stride2': 1, 'small_bn': 1, 'attn_split16': 0, 'attn_mma': 1, 'pdl': 1}


def _conv_plan(ctx):
    """The plan record of tha4_test_conv_forward_ex (plan[0]: 1 halo / 2 tensor-core / 3 mma.sync; plan[3]: consumer
    warpgroups of a halo launch) for a 3x3 conv, 64 -> 64 channels, on one raw f16 32 x 32 map: 8 tiles of 128 pixels,
    too few for the automatic plan to take 256-pixel tiles."""
    g = torch.Generator().manual_seed(7)
    N, H, W, C = 1, 32, 32, 64
    x = torch.randn(N, H, W, C, generator=g).half().to(DEV)
    w = (torch.randn(C, C, 3, 3, generator=g) / 24.0).to(DEV)
    b = torch.randn(C, generator=g).to(DEV)
    out = torch.empty(N, H, W, C, device=DEV)
    plan = (ctypes.c_int * 10)()
    with torch.cuda.device(DEV):
        ctx._call('tha4_test_conv_forward_ex', 0, _ptr(w), _ptr(b), C, C, _ptr(None), _ptr(None), 0, _ptr(x), C, N, H, W,
                  _ptr(None), 0, _ptr(out), C, _ptr(None), 0, _ptr(None), 0, 0, ctypes.c_int64(0), _ptr(None), 0, 0,
                  _ptr(None), 0, 0, ctypes.c_int64(0), 0, 0, 0, _ptr(None), _ptr(None), _ptr(None), _ptr(None), 0, 0, plan,
                  ctx._stream())
        torch.cuda.synchronize()
    return list(plan)


# option, value, default value, (plan[0], plan[3]) it gives: the tensor-core kernel / the halo kernel on 256-pixel tiles
SWITCHES = [('halo_conv', 0, 1, (2, 0)), ('halo_m256', 1, -1, (1, 2))]


@pytest.mark.parametrize('option,value,default,want', SWITCHES)
def test_a_switch_changes_the_plan_of_its_own_context_only(option, value, default, want):
    a, b = Context(DEV), Context(DEV)
    before = _conv_plan(b)
    assert (before[0], before[3]) == (1, 1), before               # halo kernel, 128-pixel tiles
    try:
        a.set_option(option, value)
        changed, other = _conv_plan(a), _conv_plan(b)
    finally:
        a.set_option(option, default)
    assert (changed[0], changed[3]) == want, changed
    assert other == before, other


def test_a_bank_keeps_posing_when_another_context_retires_the_wgmma_students():
    image, sds = synth.synthetic_image(1, 1)[0], synth.student_state_dicts(1)
    bank = CharacterBank(DEV, 1)
    bank.add('synthetic_1', image, sds['face_morpher'], sds['body_morpher'])
    poses = synth.random_poses(2, seed=60).to(DEV)
    with torch.no_grad():
        before = [t.clone() for t in bank.get_posing_outputs([0, 0], poses)]
        other = Context(DEV)
        try:
            other.set_option('siren_tc', 0)
            after = bank.get_posing_outputs([0, 0], poses)
        finally:
            other.set_option('siren_tc', 1)
    for i, (x, y) in enumerate(zip(after, before)):
        assert torch.equal(x, y), i


@pytest.fixture(scope='module')
def ctx():
    return Context(DEV)


@pytest.mark.parametrize('name', sorted(RETIRED))
def test_retired_switches_are_unknown_options(ctx, name):
    with pytest.raises(Tha4Error, match='unknown option'):
        ctx.set_option(name, RETIRED[name])


@pytest.mark.parametrize('name,value', [('halo_m256', 2), ('halo_m256', -2), ('halo_ctas', 0), ('halo_ctas', 3),
                                        ('halo_cs', 0), ('halo_cs', -2), ('microbatch', 0), ('microbatch', 1025)])
def test_out_of_range_values_are_rejected(ctx, name, value):
    with pytest.raises(Tha4Error, match=name):
        ctx.set_option(name, value)


def test_an_option_reaches_a_call_on_another_thread(ctx):
    result = []
    try:
        ctx.set_option('halo_m256', 1)
        t = threading.Thread(target=lambda: result.append(_conv_plan(ctx)))
        t.start()
        t.join()
    finally:
        ctx.set_option('halo_m256', -1)
    assert len(result) == 1, 'the call on the second thread raised'
    assert result[0][0] == 1 and result[0][3] == 2, result[0]
