"""The character bank on the GPU: a batch that mixes characters returns, for every frame, bit for bit what a mode_14 poser
holding that frame's character alone returns (the arithmetic of a tile and its order do not depend on where the tile's
weights come from), whatever the order of the batch; bad character ids are errors before any launch; and the
one-character student path is not changed by a bank on the same context."""
import os

import pytest
import torch

from oracle import image_io, synth
from oracle import tha4_oracle as O
from tha4_b200._lib import Context, Tha4Error
from tha4_b200.charmodel import CharacterBank
from tha4_b200.poser.modes import mode_14

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
DATA = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'data')
MIXED_IDS = [0, 1, 2, 3, 3, 2, 1, 0, 0, 0, 1, 1, 2, 3, 2, 0]


def _shipped(name):
    """A shipped character's state_dicts and image.  lambda_01's body checkpoint is stored with its weights rounded to
    fp16 (half the size of the reference's file); widened here, those fp32 values are the character the
    bank, the one-character poser and the CPU oracle all see."""
    sds = {}
    for k in ('face_morpher', 'body_morpher'):
        path = os.path.join(DATA, '%s_%s.pt' % (name, k))
        if not os.path.exists(path):
            path = os.path.join(DATA, '%s_%s_f16.pt' % (name, k))
        sds[k] = {key: v.float() for key, v in torch.load(path, map_location='cpu').items()}
    return sds, image_io.load_rgba_png(os.path.join(DATA, '%s.png' % name))


@pytest.fixture(scope='module')
def characters():
    """(name, state_dicts, image) of the two shipped characters and two seeded synthetic students."""
    chars = [('lambda_00',) + _shipped('lambda_00'), ('lambda_01',) + _shipped('lambda_01')]
    for seed in (1, 2):
        chars.append(('synthetic_%d' % seed, synth.student_state_dicts(seed), synth.synthetic_image(seed, 1)[0]))
    return chars


def _fill(bank, characters):
    for name, sds, image in characters:
        bank.add(name, image, sds['face_morpher'], sds['body_morpher'])
    return bank


@pytest.fixture(scope='module')
def bank(characters):
    return _fill(CharacterBank(DEV, 6), characters)          # slots 4 and 5 stay empty


@pytest.fixture(scope='module')
def posers(characters):
    return [mode_14.create_poser(DEV, state_dicts=sds) for _, sds, _ in characters]


def _alone(posers, characters, c, poses, half=False):
    """The one-character poser of character c at `poses` [b,45] (on the device)."""
    images = characters[c][2].to(DEV).unsqueeze(0).expand(poses.shape[0], -1, -1, -1).contiguous()
    with torch.no_grad():
        return posers[c].get_posing_outputs(images.half() if half else images, poses)


def _assert_bitwise(what, got, want):
    assert len(got) == len(want) == 6
    for i, (a, b) in enumerate(zip(got, want)):
        assert a.dtype == b.dtype and a.shape == b.shape, (what, i, a.dtype, b.dtype, a.shape, b.shape)
        assert torch.equal(a, b), (what, i, (a.float() - b.float()).abs().max().item())


@pytest.mark.parametrize('half', [False, True])
@pytest.mark.parametrize('B', [1, 3, 64])
def test_one_slot_equals_the_poser(characters, posers, B, half):
    name, sds, image = characters[0]
    one = CharacterBank(DEV, 1)
    one.add(name, image, sds['face_morpher'], sds['body_morpher'])
    poses = synth.random_poses(B, seed=40 + B).to(DEV)
    got = one.get_posing_outputs([0] * B, poses, half=half)
    assert all(t.dtype == (torch.float16 if half else torch.float32) for t in got)
    _assert_bitwise('one slot, B = %d' % B, got, _alone(posers, characters, 0, poses, half))


@pytest.mark.parametrize('half', [False, True])
def test_a_mixed_batch_equals_each_character_alone(bank, characters, posers, half):
    poses = synth.random_poses(len(MIXED_IDS), seed=51).to(DEV)
    got = bank.get_posing_outputs(MIXED_IDS, poses, half=half)
    ids = torch.tensor(MIXED_IDS)
    for c in range(4):
        frames = (ids == c).nonzero().flatten().to(DEV)
        want = _alone(posers, characters, c, poses[frames], half)
        _assert_bitwise('character %d in the mixed batch' % c, [t[frames] for t in got], want)
    # the four characters differ, so a frame taken from a neighbour's slot could not pass the above
    assert not torch.equal(got[0][0], got[0][1])


def test_order_does_not_matter(bank):
    poses = synth.random_poses(len(MIXED_IDS), seed=52).to(DEV)
    perm = torch.randperm(len(MIXED_IDS), generator=torch.Generator().manual_seed(7))
    got = bank.get_posing_outputs(MIXED_IDS, poses)
    permuted = bank.get_posing_outputs(torch.tensor(MIXED_IDS)[perm], poses[perm.to(DEV)])
    _assert_bitwise('permuted batch', permuted, [t[perm.to(DEV)] for t in got])


# the student tolerances tests/test_gpu_parity.py asserts for lambda_00: mean |error| per output, then max |error| of
# grid_change (normalised coordinates) and of alpha / colour change / face
STUDENT_MEAN_TOL = [4e-3, 2e-3, 2e-3, 4e-3, 1e-3, 2e-3]


def test_parity_with_the_reference_arithmetic_on_lambda_01(bank, characters):
    _, sds, image = characters[1]
    poses = synth.random_poses(2, seed=1234)
    got = [t.cpu() for t in bank.get_posing_outputs([1, 1], poses.to(DEV))]
    with torch.no_grad():
        for p in range(2):
            refs = O.mode_14_outputs(sds, image, poses[p])
            errs = [(a[p:p + 1].double() - b.double()).abs() for a, b in zip(got, refs)]
            assert len(refs) == 6 and all(e.shape[0] == 1 for e in errs)
            for i, e in enumerate(errs):
                assert e.mean().item() <= STUDENT_MEAN_TOL[i], (p, i, e.mean().item())
            assert errs[4].max().item() <= 1e-2, (p, errs[4].max().item())
            assert max(errs[i].max().item() for i in (1, 2, 5)) <= 0.1, p


def test_replacing_a_slot_leaves_the_others_unchanged(characters, posers):
    b = _fill(CharacterBank(DEV, 4), characters[:3])           # slots: lambda_00, lambda_01, synthetic_1
    ids = [0, 1, 2, 1, 0, 2]
    poses = synth.random_poses(len(ids), seed=53).to(DEV)
    before = b.get_posing_outputs(ids, poses)
    name, sds, image = characters[3]
    b.replace(1, name, image, sds['face_morpher'], sds['body_morpher'])
    after = b.get_posing_outputs(ids, poses)
    keep, moved = torch.tensor([0, 2, 4, 5], device=DEV), torch.tensor([1, 3], device=DEV)
    _assert_bitwise('slots 0 and 2 after replacing slot 1', [t[keep] for t in after], [t[keep] for t in before])
    _assert_bitwise('the replaced slot', [t[moved] for t in after], _alone(posers, characters, 3, poses[moved]))
    assert not torch.equal(after[0][1], before[0][1])


@pytest.mark.parametrize('ids', [[0, -1], [6, 0], [0, 1, 4], [1 << 30]])
def test_bad_ids_are_errors_before_any_launch(bank, ids):
    ctx = bank.get_context()
    poses = synth.random_poses(len(ids), seed=54).to(DEV)
    torch.cuda.synchronize()
    launches = ctx.counter('kernel_launches')
    with pytest.raises(Tha4Error, match='not a slot|no character'):
        bank.get_posing_outputs(ids, poses)
    with pytest.raises(Tha4Error, match='tha4_bank_forward failed.*(is not 0..5|holds no character)'):
        ctx.bank_forward(ids, poses)                           # the library's own check, past the Python one
    assert ctx.counter('kernel_launches') == launches
    torch.cuda.synchronize()
    assert len(bank.get_posing_outputs([0], poses[:1])) == 6   # the context is still usable


def test_the_bank_needs_the_wgmma_kernels(bank):
    ctx = bank.get_context()
    poses = synth.random_poses(1, seed=55).to(DEV)
    ctx.set_option('siren_tc', 0)
    try:
        with pytest.raises(Tha4Error, match='siren_tc = 1'):
            bank.get_posing_outputs([0], poses)
    finally:
        ctx.set_option('siren_tc', 1)


def test_the_single_character_path_is_untouched(characters):
    _, sds, image = characters[0]
    poser = mode_14.create_poser(DEV, state_dicts=sds)
    poses = synth.random_poses(64, seed=56).to(DEV)
    images = image.to(DEV).unsqueeze(0).expand(64, -1, -1, -1).contiguous()
    with torch.no_grad():
        before = [t.clone() for t in poser.get_posing_outputs(images, poses)]
    b = _fill(CharacterBank(DEV, 4, context=poser.get_context()), characters[1:3])
    b.get_posing_outputs([1, 0, 1], poses[:3])
    with torch.no_grad():
        after = poser.get_posing_outputs(images, poses)
    _assert_bitwise('student_forward after a bank call on the same context', after, before)
    poser.get_context().bank_destroy()
    with pytest.raises(Tha4Error, match='tha4_bank_create'):
        poser.get_context().bank_forward([0], poses[:1])
    with torch.no_grad():
        _assert_bitwise('student_forward after the bank is gone', poser.get_posing_outputs(images, poses), before)
