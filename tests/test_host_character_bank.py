"""Argument checks of tha4_b200.charmodel.CharacterBank (no GPU): the library context is replaced by a stub that records
the bank calls, so every refusal below is shown to happen before anything reaches the library."""
import pytest
import torch

from tha4_b200 import _lib, synthetic
from tha4_b200._lib import Tha4Error
from tha4_b200.charmodel import CharacterBank


class StubCtx:
    device = torch.device('cpu')

    def __init__(self):
        self.created = []
        self.set = []
        self.forwards = []

    def bank_create(self, capacity):
        self.created.append(capacity)

    def bank_set_character(self, slot, face_sd, body_sd, image):
        assert image.shape == (4, 512, 512) and image.dtype == torch.float32
        self.set.append(slot)

    def bank_forward(self, char_ids, pose, half=False):
        assert all(type(i) is int for i in char_ids) and pose.shape == (len(char_ids), 45) and not pose.requires_grad
        self.forwards.append((list(char_ids), half))
        B = len(char_ids)
        return [torch.full((B, c, 2, 2), float(i)) for i, c in enumerate((4, 1, 4, 4, 2, 4))]

    def frame_to_srgb8(self, frame, background=None, rint=False):
        return ('srgb8', frame, background, rint)


@pytest.fixture(scope='module')
def sds():
    return synthetic.student_state_dicts(3)


IMAGE = torch.zeros(4, 512, 512)


def _bank(sds, capacity=4, filled=2):
    stub = StubCtx()
    bank = CharacterBank(torch.device('cpu'), capacity, context=stub)
    for i in range(filled):
        assert bank.add('c%d' % i, IMAGE, sds['face_morpher'], sds['body_morpher']) == i
    return bank, stub


def test_slots_fill_in_order_and_replace_keeps_the_others(sds):
    bank, stub = _bank(sds)
    assert stub.created == [4] and stub.set == [0, 1] and bank.names == ['c0', 'c1', None, None]
    bank.replace(0, 'other', IMAGE, sds['face_morpher'], sds['body_morpher'])
    assert stub.set == [0, 1, 0] and bank.names == ['other', 'c1', None, None]
    bank.replace(3, 'last', IMAGE, sds['face_morpher'], sds['body_morpher'])
    assert bank.add('third', IMAGE, sds['face_morpher'], sds['body_morpher']) == 2
    with pytest.raises(Tha4Error, match='filled'):
        bank.add('fifth', IMAGE, sds['face_morpher'], sds['body_morpher'])
    with pytest.raises(Tha4Error, match='slot 4'):
        bank.replace(4, 'x', IMAGE, sds['face_morpher'], sds['body_morpher'])
    with pytest.raises(Tha4Error, match='capacity'):
        CharacterBank(torch.device('cpu'), 0, context=StubCtx())


def test_wrong_state_dicts_and_images_are_refused_before_the_upload(sds):
    bank, stub = _bank(sds, filled=0)
    face, body = sds['face_morpher'], sds['body_morpher']
    with pytest.raises(Tha4Error, match='face_morpher state_dict'):
        bank.add('swapped', IMAGE, body, face)
    missing = {k: v for k, v in body.items() if k != 'last_linear.bias'}
    with pytest.raises(Tha4Error, match='last_linear.bias'):
        bank.add('missing', IMAGE, face, missing)
    with pytest.raises(Tha4Error, match='unexpected'):
        bank.add('extra', IMAGE, dict(face, extra=torch.zeros(1)), body)
    reshaped = dict(body)
    reshaped['siren_layers.0.0.linear.weight'] = torch.zeros(360, 46, 1, 1)
    with pytest.raises(Tha4Error, match='shape'):
        bank.add('reshaped', IMAGE, face, reshaped)
    with pytest.raises(Tha4Error, match='image'):
        bank.add('small', torch.zeros(4, 256, 256), face, body)
    assert stub.set == [] and bank.names == [None] * 4


@pytest.mark.parametrize('ids, what', [([-1], 'not a slot'), ([0, 4], 'not a slot'), ([2], 'no character'), ([0, 3, 1], 'no character'),
                                       ([], 'empty'), ([0.0], 'not an integer'), ([True], 'not an integer'),
                                       (torch.tensor([0.0, 1.0]), 'integer tensor'), (torch.tensor([[0, 1]]), 'integer tensor'),
                                       (torch.tensor([0, 7]), 'not a slot')])
def test_bad_character_ids_are_refused_before_the_call(sds, ids, what):
    bank, stub = _bank(sds)
    with pytest.raises(Tha4Error, match=what):
        bank.get_posing_outputs(ids, torch.zeros(max(len(ids), 1), 45))
    assert stub.forwards == []


def test_ids_as_list_and_as_tensor_reach_the_library_alike(sds):
    bank, stub = _bank(sds)
    poses = torch.zeros(3, 45)
    outs = bank.get_posing_outputs([1, 0, 1], poses)
    assert len(outs) == 6
    bank.get_posing_outputs(torch.tensor([1, 0, 1]), poses)
    bank.get_posing_outputs(torch.tensor([1, 0, 1], dtype=torch.int32), poses, half=True)
    assert stub.forwards == [([1, 0, 1], False), ([1, 0, 1], False), ([1, 0, 1], True)]
    assert bank.pose([0], torch.zeros(45)).shape == (1, 4, 2, 2)               # a [45] pose is a batch of one
    assert torch.equal(bank.pose([0, 1], poses[:2], output_index=4), torch.full((2, 2, 2, 2), 4.0))
    tag, frame, background, rint = bank.pose_to_srgb8([0, 1], poses[:2], background='green')
    assert tag == 'srgb8' and frame.shape == (2, 4, 2, 2) and background == 'green' and rint is False
    with pytest.raises(Tha4Error, match=r'\[2,45\]'):
        bank.get_posing_outputs([0, 1], poses)


def test_an_input_that_requires_grad_is_refused(sds):
    bank, stub = _bank(sds)
    poses = torch.zeros(1, 45, requires_grad=True)
    with pytest.raises(Tha4Error, match='INTEGRATION.md'):
        bank.get_posing_outputs([0], poses)
    assert stub.forwards == []
    with torch.no_grad():
        outs = bank.get_posing_outputs([0], poses)
    assert stub.forwards == [([0], False)] and all(o.grad_fn is None for o in outs)


def test_the_binding_lists_the_bank_entries():
    for name in ('tha4_bank_create', 'tha4_bank_destroy', 'tha4_bank_set_character', 'tha4_bank_forward'):
        assert name in _lib.EXPORTED_SYMBOLS
    for name in ('bank_create', 'bank_destroy', 'bank_set_character', 'bank_forward'):
        assert callable(getattr(_lib.Context, name))
