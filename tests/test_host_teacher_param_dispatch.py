"""Dispatch of the encoder-decoder teachers' opt-in parameter gradients (no GPU): a module that is not trainable keeps the
input-gradient rule; a trainable one takes the autograd path for plain inputs, and its backward makes ONE library call that
fills a flat state_dict-order d_params, handed out per parameter (None for frozen ones).  The library context is replaced
by a stub that records the calls and writes a ramp into d_params."""
import types

import pytest
import torch

from tha4_b200.nn.eyebrow_decomposer.eyebrow_decomposer_00 import EyebrowDecomposer00
from tha4_b200.nn.eyebrow_morphing_combiner.eyebrow_morphing_combiner_00 import EyebrowMorphingCombiner00
from tha4_b200.nn.face_morpher.face_morpher_08 import FaceMorpher08

CLASSES = (EyebrowDecomposer00, EyebrowMorphingCombiner00, FaceMorpher08)


def _ramp(first, n):
    # exactly representable in fp32 (the buffers hold 31 M floats)
    return (torch.arange(first, first + n, dtype=torch.int64) % 4099).float()


class StubCtx:
    def __init__(self, module):
        self.calls = []
        self.n = sum(p.numel() for p in module.parameters())

    def param_count(self, net):
        return self.n

    def _outs(self, name, B):
        self.calls.append(name)
        return [torch.full((B, 4, 8, 8), float(i)) for i in range(6 if name == 'decomposer' else 8)]

    def eyebrow_decomposer(self, image):
        return self._outs('decomposer', image.shape[0])

    def eyebrow_morphing_combiner(self, background_layer, eyebrow_layer, pose):
        return self._outs('combiner', background_layer.shape[0])

    def face_morpher(self, image, pose):
        return self._outs('face', image.shape[0])

    def _bwd(self, name, d_params, **inputs):
        self.calls.append((name, d_params is None, tuple(k for k, v in inputs.items() if v is not None)))
        if d_params is not None:
            assert d_params.shape == (self.n,)
            d_params.copy_(_ramp(0, self.n))
        for v in inputs.values():
            if v is not None:
                v.fill_(7.0)

    def eyebrow_decomposer_backward(self, image, grads, d_image=None, d_params=None):
        self._bwd('decomposer_backward', d_params, d_image=d_image)

    def eyebrow_morphing_combiner_backward(self, bg, eb, pose, grads, d_background_layer=None, d_eyebrow_layer=None, d_pose=None,
                                           d_params=None):
        self._bwd('combiner_backward', d_params, d_background_layer=d_background_layer, d_eyebrow_layer=d_eyebrow_layer, d_pose=d_pose)

    def face_morpher_backward(self, image, pose, grads, d_image=None, d_pose=None, d_params=None):
        self._bwd('face_backward', d_params, d_image=d_image, d_pose=d_pose)


def _with_stub(module):
    stub = StubCtx(module)
    module.sync_weights = lambda: stub
    return module, stub


def _inputs(cls, rg=False):
    if cls is EyebrowDecomposer00:
        return (torch.zeros(2, 4, 8, 8, requires_grad=rg),)
    if cls is EyebrowMorphingCombiner00:
        return (torch.zeros(2, 4, 8, 8), torch.zeros(2, 4, 8, 8), torch.zeros(2, 12, requires_grad=rg))
    return (torch.zeros(2, 4, 8, 8), torch.zeros(2, 27, requires_grad=rg))


@pytest.mark.parametrize('cls', CLASSES)
def test_not_trainable_is_unchanged(cls):
    m, stub = _with_stub(cls())
    assert not m.is_trainable()
    outs = m(*_inputs(cls))
    assert all(o.grad_fn is None for o in outs) and len(stub.calls) == 1


@pytest.mark.parametrize('cls', CLASSES)
def test_trainable_plain_inputs_fill_every_grad_from_one_call(cls):
    m, stub = _with_stub(cls())
    assert m.trainable_(True) is m and m.is_trainable()
    outs = m(*_inputs(cls))
    assert all(o.grad_fn is not None for o in outs) and len(stub.calls) == 1
    sum(o.sum() for o in outs).backward()
    assert len(stub.calls) == 2 and stub.calls[1][1] is False and stub.calls[1][2] == ()     # d_params only
    off = 0
    for k, p in m.named_parameters():
        assert p.grad is not None and p.grad.shape == p.shape, k
        assert torch.equal(p.grad.flatten(), _ramp(off, p.numel())), k
        off += p.numel()
    assert off == stub.n


@pytest.mark.parametrize('cls', CLASSES)
def test_frozen_parameters_get_none_and_inputs_come_from_the_same_call(cls):
    m, stub = _with_stub(cls().trainable_())
    params = list(m.parameters())
    for p in params[::2]:
        p.requires_grad_(False)
    ins = _inputs(cls, rg=True)
    outs = m(*ins)
    sum(o.sum() for o in outs).backward()
    assert len(stub.calls) == 2 and stub.calls[1][1] is False and len(stub.calls[1][2]) == 1
    off = 0
    for i, p in enumerate(params):
        if i % 2 == 0:
            assert p.grad is None
        else:
            assert torch.equal(p.grad.flatten(), _ramp(off, p.numel()))
        off += p.numel()
    rg = [t for t in ins if t.requires_grad][0]
    assert torch.all(rg.grad == 7.0)


@pytest.mark.parametrize('cls', CLASSES)
def test_trainable_under_no_grad_or_all_frozen_takes_the_single_call(cls):
    m, stub = _with_stub(cls().trainable_())
    with torch.no_grad():
        outs = m(*_inputs(cls))
    assert all(o.grad_fn is None for o in outs) and len(stub.calls) == 1
    m.requires_grad_(False)
    outs = m(*_inputs(cls))
    assert all(o.grad_fn is None for o in outs) and len(stub.calls) == 2
    m.trainable_(False).requires_grad_(True)
    outs = m(*_inputs(cls))
    assert all(o.grad_fn is None for o in outs) and len(stub.calls) == 3


def test_parameters_are_in_state_dict_order():
    for cls in CLASSES:
        m = cls()
        assert [k for k, _ in m.named_parameters()] == list(m.state_dict().keys())


def test_posers_take_the_composed_path_for_trainable_teachers():
    from tha4_b200.poser.modes import mode_07
    proto = mode_07.FiveStepPoserComputationProtocol
    mods = {'eyebrow_decomposer': EyebrowDecomposer00(), 'eyebrow_morphing_combiner': EyebrowMorphingCombiner00(),
            'face_morpher': FaceMorpher08()}
    state = types.SimpleNamespace(modules=mods)
    assert not proto._trains_teacher(state)
    for k in mods:
        mods[k].trainable_()
        assert proto._trains_teacher(state), k
        with torch.no_grad():
            assert not proto._trains_teacher(state)
        mods[k].requires_grad_(False)
        assert not proto._trains_teacher(state), k
        mods[k].requires_grad_(True).trainable_(False)
    # the U-Nets of mode_07 are not asked
    state.modules = dict(mods, body_morpher=object(), upscaler=object())
    assert not proto._trains_teacher(state)
