"""Dispatch rule of the SIREN student modules (no GPU): without grad mode, or with neither a parameter nor an input
requiring grad, forward is the single library call; otherwise it goes through the module's autograd.Function, whose
backward requests exactly the gradients autograd needs.  The library context is replaced by a stub that records the
forward calls and, for every backward call, which outputs were requested."""
import pytest
import torch

from tha4_b200._lib import Tha4Error
from tha4_b200.nn.siren.face_morpher.siren_face_morpher_00 import SirenFaceMorpher00
from tha4_b200.nn.siren.morpher.siren_morpher_03 import SirenMorpher03


class StubCtx:
    SIREN_MORPHER_SPECS = [(4, 8), (1, 8), (4, 8), (4, 8), (2, 8)]
    device = torch.device('cpu')

    def __init__(self):
        self.forwards = []
        self.backwards = []

    def _outs(self, B):
        return [torch.full((B, c, s, s), float(i)) for i, (c, s) in enumerate(self.SIREN_MORPHER_SPECS)]

    def siren_morpher(self, image, pose):
        self.forwards.append('body')
        return self._outs(image.shape[0])

    def siren_morpher_into(self, image, pose, outs):
        self.forwards.append('body')
        for o, v in zip(outs, self._outs(image.shape[0])):
            o.copy_(v)
        return outs

    def siren_face_morpher(self, pose):
        self.forwards.append('face')
        return torch.ones(pose.shape[0], 4, 8, 8)

    def _record(self, **outputs):
        self.backwards.append({k for k, v in outputs.items() if v is not None})
        for v in outputs.values():
            if v is not None:
                v.fill_(1.0)

    def siren_morpher_backward(self, image, pose, grad_outputs, *, grid_change=None, alpha=None, params=None, grads=None,
                               d_image=None, d_pose=None):
        assert (grid_change is not None) == (d_image is not None or d_pose is not None)
        self._record(grads=grads, d_image=d_image, d_pose=d_pose)

    def siren_face_morpher_backward(self, pose, grad_output, params, *, grads=None, d_pose=None):
        self._record(grads=grads, d_pose=d_pose)


def _with_stub(module, frozen):
    stub = StubCtx()
    module.sync_weights = lambda: stub
    module.requires_grad_(not frozen)
    return module, stub


def _body_inputs(image_rg=False, pose_rg=False):
    return torch.zeros(1, 4, 512, 512, requires_grad=image_rg), torch.zeros(1, 45, requires_grad=pose_rg)


def test_plain_inputs_and_no_grad_take_the_single_call():
    for frozen in (False, True):
        body, stub = _with_stub(SirenMorpher03(), frozen)
        with torch.no_grad():
            outs = body(*_body_inputs(True, True))
        assert all(o.grad_fn is None for o in outs) and stub.forwards == ['body']
        face, fstub = _with_stub(SirenFaceMorpher00(), frozen)
        with torch.no_grad():
            out = face(torch.zeros(1, 39, requires_grad=True))
        assert out.grad_fn is None and fstub.forwards == ['face']
    body, stub = _with_stub(SirenMorpher03(), frozen=True)              # grad mode on, frozen, plain inputs
    assert all(o.grad_fn is None for o in body(*_body_inputs())) and stub.forwards == ['body']
    face, fstub = _with_stub(SirenFaceMorpher00(), frozen=True)
    assert face(torch.zeros(1, 39)).grad_fn is None and fstub.forwards == ['face']
    assert stub.backwards == [] and fstub.backwards == []


def test_trainable_module_requests_parameter_gradients_only():
    body, stub = _with_stub(SirenMorpher03(), frozen=False)
    outs = body(*_body_inputs())
    assert all(o.grad_fn is not None for o in outs) and stub.forwards == ['body']
    assert len({o.data_ptr() for o in outs}) == len(outs)              # one allocation per output
    outs[0].sum().backward()
    assert stub.backwards == [{'grads'}]
    assert all(p.grad is not None for p in body.parameters())
    face, fstub = _with_stub(SirenFaceMorpher00(), frozen=False)
    out = face(torch.zeros(2, 39))
    assert out.grad_fn is not None
    out.sum().backward()
    assert fstub.backwards == [{'grads'}]
    assert all(p.grad is not None for p in face.parameters())


@pytest.mark.parametrize('image_rg, pose_rg, requested', [(True, False, {'d_image'}), (False, True, {'d_pose'}),
                                                           (True, True, {'d_image', 'd_pose'})])
def test_frozen_body_requests_exactly_the_input_gradients(image_rg, pose_rg, requested):
    body, stub = _with_stub(SirenMorpher03(), frozen=True)
    image, pose = _body_inputs(image_rg, pose_rg)
    outs = body(image, pose)
    assert all(o.grad_fn is not None for o in outs)
    outs[3].sum().backward()
    assert stub.backwards == [requested]
    assert (image.grad is not None) == image_rg and (pose.grad is not None) == pose_rg
    assert all(p.grad is None for p in body.parameters())


def test_frozen_face_requests_the_pose_gradient_only():
    face, stub = _with_stub(SirenFaceMorpher00(), frozen=True)
    pose = torch.zeros(2, 39, requires_grad=True)
    face(pose).sum().backward()
    assert stub.backwards == [{'d_pose'}] and pose.grad.shape == (2, 39)
    assert all(p.grad is None for p in face.parameters())


def test_trainable_module_refuses_input_gradients_before_any_call():
    for image_rg, pose_rg in ((True, False), (False, True)):
        body, stub = _with_stub(SirenMorpher03(), frozen=False)
        with pytest.raises(Tha4Error, match='image' if image_rg else 'pose'):
            body(*_body_inputs(image_rg, pose_rg))
        assert stub.forwards == [] and stub.backwards == []
    face, fstub = _with_stub(SirenFaceMorpher00(), frozen=False)
    with pytest.raises(Tha4Error, match='pose'):
        face(torch.zeros(1, 39, requires_grad=True))
    assert fstub.forwards == [] and fstub.backwards == []


def test_inplace_ops_on_outputs():
    """The parameter path leaves the outputs free for in-place ops; the input path saves the returned alpha / grid_change
    for d(image), so an in-place write to them fails the backward."""
    body, stub = _with_stub(SirenMorpher03(), frozen=False)
    outs = body(*_body_inputs())
    outs[1].mul_(2.0)
    outs[0].sum().backward()
    assert stub.backwards == [{'grads'}]
    body, stub = _with_stub(SirenMorpher03(), frozen=True)
    outs = body(*_body_inputs(image_rg=True))
    outs[1].mul_(2.0)
    with pytest.raises(RuntimeError, match='inplace'):
        outs[0].sum().backward()
    assert stub.backwards == []
    for frozen in (False, True):
        face, fstub = _with_stub(SirenFaceMorpher00(), frozen)
        out = face(torch.zeros(1, 39, requires_grad=frozen))
        out.clamp_(-1.0, 1.0)
        out.sum().backward()
        assert fstub.backwards == [{'d_pose'} if frozen else {'grads'}]
