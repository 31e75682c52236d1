"""Dispatch rule of Morpher00 (no GPU): without grad mode, or with inputs that do not require grad, forward is today's single
library call; only with grad mode on and the image or the pose requiring grad does it go through the autograd.Function, and
only then do the outputs carry a grad_fn.  The library context is replaced by a stub that records the calls."""
import pytest
import torch

from tha4_b200._lib import Tha4Error
from tha4_b200.nn.morpher.morpher_00 import Morpher00

SPECS = [(4, 256), (1, 256), (4, 256), (2, 256), (4, 256)]


class StubCtx:
    def __init__(self):
        self.calls = []

    def morpher(self, image, pose):
        self.calls.append(('morpher',))
        return [torch.full((image.shape[0], c, s, s), float(i)) for i, (c, s) in enumerate(SPECS)]

    def morpher_backward(self, image, pose, grad_outputs, d_image=None, d_pose=None):
        self.calls.append(('backward', d_image is not None, d_pose is not None))
        if d_image is not None:
            d_image.fill_(1.0)
        if d_pose is not None:
            d_pose.fill_(2.0)


def _module():
    m = Morpher00()
    stub = StubCtx()
    m.sync_weights = lambda: stub
    return m, stub


def _inputs(image_rg=False, pose_rg=False):
    return torch.zeros(1, 4, 256, 256, requires_grad=image_rg), torch.zeros(1, 6, requires_grad=pose_rg)


def test_plain_inputs_and_no_grad_take_the_single_call():
    m, stub = _module()
    outs = m(*_inputs())                                 # grad mode on, plain inputs (parameters require grad)
    assert all(o.grad_fn is None for o in outs) and stub.calls == [('morpher',)]
    with torch.no_grad():
        outs = m(*_inputs(True, True))                   # inputs require grad, grad mode off
    assert all(o.grad_fn is None for o in outs) and stub.calls == [('morpher',)] * 2


@pytest.mark.parametrize('image_rg,pose_rg', [(True, False), (False, True), (True, True)])
def test_input_requiring_grad_takes_the_autograd_path(image_rg, pose_rg):
    m, stub = _module()
    image, pose = _inputs(image_rg, pose_rg)
    outs = m(image, pose)
    assert all(o.grad_fn is not None for o in outs) and stub.calls == [('morpher',)]
    assert len({o.data_ptr() for o in outs}) == len(outs)            # one allocation per output
    outs[0].sum().backward()
    assert stub.calls[1] == ('backward', image_rg, pose_rg)           # exactly the gradients autograd asks for
    assert (image.grad is not None) == image_rg and (pose.grad is not None) == pose_rg
    assert all(p.grad is None for p in m.parameters())


def test_double_backward_raises():
    m, _ = _module()
    image, pose = _inputs(pose_rg=True)
    outs = m(image, pose)
    with pytest.raises(Tha4Error):
        torch.autograd.grad(outs[0].sum(), pose, create_graph=True)
