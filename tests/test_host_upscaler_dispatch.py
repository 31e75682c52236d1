"""Dispatch rule of Upscaler02 (no GPU): without grad mode, or with inputs that do not require grad, forward is today's single
library call; only with grad mode on and one of its four inputs requiring grad does it go through the autograd.Function, and
only then do the outputs carry a grad_fn.  The library context is replaced by a stub that records the calls."""
import pytest
import torch

from tha4_b200._lib import Tha4Error
from tha4_b200.nn.upscaler.upscaler_02 import Upscaler02

SPECS = [(4, 512), (1, 512), (4, 512), (2, 512), (4, 512)]
NAMES = ('rest', 'posed', 'grid', 'pose')


class StubCtx:
    def __init__(self):
        self.calls = []

    def upscaler(self, rest_image, coarse_posed, coarse_grid, pose):
        self.calls.append(('upscaler',))
        return [torch.full((rest_image.shape[0], c, s, s), float(i)) for i, (c, s) in enumerate(SPECS)]

    def upscaler_backward(self, rest_image, coarse_posed, coarse_grid, pose, grad_outputs, d_rest_image=None, d_coarse_posed=None,
                          d_coarse_grid=None, d_pose=None):
        outs = (d_rest_image, d_coarse_posed, d_coarse_grid, d_pose)
        self.calls.append(('backward',) + tuple(o is not None for o in outs))
        for k, o in enumerate(outs):
            if o is not None:
                o.fill_(float(k + 1))


def _module():
    m = Upscaler02()
    stub = StubCtx()
    m.sync_weights = lambda: stub
    return m, stub


def _inputs(size=256, rg=()):
    return (torch.zeros(1, 4, 512, 512, requires_grad='rest' in rg), torch.zeros(1, 4, size, size, requires_grad='posed' in rg),
            torch.zeros(1, 2, size, size, requires_grad='grid' in rg), torch.zeros(1, 6, requires_grad='pose' in rg))


def test_plain_inputs_and_no_grad_take_the_single_call():
    m, stub = _module()
    outs = m(*_inputs())                                 # grad mode on, plain inputs (parameters require grad)
    assert all(o.grad_fn is None for o in outs) and stub.calls == [('upscaler',)]
    with torch.no_grad():
        outs = m(*_inputs(rg=NAMES))                     # inputs require grad, grad mode off
    assert all(o.grad_fn is None for o in outs) and stub.calls == [('upscaler',)] * 2


@pytest.mark.parametrize('size', [256, 512])
@pytest.mark.parametrize('rg', [('rest',), ('posed',), ('grid',), ('pose',), ('posed', 'pose'), NAMES])
def test_input_requiring_grad_takes_the_autograd_path(size, rg):
    m, stub = _module()
    inputs = _inputs(size, rg)
    outs = m(*inputs)
    assert all(o.grad_fn is not None for o in outs) and stub.calls == [('upscaler',)]
    assert len({o.data_ptr() for o in outs}) == len(outs)            # one allocation per output
    outs[0].sum().backward()
    assert stub.calls[1] == ('backward',) + tuple(n in rg for n in NAMES)     # exactly the gradients autograd asks for
    for k, (t, n) in enumerate(zip(inputs, NAMES)):
        assert (t.grad is not None) == (n in rg)
        if t.grad is not None:
            assert t.grad.shape == t.shape and torch.all(t.grad == k + 1)
    assert all(p.grad is None for p in m.parameters())


def test_double_backward_raises():
    m, _ = _module()
    inputs = _inputs(rg=('pose',))
    outs = m(*inputs)
    with pytest.raises(Tha4Error):
        torch.autograd.grad(outs[0].sum(), inputs[3], create_graph=True)
