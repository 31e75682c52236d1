"""Dispatch rule of the encoder-decoder teacher modules (no GPU): without grad mode, or with inputs that do not require
grad, forward is today's single library call; only with grad mode on and an input requiring grad does it go through the
autograd.Function.  The library context is replaced by a stub that records the calls."""
import torch

from tha4_b200.nn.eyebrow_decomposer.eyebrow_decomposer_00 import EyebrowDecomposer00
from tha4_b200.nn.eyebrow_morphing_combiner.eyebrow_morphing_combiner_00 import EyebrowMorphingCombiner00
from tha4_b200.nn.face_morpher.face_morpher_08 import FaceMorpher08


class StubCtx:
    def __init__(self):
        self.calls = []

    def _outs(self, name, B, specs):
        self.calls.append(name)
        return [torch.full((B, c, s, s), float(i)) for i, (c, s) in enumerate(specs)]

    def eyebrow_decomposer(self, image):
        return self._outs('decomposer', image.shape[0], [(4, 8)] * 6)

    def eyebrow_morphing_combiner(self, background_layer, eyebrow_layer, pose):
        return self._outs('combiner', background_layer.shape[0], [(4, 8)] * 8)

    def face_morpher(self, image, pose):
        return self._outs('face', image.shape[0], [(4, 8)] * 8)


def _with_stub(module):
    stub = StubCtx()
    module.sync_weights = lambda: stub
    return module, stub


def _cases(cls):
    if cls is EyebrowDecomposer00:
        return lambda rg: (torch.zeros(2, 4, 8, 8, requires_grad=rg),)
    if cls is EyebrowMorphingCombiner00:
        return lambda rg: (torch.zeros(2, 4, 8, 8), torch.zeros(2, 4, 8, 8), torch.zeros(2, 12, requires_grad=rg))
    return lambda rg: (torch.zeros(2, 4, 8, 8), torch.zeros(2, 27, requires_grad=rg))


def test_plain_inputs_and_no_grad_take_the_single_call():
    for cls in (EyebrowDecomposer00, EyebrowMorphingCombiner00, FaceMorpher08):
        m, stub = _with_stub(cls())
        make = _cases(cls)
        outs = m(*make(False))                        # grad mode on, plain inputs (parameters require grad)
        assert all(o.grad_fn is None for o in outs) and len(stub.calls) == 1
        with torch.no_grad():
            outs = m(*make(True))                     # input requires grad, grad mode off
        assert all(o.grad_fn is None for o in outs) and len(stub.calls) == 2


def test_input_requiring_grad_takes_the_autograd_path():
    for cls in (EyebrowDecomposer00, EyebrowMorphingCombiner00, FaceMorpher08):
        m, stub = _with_stub(cls())
        outs = m(*_cases(cls)(True))
        assert all(o.grad_fn is not None for o in outs) and len(stub.calls) == 1
        assert len({o.data_ptr() for o in outs}) == len(outs)        # one allocation per output
