"""Dispatch of the body morpher's opt-in parameter gradients (no GPU), after the encoder-decoder teachers': a trainable
Morpher00 takes the autograd path for plain inputs and its backward makes ONE library call that fills a flat state_dict-order
d_params, handed out per parameter (None for frozen ones); a module that is not trainable never passes d_params.  The library
context is replaced by a stub that records the calls and writes a ramp into d_params."""
import types

import torch

from tha4_b200.nn.morpher.morpher_00 import Morpher00

SPECS = [(4, 256), (1, 256), (4, 256), (2, 256), (4, 256)]


def _ramp(first, n):
    return (torch.arange(first, first + n, dtype=torch.int64) % 4099).float()


class StubCtx:
    def __init__(self, module):
        self.calls = []
        self.n = sum(p.numel() for p in module.parameters())

    def param_count(self, net):
        assert net == 'body_morpher'
        return self.n

    def morpher(self, image, pose):
        self.calls.append('morpher')
        return [torch.full((image.shape[0], c, 8, 8), float(i)) for i, (c, s) in enumerate(SPECS)]

    def morpher_backward(self, image, pose, grads, d_image=None, d_pose=None, **kw):
        self.calls.append(('backward', tuple(sorted(kw)), kw.get('d_params') is None, d_image is not None, d_pose is not None))
        d_params = kw.get('d_params')
        if d_params is not None:
            assert d_params.shape == (self.n,)
            d_params.copy_(_ramp(0, self.n))
        for v in (d_image, d_pose):
            if v is not None:
                v.fill_(7.0)


def _module(trainable=False):
    m = Morpher00().trainable_(trainable)
    stub = StubCtx(m)
    m.sync_weights = lambda: stub
    return m, stub


def _inputs(image_rg=False, pose_rg=False):
    return torch.zeros(2, 4, 256, 256, requires_grad=image_rg), torch.zeros(2, 6, requires_grad=pose_rg)


def test_parameter_count_and_order():
    m = Morpher00()
    assert [k for k, _ in m.named_parameters()] == list(m.state_dict().keys())
    assert len(m.state_dict()) == 398 and sum(p.numel() for p in m.parameters()) == 34682119


def test_trainable_plain_inputs_fill_every_grad_from_one_call():
    m, stub = _module(True)
    outs = m(*_inputs())
    assert all(o.grad_fn is not None for o in outs) and stub.calls == ['morpher']
    sum(o.sum() for o in outs).backward()
    assert stub.calls[1] == ('backward', ('d_params',), False, False, False)        # d_params only, one call
    off = 0
    for k, p in m.named_parameters():
        assert p.grad is not None and p.grad.shape == p.shape, k
        assert torch.equal(p.grad.flatten(), _ramp(off, p.numel())), k
        off += p.numel()
    assert off == stub.n


def test_frozen_parameters_get_none_and_inputs_come_from_the_same_call():
    m, stub = _module(True)
    params = list(m.parameters())
    for p in params[::2]:
        p.requires_grad_(False)
    image, pose = _inputs(pose_rg=True)
    sum(o.sum() for o in m(image, pose)).backward()
    assert len(stub.calls) == 2 and stub.calls[1] == ('backward', ('d_params',), False, False, True)
    off = 0
    for i, p in enumerate(params):
        if i % 2 == 0:
            assert p.grad is None
        else:
            assert torch.equal(p.grad.flatten(), _ramp(off, p.numel()))
        off += p.numel()
    assert torch.all(pose.grad == 7.0) and image.grad is None


def test_no_grad_or_all_frozen_take_the_single_call():
    m, stub = _module(True)
    with torch.no_grad():
        outs = m(*_inputs(True, True))
    assert all(o.grad_fn is None for o in outs) and stub.calls == ['morpher']
    m.requires_grad_(False)
    outs = m(*_inputs())
    assert all(o.grad_fn is None for o in outs) and stub.calls == ['morpher'] * 2


def test_not_trainable_never_passes_d_params():
    m, stub = _module(False)
    outs = m(*_inputs())
    assert all(o.grad_fn is None for o in outs) and stub.calls == ['morpher']
    image, pose = _inputs(image_rg=True)
    sum(o.sum() for o in m(image, pose)).backward()
    assert stub.calls[-1] == ('backward', (), True, True, False)
    assert all(p.grad is None for p in m.parameters())


def test_mode_07_takes_the_composed_path_for_a_trainable_body_morpher():
    from tha4_b200.poser.modes import mode_07
    proto = mode_07.FiveStepPoserComputationProtocol
    body = Morpher00()
    state = types.SimpleNamespace(modules={'body_morpher': body, 'upscaler': object()})
    assert not proto._trains_teacher(state)
    body.trainable_()
    assert proto._trains_teacher(state)
    with torch.no_grad():
        assert not proto._trains_teacher(state)
    body.requires_grad_(False)
    assert not proto._trains_teacher(state)
