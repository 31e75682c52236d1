"""Dispatch of the upscaler's opt-in parameter gradients (no GPU), after the body morpher's: a trainable Upscaler02 takes the
autograd path for plain inputs and its backward makes ONE library call that fills a flat state_dict-order d_params, handed
out per parameter (None for frozen ones; coarse_image_conv last); a module that is not trainable keeps the single call and
never passes d_params.  The library context is replaced by a stub that records the calls and writes a ramp into d_params."""
import types

import torch

from tha4_b200.nn.upscaler.upscaler_02 import Upscaler02

SPECS = [(4, 512), (1, 512), (4, 512), (2, 512), (4, 512)]
NAMES = ('rest', 'posed', 'grid', 'pose')


def _ramp(first, n):
    return (torch.arange(first, first + n, dtype=torch.int64) % 4099).float()


class StubCtx:
    def __init__(self, module):
        self.calls = []
        self.n = sum(p.numel() for p in module.parameters())

    def param_count(self, net):
        assert net == 'upscaler'
        return self.n

    def upscaler(self, rest_image, coarse_posed, coarse_grid, pose):
        self.calls.append('upscaler')
        return [torch.full((rest_image.shape[0], c, 8, 8), float(i)) for i, (c, s) in enumerate(SPECS)]

    def upscaler_backward(self, rest_image, coarse_posed, coarse_grid, pose, grad_outputs, d_rest_image=None, d_coarse_posed=None,
                          d_coarse_grid=None, d_pose=None, **kw):
        outs = (d_rest_image, d_coarse_posed, d_coarse_grid, d_pose)
        self.calls.append(('backward', tuple(sorted(kw)), kw.get('d_params') is None) + tuple(o is not None for o in outs))
        d_params = kw.get('d_params')
        if d_params is not None:
            assert d_params.shape == (self.n,)
            d_params.copy_(_ramp(0, self.n))
        for k, o in enumerate(outs):
            if o is not None:
                o.fill_(float(k + 1))


def _module(trainable=False):
    m = Upscaler02().trainable_(trainable)
    stub = StubCtx(m)
    m.sync_weights = lambda: stub
    return m, stub


def _inputs(size=256, rg=()):
    return (torch.zeros(1, 4, 512, 512, requires_grad='rest' in rg), torch.zeros(1, 4, size, size, requires_grad='posed' in rg),
            torch.zeros(1, 2, size, size, requires_grad='grid' in rg), torch.zeros(1, 6, requires_grad='pose' in rg))


def test_parameter_count_and_order():
    m = Upscaler02()
    keys = [k for k, _ in m.named_parameters()]
    assert keys == list(m.state_dict().keys())
    assert len(keys) == 466 and sum(p.numel() for p in m.parameters()) == 35015655
    assert keys[-2:] == ['coarse_image_conv.weight', 'coarse_image_conv.bias']


def test_trainable_plain_inputs_fill_every_grad_from_one_call():
    m, stub = _module(True)
    outs = m(*_inputs())
    assert all(o.grad_fn is not None for o in outs) and stub.calls == ['upscaler']
    sum(o.sum() for o in outs).backward()
    assert stub.calls[1] == ('backward', ('d_params',), False, False, False, False, False)      # d_params only, one call
    off = 0
    for k, p in m.named_parameters():
        assert p.grad is not None and p.grad.shape == p.shape, k
        assert torch.equal(p.grad.flatten(), _ramp(off, p.numel())), k
        off += p.numel()
    assert off == stub.n


def test_coarse_image_conv_is_last_in_the_flat_buffer():
    m, stub = _module(True)
    sum(o.sum() for o in m(*_inputs(512))).backward()
    params = dict(m.named_parameters())
    w, b = params['coarse_image_conv.weight'], params['coarse_image_conv.bias']
    assert w.shape == (32, 10, 3, 3) and b.shape == (32,)
    assert torch.equal(b.grad, _ramp(stub.n - 32, 32))
    assert torch.equal(w.grad.flatten(), _ramp(stub.n - 32 - w.numel(), w.numel()))


def test_frozen_parameters_get_none_and_inputs_come_from_the_same_call():
    m, stub = _module(True)
    params = list(m.parameters())
    for p in params[::2]:
        p.requires_grad_(False)
    inputs = _inputs(rg=('posed', 'pose'))
    sum(o.sum() for o in m(*inputs)).backward()
    assert len(stub.calls) == 2 and stub.calls[1] == ('backward', ('d_params',), False, False, True, False, True)
    off = 0
    for i, p in enumerate(params):
        if i % 2 == 0:
            assert p.grad is None
        else:
            assert torch.equal(p.grad.flatten(), _ramp(off, p.numel()))
        off += p.numel()
    assert torch.all(inputs[1].grad == 2.0) and torch.all(inputs[3].grad == 4.0)
    assert inputs[0].grad is None and inputs[2].grad is None


def test_no_grad_or_all_frozen_take_the_single_call():
    m, stub = _module(True)
    with torch.no_grad():
        outs = m(*_inputs(rg=NAMES))
    assert all(o.grad_fn is None for o in outs) and stub.calls == ['upscaler']
    m.requires_grad_(False)
    outs = m(*_inputs())
    assert all(o.grad_fn is None for o in outs) and stub.calls == ['upscaler'] * 2


def test_not_trainable_never_passes_d_params():
    m, stub = _module(False)
    outs = m(*_inputs())
    assert all(o.grad_fn is None for o in outs) and stub.calls == ['upscaler']
    inputs = _inputs(rg=('rest',))
    sum(o.sum() for o in m(*inputs)).backward()
    assert stub.calls[-1] == ('backward', (), True, True, False, False, False)
    assert all(p.grad is None for p in m.parameters())


def test_mode_07_takes_the_composed_path_for_a_trainable_upscaler():
    from tha4_b200.poser.modes import mode_07
    proto = mode_07.FiveStepPoserComputationProtocol
    up = Upscaler02()
    state = types.SimpleNamespace(modules={'body_morpher': object(), 'upscaler': up})
    assert not proto._trains_teacher(state)
    up.trainable_()
    assert proto._trains_teacher(state)
    with torch.no_grad():
        assert not proto._trains_teacher(state)
    up.requires_grad_(False)
    assert not proto._trains_teacher(state)
