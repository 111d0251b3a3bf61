"""CPU: the upstream configuration values `lagrange_cfgs.lambda_optimizer` and `model_cfgs.weight_initialization_mode`.

- the optimisers that fail on upstream's multiplier too (LBFGS, SparseAdam, Muon) are refused when the Lagrange is
  built, with a message naming them; an unknown name raises upstream's assertion;
- every upstream init mode, at [64, 64] and at actor [24, 40] / critic [8, 64]: pads stay +0, kaiming_uniform keeps
  its bits, orthogonal blocks are sqrt(2)-scaled orthogonal, xavier bounds and std follow the real fans, a seeded
  init is deterministic.
"""
from __future__ import annotations

import math
from types import SimpleNamespace as NS

import pytest
import torch

from omnisafe_b200.common.lagrange import REFUSED, Lagrange
from omnisafe_b200.models import ConstraintActorCritic, ParamMap

O, A = 12, 3
WIDTHS = [([64, 64], [64, 64]), ([24, 40], [8, 64])]
MODES = ['kaiming_uniform', 'xavier_normal', 'glorot', 'xavier_uniform', 'orthogonal']
NETS = ('actor', 'reward_critic', 'cost_critic')


@pytest.mark.parametrize('name', sorted(REFUSED))
def test_refused_lambda_optimizers_name_themselves(name):
    with pytest.raises(ValueError, match=f"lambda_optimizer='{name}' cannot step the Lagrange multiplier"):
        Lagrange(25.0, 0.001, 0.035, name, device='cpu')


def test_unknown_lambda_optimizer_raises_upstreams_assertion():
    with pytest.raises(AssertionError, match='Optimizer=Adamm not found in torch.'):
        Lagrange(25.0, 0.001, 0.035, 'Adamm', device='cpu')


def test_torch_optim_non_optimizer_is_refused():
    with pytest.raises(ValueError, match='not a torch.optim optimiser'):
        Lagrange(25.0, 0.001, 0.035, 'lr_scheduler', device='cpu')


def _model(mode, actor, critic, seed=0):
    net = lambda hs: NS(hidden_sizes=list(hs), activation='tanh', lr=3e-4)   # noqa: E731
    cfgs = NS(actor=net(actor), critic=net(critic), actor_type='gaussian_learning', linear_lr_decay=False,
              weight_initialization_mode=mode)
    return ConstraintActorCritic(O, A, cfgs, epochs=1, device='cpu', generator=torch.Generator().manual_seed(seed))


def _linears(model, net):
    views = model.named_views(net)
    names = list(views)
    return [(views[w], views[b]) for w, b in zip(names[-6::2], names[-5::2])]


def test_unknown_init_mode_raises_upstreams_error():
    with pytest.raises(TypeError, match='Invalid initialization function: he_normal'):
        _model('he_normal', [64, 64], [64, 64])


@pytest.mark.parametrize('actor,critic', WIDTHS)
@pytest.mark.parametrize('mode', MODES)
def test_init_mode_pads_determinism_and_bias(mode, actor, critic):
    m = _model(mode, actor, critic)
    pmap = ParamMap(O, A, actor, critic)
    real = torch.zeros(pmap.kernel['total'], dtype=torch.bool)
    for net in NETS:
        for v in pmap.views(real, net).values():
            v.fill_(True)
    pads = m.theta[~real]
    assert torch.equal(pads, torch.zeros_like(pads)) and not torch.signbit(pads).any()   # +0, not -0
    assert torch.equal(m.theta, _model(mode, actor, critic).theta)
    assert not torch.equal(m.theta, _model(mode, actor, critic, seed=1).theta)
    for net in NETS:
        for w, b in _linears(m, net):
            assert b.abs().max() <= 1.0 / math.sqrt(w.shape[1])   # nn.Linear's default bias, real fan-in


@pytest.mark.parametrize('actor,critic', WIDTHS)
def test_kaiming_uniform_keeps_its_bits(actor, critic):
    """The draw every earlier version made: U(+-sqrt(6 / (6 fan_in))) weight then U(+-1/sqrt(fan_in)) bias, per layer."""
    gen = torch.Generator().manual_seed(0)
    pmap = ParamMap(O, A, actor, critic)
    theta = torch.zeros(pmap.kernel['total'])
    for net in NETS:
        views = pmap.views(theta, net)
        names = list(views)
        for wname, bname in zip(names[-6::2], names[-5::2]):
            w, b = views[wname], views[bname]
            bw = math.sqrt(6.0 / ((1.0 + 5.0) * w.shape[1]))
            w.copy_(torch.empty(w.shape).uniform_(-bw, bw, generator=gen))
            bb = 1.0 / math.sqrt(w.shape[1])
            b.copy_(torch.empty(b.shape).uniform_(-bb, bb, generator=gen))
    assert torch.equal(_model('kaiming_uniform', actor, critic).theta, theta)


@pytest.mark.parametrize('actor,critic', WIDTHS)
def test_orthogonal_blocks_are_scaled_orthogonal(actor, critic):
    m = _model('orthogonal', actor, critic)
    for net in NETS:
        for w, _ in _linears(m, net):
            w = w.double()
            gram = w.T @ w if w.shape[0] >= w.shape[1] else w @ w.T   # tall: W^T W, wide: W W^T
            torch.testing.assert_close(gram, 2.0 * torch.eye(gram.shape[0], dtype=torch.float64),
                                       atol=1e-5, rtol=0)


@pytest.mark.parametrize('actor,critic', WIDTHS)
@pytest.mark.parametrize('mode', ['glorot', 'xavier_uniform', 'xavier_normal'])
def test_xavier_scale_follows_the_real_fans(mode, actor, critic):
    m = _model(mode, actor, critic, seed=3)
    for net in NETS:
        for w, _ in _linears(m, net):
            fan_out, fan_in = w.shape
            std = math.sqrt(2.0 / (fan_in + fan_out))
            if mode == 'xavier_normal':
                if w.numel() >= 500:   # the sample std of the big blocks within 15 %
                    assert abs(float(w.std()) / std - 1.0) < 0.15
            else:
                bound = math.sqrt(3.0) * std
                assert float(w.abs().max()) <= bound
                if w.numel() >= 500:   # and the draw reaches close to the bound
                    assert float(w.abs().max()) > 0.9 * bound
