"""CPU: which classes train their actor through a PyTorch loss, the library's PyTorch statements of its own losses
against the oracle's formulas (oracle/learner.py), and the sample order the PyTorch path draws."""
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch
from torch.distributions import Normal

from oracle import actor_critic as oac
from oracle import learner as ol

O, A, B = 7, 3, 96


def _classes():
    from omnisafe_b200.algorithms import on_policy, registry

    return on_policy, registry


def test_library_classes_stay_fused():
    from omnisafe_b200.algorithms.torch_loss import overridden_hooks

    on_policy, registry = _classes()
    for name in on_policy.ON_POLICY:
        assert overridden_hooks(registry.get(name)) == [], name


@pytest.mark.parametrize('hook', ['_loss_pi', '_compute_adv_surrogate', '_loss_pi_cost'])
@pytest.mark.parametrize('base', ['PPOLag', 'CPO', 'FOCOPS', 'TRPOEarlyTerminated'])
def test_user_override_switches_the_path(base, hook):
    from omnisafe_b200.algorithms.torch_loss import overridden_hooks

    _, registry = _classes()
    cls = type('User', (registry.get(base),), {hook: lambda self, *a: None})
    found = overridden_hooks(cls)
    assert [h for h, _ in found] == [hook] and found[0][1].endswith('.User')
    # a further library-free subclass inherits the user's override
    assert [h for h, _ in overridden_hooks(type('Deeper', (cls,), {}))] == [hook]
    assert overridden_hooks(type('Plain', (registry.get(base),), {})) == []


class _Actor:
    """The TrainingActor API on the oracle's float64 MLP."""

    def __init__(self, params):
        self.params, self._d = params, None

    def __call__(self, obs):
        self._d = oac.actor_dist(self.params, obs)
        return self._d

    def log_prob(self, act):
        return self._d.log_prob(act).sum(-1)


class _Stats:
    def __init__(self):
        self.vals = {}

    def store(self, d):
        self.vals.update({k: torch.as_tensor(v).mean() for k, v in d.items()})


def _algo(name, **algo_cfgs):
    """A bare instance of library class `name` with what its PyTorch losses read."""
    _, registry = _classes()
    obj = object.__new__(registry.get(name))
    theta = torch.as_tensor(oac.init_theta(O, A, seed=1), dtype=torch.float64)
    params = oac.unflatten(theta, O, A)['actor']
    params['log_std'] += 0.1
    obj._actor_critic = NS(actor=_Actor(params))
    obj._cfgs = NS(algo_cfgs=NS(clip=0.2, entropy_coef=0.01, focops_lam=1.5, focops_eta=0.02, kappa=20.0, **algo_cfgs))
    obj._loss_stats = _Stats()
    return obj, params


def _batch(seed=0):
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(B, O, generator=g, dtype=torch.float64)
    act = torch.randn(B, A, generator=g, dtype=torch.float64)
    logp = torch.randn(B, generator=g, dtype=torch.float64) * 0.3 - 3.0
    return obs, act, logp, torch.randn(B, generator=g, dtype=torch.float64), torch.randn(B, generator=g, dtype=torch.float64)


class _Oracle(ol.Learner):
    def __init__(self, params):      # noqa: super().__init__ casts to float32; the formulas are what is compared
        self.params = {'actor': params}


def test_ratio_and_cost_surrogates_match_the_oracle():
    obj, p = _algo('PolicyGradient')
    obs, act, logp, adv_r, adv_c = _batch()
    L = _Oracle(p)
    torch.testing.assert_close(obj._loss_pi(obs, act, logp, adv_r), L.loss_pi_plain(obs, act, logp, adv_r))
    torch.testing.assert_close(obj._loss_pi_cost(obs, act, logp, adv_c), L.loss_pi_cost(obs, act, logp, adv_c))
    assert set(obj._loss_stats.vals) >= {'Loss/Loss_pi', 'Train/PolicyRatio', 'Train/Entropy', 'Loss/Loss_pi_cost'}
    torch.testing.assert_close(obj._compute_adv_surrogate(adv_r, adv_c), adv_r)


def test_ppo_clip_matches_the_oracle():
    obj, p = _algo('PPO')
    obs, act, logp, adv, _ = _batch(1)
    want, ratio = _Oracle(p).loss_pi_ppo(obs, act, logp, adv, 0.2, 0.01)
    torch.testing.assert_close(obj._loss_pi(obs, act, logp, adv), want)
    torch.testing.assert_close(obj._loss_stats.vals['Train/PolicyRatio'], ratio.mean())


def test_focops_matches_the_oracle_broadcast_form():
    obj, p = _algo('FOCOPS')
    obs, act, logp, adv, _ = _batch(2)
    with torch.no_grad():
        d = oac.actor_dist(p, obs)
        old_mean, old_std = d.loc + 0.05 * torch.randn_like(d.loc), d.scale * 1.02
    obj._p_dist_b = Normal(old_mean, old_std)
    want, _ = _Oracle(p).loss_pi_focops(obs, act, logp, adv, old_mean, old_std, 1.5, 0.02, 0.01)
    torch.testing.assert_close(obj._loss_pi(obs, act, logp, adv), want)


@pytest.mark.parametrize('jc', [-0.5, 0.5])
def test_p3o_matches_the_oracle(jc):
    obj, p = _algo('P3O')
    obj._jc_minus_limit = jc
    obs, act, logp, adv_r, adv_c = _batch(3)
    want, _ = _Oracle(p).loss_pi_p3o(obs, act, logp, adv_r, adv_c, 0.2, 20.0, jc, 0.01)
    torch.testing.assert_close(obj._actor_loss(obs, act, logp, adv_r, adv_c), want)


def test_lagrangian_ipo_and_oncrpo_surrogates():
    from omnisafe_b200.algorithms.engine import LOSS_COST, LOSS_RATIO

    _, _, _, adv_r, adv_c = _batch(4)
    for name in ('PPOLag', 'TRPOLag', 'FOCOPS', 'PDO', 'RCPO', 'CPPOPID', 'TRPOPID'):
        obj, _ = _algo(name)
        obj._lagrange = NS(state=torch.tensor([0.7, 0.0, 0.0, 0.0], dtype=torch.float64))
        torch.testing.assert_close(obj._compute_adv_surrogate(adv_r, adv_c), (adv_r - 0.7 * adv_c) / 1.7)
    obj, _ = _algo('IPO')
    obj._penalty = 2.5
    torch.testing.assert_close(obj._compute_adv_surrogate(adv_r, adv_c), (adv_r - 2.5 * adv_c) / 3.5)
    obj, p = _algo('OnCRPO')
    obs, act, logp, _, _ = _batch(4)
    obj._kind = LOSS_RATIO
    torch.testing.assert_close(obj._compute_adv_surrogate(adv_r, adv_c), adv_r)
    obj._kind = LOSS_COST     # the cost branch minimises mean(ratio * adv_c) through the reward loss
    loss = obj._loss_pi(obs, act, logp, obj._compute_adv_surrogate(adv_r, adv_c))
    torch.testing.assert_close(loss, _Oracle(p).loss_pi_cost(obs, act, logp, adv_c))
    for name in ('CPO', 'PCPO', 'PPO', 'TRPO'):
        obj, _ = _algo(name)
        torch.testing.assert_close(obj._compute_adv_surrogate(adv_r, adv_c), adv_r)


def _feistel_ref(k, n, seed):
    """csrc/loss.cuh feistel_perm, one sample at a time in Python integers."""
    def mix32(x):
        x ^= x >> 16
        x = (x * 0x7FEB352D) & 0xFFFFFFFF
        x ^= x >> 15
        x = (x * 0x846CA68B) & 0xFFFFFFFF
        return x ^ (x >> 16)
    bits = 2
    while (1 << bits) < n:
        bits += 2
    half, mask = bits >> 1, (1 << (bits >> 1)) - 1
    x = k
    while True:
        left, right = (x >> half) & mask, x & mask
        for r in range(4):
            f = mix32(right ^ ((seed + 0x9E3779B9 * (r + 1)) & 0xFFFFFFFF)) & mask
            left, right = right, left ^ f
        x = (left << half) | right
        if x < n:
            return x


@pytest.mark.parametrize('n', [1, 3, 200, 4099])
def test_feistel_order_is_the_kernels(n):
    from omnisafe_b200.algorithms.torch_loss import feistel_order

    seed = (0x1234567 * 1664525 + 1013904223 + 0x9E3779B9 * 3) & 0xFFFFFFFF
    got = feistel_order(n, seed, 'cpu').tolist()
    assert sorted(got) == list(range(n))
    assert got == [_feistel_ref(k, n, seed) for k in range(n)]


def test_device_stats_average_per_key():
    from omnisafe_b200.algorithms.torch_loss import DeviceStats

    s = DeviceStats()
    s.store({'Loss/Loss_pi': torch.tensor(1.0), 'Train/PolicyRatio': torch.tensor([1.0, 3.0])})
    s.store({'Loss/Loss_pi': torch.tensor(3.0), 'Train/PolicyRatio': torch.tensor([0.0, 0.0])})
    assert s.means() == {'Loss/Loss_pi': 2.0, 'Train/PolicyRatio': 1.0}
    s.clear()
    assert s.means() == {}
