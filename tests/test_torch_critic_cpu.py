"""CPU: which classes train a critic through its PyTorch hook, and the library's PyTorch `_update_reward_critic` /
`_update_cost_critic` against the oracle's formulas (oracle/learner.py critic_step, oracle/optim64.py _net_step): loss,
critic-norm gradient, clipping and the Adam step."""
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from oracle import actor_critic as oac
from oracle import optim64

O, A, B = 7, 3, 96
CRITIC_HOOKS = ('_update_reward_critic', '_update_cost_critic')


def _registry():
    from omnisafe_b200.algorithms import registry

    return registry


@pytest.mark.parametrize('hook', CRITIC_HOOKS)
@pytest.mark.parametrize('base', ['PPOLag', 'CPO', 'FOCOPS', 'PPOSaute', 'TRPOEarlyTerminated'])
def test_critic_override_is_detected(base, hook):
    from omnisafe_b200.algorithms.torch_loss import overridden_hooks

    cls = type('User', (_registry().get(base),), {hook: lambda self, obs, target: None})
    found = overridden_hooks(cls)
    assert [h for h, _ in found] == [hook] and found[0][1].endswith('.User')
    # a further library-free subclass inherits the user's override
    assert [h for h, _ in overridden_hooks(type('Deeper', (cls,), {}))] == [hook]
    assert overridden_hooks(type('Plain', (_registry().get(base),), {})) == []


def test_critic_and_actor_overrides_together():
    from omnisafe_b200.algorithms.torch_loss import overridden_hooks

    body = {h: (lambda self, *a: None) for h in ('_loss_pi', *CRITIC_HOOKS)}
    found = overridden_hooks(type('User', (_registry().get('PPOLag'),), body))
    assert sorted(h for h, _ in found) == sorted(body)


def test_library_defines_the_critic_hooks():
    """super() reaches the library's own statement of the critic step on every on-policy class."""
    from omnisafe_b200.algorithms import on_policy

    for name in on_policy.ON_POLICY:
        cls = _registry().get(name)
        for hook in CRITIC_HOOKS:
            assert getattr(cls, hook).__module__ == on_policy.__name__, (name, hook)


class _Critic:
    """The TrainingCritic API on the oracle's float64 MLP."""

    def __init__(self, params):
        self.params = params

    def __call__(self, obs):
        return [oac.critic_value(self.params, obs)]

    def parameters(self):
        return iter(self.params.values())


class _Stats:
    def __init__(self):
        self.vals = {}

    def store(self, d):
        self.vals.update({k: torch.as_tensor(v) for k, v in d.items()})


@pytest.mark.parametrize('net', ['reward_critic', 'cost_critic'])
@pytest.mark.parametrize('use_critic_norm,use_max_grad_norm,max_grad_norm', [
    (True, True, 40.0),      # the defaults: clipping inactive
    (True, True, 0.05),      # clipping active
    (False, False, 0.05),
])
def test_library_critic_step_matches_the_oracle(net, use_critic_norm, use_max_grad_norm, max_grad_norm):
    coef, lr = 0.001, 3e-4
    theta = oac.init_theta(O, A, seed=2).astype(np.float64)
    lay = oac.layout(O, A)
    g = torch.Generator().manual_seed(5)
    obs = torch.randn(B, O, generator=g, dtype=torch.float64)
    target = torch.randn(B, generator=g, dtype=torch.float64)

    # the oracle: one step of oracle/optim64.py (the critic L2 term as Learner.critic_step adds it)
    state = optim64.init_state(theta)
    _, clip_coef, want_grad, want_loss = optim64._net_step(
        state, lay, net, lambda p: torch.nn.functional.mse_loss(oac.critic_value(p, obs), target),
        max_grad_norm=max_grad_norm if use_max_grad_norm else 0.0, lr=lr,
        critic_norm_coef=coef if use_critic_norm else 0.0)
    assert (clip_coef < 1.0) == (use_max_grad_norm and max_grad_norm < 1.0)

    # the library's PyTorch statement on float64 leaves, a torch Adam as the optimiser
    obj = object.__new__(_registry().get('PPOLag'))
    s, n = lay[net]['start'], lay[net]['size']
    leaves = optim64._leaves(theta, lay, net, grad=True)
    opt = torch.optim.Adam(list(leaves.values()), lr=lr)
    grads = {}
    orig_step = opt.step

    def step():
        grads['g'] = torch.cat([p.grad.reshape(-1) for p in leaves.values()]).detach().numpy().copy()
        orig_step()
    opt.step = step
    obj._actor_critic = NS(**{net: _Critic(leaves), f'{net}_optimizer': opt})
    obj._cfgs = NS(algo_cfgs=NS(use_critic_norm=use_critic_norm, critic_norm_coef=coef,
                                use_max_grad_norm=use_max_grad_norm, max_grad_norm=max_grad_norm))
    obj._logger = _Stats()
    getattr(obj, '_update_reward_critic' if net == 'reward_critic' else '_update_cost_critic')(obs, target)

    key = 'Loss/Loss_reward_critic' if net == 'reward_critic' else 'Loss/Loss_cost_critic'
    np.testing.assert_allclose(float(obj._logger.vals[key]), want_loss, rtol=1e-12)
    np.testing.assert_allclose(grads['g'], want_grad, rtol=1e-10, atol=1e-14)
    got_theta = torch.cat([p.detach().reshape(-1) for p in leaves.values()]).numpy()
    np.testing.assert_allclose(got_theta, state['theta'][s:s + n], rtol=1e-12, atol=1e-15)


def test_device_stats_keep_python_numbers_on_their_device():
    from omnisafe_b200.algorithms.torch_loss import DeviceStats

    s = DeviceStats('cpu')
    s.store({'Loss/Loss_reward_critic': 1.5, 'Loss/Loss_pi': torch.tensor(2.0)})
    s.store({'Loss/Loss_reward_critic': 2.5, 'Loss/Loss_pi': torch.tensor(4.0)})
    assert s.means() == {'Loss/Loss_reward_critic': 2.0, 'Loss/Loss_pi': 3.0}


def test_hook_logger_routes_store_and_forwards_the_rest():
    from omnisafe_b200.algorithms.torch_loss import DeviceStats, HookLogger

    logged = []
    real = NS(store=lambda d: logged.append(d), log=lambda msg: logged.append(msg))
    stats = DeviceStats()
    hl = HookLogger(real, stats)
    hl.store({'Loss/Loss_cost_critic': 0.25})
    hl.log('hello')
    assert logged == ['hello'] and stats.means() == {'Loss/Loss_cost_critic': 0.25}
