"""CPU: the hidden activations of model_cfgs.actor / critic.activation (identity, relu, sigmoid, softplus, tanh).

- the fixtures make_golden_activation.py recorded from the unmodified reference are the networks of their activations:
  the first rollout step's values, actions and log-probabilities and the reference actor's mean are the float64 MLPs
  with those activations, and not the tanh ones;
- the same float64 forward through the zero-padded 64-wide layout, with the kernels' rule that a sigmoid or softplus
  unit past its layer's width outputs 0, is the narrow network, and the rule keeps the weight gradient's pads at 0;
- the model records the activation codes and widths it hands to the kernels; a name outside the five fails with an
  AssertionError when the model is built, as upstream's build does;
- the 'pi' of an epoch-k.pt and the activation in config.json round-trip through the Evaluator.
"""
from __future__ import annotations

import json
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from omnisafe_b200.models import ConstraintActorCritic, ParamMap
from omnisafe_b200.models.actor_critic import ACTIVATIONS

HERE = os.path.dirname(os.path.abspath(__file__))
TAGS = ['identity', 'relu', 'sigmoid', 'softplus']
FN = {'identity': lambda x: x, 'relu': torch.relu, 'sigmoid': torch.sigmoid, 'softplus': F.softplus, 'tanh': torch.tanh}


def _model_cfgs(actor_act='tanh', critic_act='tanh', actor=(24, 40), critic=(8, 64)):
    return NS(actor=NS(hidden_sizes=list(actor), activation=actor_act, lr=3e-4),
              critic=NS(hidden_sizes=list(critic), activation=critic_act, lr=3e-4),
              actor_type='gaussian_learning', linear_lr_decay=False, weight_initialization_mode='kaiming_uniform')


def _golden(name, tag):
    g = np.load(os.path.join(HERE, 'golden', f'{name}_act_{tag}.npz'))
    return g, str(g['actor_activation']), str(g['critic_activation'])


def _mlp64(p, x, act, widths=None):
    """Linear-act-Linear-act-Linear in float64; `widths`: the kernels' pad rule on a zero-padded 64-wide network (a
    sigmoid / softplus unit at or past its layer's width outputs 0)."""
    names = list(p)[-6:]
    h = x
    for layer in range(2):
        h = FN[act](F.linear(h, p[names[2 * layer]].double(), p[names[2 * layer + 1]].double()))
        if widths is not None and act in ('sigmoid', 'softplus'):
            h = torch.where(torch.arange(h.shape[-1]) < widths[layer], h, torch.zeros((), dtype=h.dtype))
    return F.linear(h, p[names[4]].double(), p[names[5]].double())


@pytest.mark.parametrize('tag', TAGS)
def test_rollout_fixture_is_the_network_of_its_activations(tag):
    g, aa, ca = _golden('rollout_ppolag', tag)
    O, A = int(g['O']), int(g['A'])
    pmap = ParamMap(O, A, [int(x) for x in g['actor_hidden']], [int(x) for x in g['critic_hidden']])
    theta = pmap.to_kernel(torch.as_tensor(g['theta']))
    obs = torch.as_tensor(g['slab_obs'][0], dtype=torch.float64)
    nets = {n: pmap.views(theta, n) for n in ('actor', 'reward_critic', 'cost_critic')}
    std = torch.exp(nets['actor']['log_std'].double())
    for act_a, act_c, close in ((aa, ca, True), ('tanh', 'tanh', False)):
        mean = _mlp64(nets['actor'], obs, act_a)
        act = mean + torch.as_tensor(g['eps'][0], dtype=torch.float64) * std
        v_r = _mlp64(nets['reward_critic'], obs, act_c)[:, 0]
        v_c = _mlp64(nets['cost_critic'], obs, act_c)[:, 0]
        ok = all(np.allclose(x.numpy(), g[k][0], rtol=1e-5, atol=1e-5)
                 for x, k in ((act, 'slab_act'), (v_r, 'slab_value_r'), (v_c, 'slab_value_c')))
        assert ok == close, (tag, act_a, act_c)
    # the zero-padded 64-wide layout with the kernels' pad rule computes the same function
    pad64 = ParamMap(O, A)
    for net, act_name, widths in (('actor', aa, pmap.actor_hidden), ('reward_critic', ca, pmap.critic_hidden)):
        want = _mlp64(nets[net], obs, act_name)
        got = _mlp64(pad64.views(theta, net), obs, act_name, widths)
        torch.testing.assert_close(got, want, rtol=0, atol=1e-12)
        if act_name in ('sigmoid', 'softplus'):
            # the rule is what keeps the pads of the layer-2 weight gradient at 0: an unmasked pad unit outputs f(0) != 0
            for rule, zero in ((widths, True), (None, False)):
                p64 = {k: v.double().clone().requires_grad_(True) for k, v in pad64.views(theta, net).items()}
                _mlp64(p64, obs, act_name, rule).sum().backward()
                w2 = p64[list(p64)[-4]].grad
                assert bool((w2[:, widths[0]:] == 0).all()) == zero, (net, rule)


@pytest.mark.parametrize('tag', TAGS)
def test_saved_actor_is_the_reference_actor(tag):
    g, aa, ca = _golden('evaluate_actor', tag)
    actor, critic = [int(x) for x in g['actor_hidden']], [int(x) for x in g['critic_hidden']]
    m = ConstraintActorCritic(int(g['O']), int(g['A']), _model_cfgs(aa, ca, actor, critic), epochs=1, device='cpu',
                              generator=torch.Generator().manual_seed(int(g['seed'])))
    pi = m.actor_state_dict()
    for k, v in pi.items():
        assert torch.equal(v, torch.as_tensor(g['pi_' + k])), k
    mean = _mlp64(pi, torch.as_tensor(g['obs'], dtype=torch.float64), aa)
    np.testing.assert_allclose(g['mean'], mean.numpy(), rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize('aa,ca', [('tanh', 'tanh'), ('relu', 'sigmoid'), ('softplus', 'identity'), ('identity', 'relu')])
def test_model_hands_its_activations_and_widths_to_the_kernels(aa, ca):
    m = ConstraintActorCritic(12, 3, _model_cfgs(aa, ca), epochs=1, device='cpu')
    assert m.activation == (aa, ca)
    assert m.net_spec == (ACTIVATIONS.index(aa), ACTIVATIONS.index(ca), (24, 40), (8, 64))
    assert ACTIVATIONS.index('tanh') == 0      # OSB_ACT_TANH, the kernels' default


@pytest.mark.parametrize('which', ['actor', 'critic'])
@pytest.mark.parametrize('name', ['gelu', 'Tanh', 'leaky_relu', None])
def test_unknown_activation_is_refused(which, name):
    acts = {'actor': 'tanh', 'critic': 'tanh', which: name}
    with pytest.raises(AssertionError, match=f'model_cfgs.{which}.activation'):
        ConstraintActorCritic(12, 3, _model_cfgs(acts['actor'], acts['critic']), epochs=1, device='cpu')


@pytest.mark.parametrize('act', ['relu', 'softplus', None])
def test_evaluator_reads_the_activation_from_config(tmp_path, act):
    from omnisafe_b200 import Evaluator

    m = ConstraintActorCritic(12, 3, _model_cfgs(act or 'tanh', 'sigmoid'), epochs=1, device='cpu',
                              generator=torch.Generator().manual_seed(4))
    os.makedirs(tmp_path / 'torch_save')
    actor_cfg = {'hidden_sizes': [24, 40], **({'activation': act} if act else {})}
    cfg = {'algo': 'PPOLag', 'env_id': 'SyntheticBox-v0', 'env_cfgs': {'obs_dim': 12, 'act_dim': 3},
           'algo_cfgs': {'obs_normalize': False}, 'train_cfgs': {'matmul_precision': 'fp32'},
           'model_cfgs': {'actor': actor_cfg}}
    (tmp_path / 'config.json').write_text(json.dumps(cfg))
    torch.save({'pi': m.actor_state_dict()}, tmp_path / 'torch_save' / 'epoch-1.pt')
    ev = Evaluator(device='cpu')
    ev.load_saved(str(tmp_path), 'epoch-1.pt')
    assert ev._actor_act == ACTIVATIONS.index(act or 'tanh') and ev._actor_hidden == (24, 40)
    Pa = m.layout['actor']['size']
    assert torch.equal(ev._theta[:Pa], m.theta[:Pa])
    cfg['model_cfgs']['actor']['activation'] = 'swish'
    (tmp_path / 'config.json').write_text(json.dumps(cfg))
    with pytest.raises(AssertionError, match='model_cfgs.actor.activation'):
        Evaluator(device='cpu').load_saved(str(tmp_path), 'epoch-1.pt')
