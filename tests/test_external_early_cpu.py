"""CPU: the EarlyTerminated rollout on registered envs -- the oracle (oracle/early_external.py) against an unmodified
PPOEarlyTerminated rollout with one env (tests/golden/make_golden_external_early.py), and the configurations the adapter
refuses."""
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest

import early_envs as ee
import external_envs as xe
from oracle.early_external import rollout_epoch_early
from oracle.normalizer import Normalizer as ONormalizer


@pytest.fixture(scope='module', autouse=True)
def _registered():
    """Registers the test envs for this module and removes them afterwards (other modules expect a clean registry)."""
    from omnisafe_b200.envs import CMDP, Box, ENV_REGISTRY, env_register, env_unregister

    before = set(ENV_REGISTRY.support_envs())
    xe.register(CMDP, Box, env_register, ENV_REGISTRY.support_envs())
    ee.register(CMDP, Box, env_register, ENV_REGISTRY.support_envs())
    yield
    for env_id in set(ENV_REGISTRY.support_envs()) - before:
        env_unregister(ENV_REGISTRY.get_class(env_id))


def test_fixture_covers_the_rule(golden_dir):
    g = np.load(os.path.join(golden_dir, 'rollout_external_early.npz'))
    assert int(g['N']) == 1
    acc = g['acc']
    T = int(g['T'])
    after = acc.copy()
    after[-1] = acc[-1] + g['slab_cost'][:, 0]
    trig_last = after[-1] > g['cost_limit']
    assert trig_last.sum() >= 5 and (g['slab_reward'][trig_last, 0] == 0).all()
    # the accumulator before each step is the one after the previous step, cleared where the rule fired
    nxt = np.where(trig_last[:-1], 0, after[-1][:-1])
    assert np.array_equal(acc[-1][1:T], nxt.astype(np.float32))


def test_oracle_matches_reference_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, 'rollout_external_early.npz'))
    N, T, O, A, E = int(g['N']), int(g['T']), int(g['O']), int(g['A']), int(g['epochs_rolled'])
    env = ee.WideBoxResetOracle(N, O, A, int(g['tmax']), seed=int(g['seed']))
    norm, window = ONormalizer((O,)), []
    early = {'cost_limit': float(g['cost_limit']), 'acc': np.zeros(N, np.float32)}
    eps = g['eps'].reshape(E, T, N, A)
    trig = []
    for e in range(E):
        sl = rollout_epoch_early(env, norm, g['theta'], T, eps[e], early, g['act_lo'], g['act_hi'], window=window)
        trig.append(early['trig'][:, 0])
    trig = np.array(trig)
    assert trig.sum() >= 10
    assert (trig & g['env_trunc']).any() and (trig & g['env_term']).any()
    t = dict(rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(sl['obs'], g['slab_obs'], **t)
    np.testing.assert_allclose(sl['act'], g['slab_act'], **t)
    np.testing.assert_allclose(sl['rew'], g['slab_reward'], **t)
    assert np.array_equal(sl['cost'], g['slab_cost'])
    np.testing.assert_allclose(sl['val_r'], g['slab_value_r'], **t)
    np.testing.assert_allclose(sl['val_c'], g['slab_value_c'], **t)
    np.testing.assert_allclose(sl['logp'], g['slab_logp'], rtol=2e-5, atol=5e-5)
    np.testing.assert_allclose(norm.mean, g['norm_mean'], **t)
    np.testing.assert_allclose(norm.std, g['norm_std'], **t)
    assert norm.count == int(g['norm_count'])
    w = np.array(window[-10:], np.float32)
    np.testing.assert_allclose(w[:, 0], g['win_ret'], **t)
    np.testing.assert_allclose(w[:, 1], g['win_cost'])
    np.testing.assert_allclose(w[:, 2], g['win_len'])


def _cfgs(reward_normalize=False, **env_cfgs):
    return NS(algo_cfgs=NS(obs_normalize=True, reward_normalize=reward_normalize, cost_normalize=False, cost_limit=2.0),
              logger_cfgs=NS(window_lens=10), env_cfgs=dict(obs_dim=17, act_dim=3, max_episode_steps=5, **env_cfgs))


def test_refuses_many_envs_without_reset_hook():
    from omnisafe_b200.adapter.early_terminated_adapter import ExternalEarlyTerminatedAdapter

    with pytest.raises(NotImplementedError, match='reset_envs') as err:
        ExternalEarlyTerminatedAdapter(xe.WIDE_BOX_ID, 4, 0, _cfgs(), device='cpu')
    assert 'num_envs == 1' in str(err.value)
    ad = ExternalEarlyTerminatedAdapter(ee.RESET_WIDE_ID, 4, 0, _cfgs(), device='cpu')
    assert ad.num_envs == 4 and ad._hook


@pytest.mark.parametrize('env_id', [xe.WIDE_BOX_ID, ee.RESET_WIDE_ID])
def test_refuses_reward_normalize(env_id):
    from omnisafe_b200.adapter.early_terminated_adapter import ExternalEarlyTerminatedAdapter

    with pytest.raises(NotImplementedError, match='reward_normalize'):
        ExternalEarlyTerminatedAdapter(env_id, 1, 0, _cfgs(reward_normalize=True), device='cpu')
