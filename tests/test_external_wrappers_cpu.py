"""CPU: registered envs behind TimeLimit and AutoReset -- the oracle (oracle/wrapped_external.py) against unmodified
PPOLag rollouts with one env (tests/golden/make_golden_external_wrappers.py), and the configurations the adapters, the
EarlyTerminated algorithms, the evaluator and `check_env` refuse."""
import json
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

import wrapper_envs as we
from oracle.normalizer import Normalizer as ONormalizer
from oracle.wrapped_external import rollout_epoch_wrapped

GOLDENS = ['rollout_external_wrappers.npz', 'rollout_external_autoreset.npz']


@pytest.fixture(scope='module', autouse=True)
def _registered():
    """Registers the test envs for this module and removes them afterwards (other modules expect a clean registry)."""
    from omnisafe_b200.envs import CMDP, Box, ENV_REGISTRY, env_register, env_unregister

    before = set(ENV_REGISTRY.support_envs())
    we.register(CMDP, Box, env_register, ENV_REGISTRY.support_envs())
    yield
    for env_id in set(ENV_REGISTRY.support_envs()) - before:
        env_unregister(ENV_REGISTRY.get_class(env_id))


def _steps_done(g):
    """The wrapper's truncated and done of every step of the fixture, from the env's own flags."""
    T, tmax, tl = int(g['T']), int(g['tmax']), bool(g['time_limit'])
    trunc, done = np.zeros_like(g['env_term']), np.zeros_like(g['env_term'])
    for e in range(trunc.shape[0]):
        k = 0
        for t in range(T):
            k += 1
            trunc[e, t] = k >= tmax if tl else g['env_trunc'][e, t]
            done[e, t] = trunc[e, t] or g['env_term'][e, t]
            k = 0 if done[e, t] else k
    return trunc, done


@pytest.mark.parametrize('fname', GOLDENS)
def test_fixture_covers_the_wrappers(golden_dir, fname):
    g = np.load(os.path.join(golden_dir, fname))
    assert int(g['N']) == 1
    trunc, done = _steps_done(g)
    assert done.sum() >= 10 and not done[:, -1].all()
    if bool(g['time_limit']):
        assert (g['env_trunc'] & ~trunc & ~g['env_term']).any()           # the env's own truncation discarded
        assert (g['env_term'] & trunc).any()                              # termination at the limit
    else:
        assert np.array_equal(trunc, g['env_trunc'])


@pytest.mark.parametrize('fname', GOLDENS)
def test_oracle_matches_reference_golden(golden_dir, fname):
    g = np.load(os.path.join(golden_dir, fname))
    N, T, O, A, E = int(g['N']), int(g['T']), int(g['O']), int(g['A']), int(g['epochs_rolled'])
    env = we.WrappedBoxOracle(N, O, A, seed=int(g['seed']))
    norm, window = ONormalizer((O,)), []
    limit = int(g['tmax']) if bool(g['time_limit']) else 0
    eps = g['eps'].reshape(E, T, N, A)
    trunc, done = _steps_done(g)
    for e in range(E):
        sl = rollout_epoch_wrapped(env, norm, g['theta'], T, eps[e], limit, g['act_lo'], g['act_hi'], window=window)
        assert np.array_equal(sl['done'][:, 0], done[e])
        assert np.array_equal((sl['flags'][:, 0] & 2) != 0, trunc[e])
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


def _cfgs(**env_cfgs):
    return NS(algo_cfgs=NS(obs_normalize=True, reward_normalize=False, cost_normalize=False, cost_limit=2.0),
              logger_cfgs=NS(window_lens=10), env_cfgs=dict(obs_dim=17, act_dim=3, max_episode_steps=5, **env_cfgs))


def test_check_env_needs_the_opt_in():
    from omnisafe_b200.envs import check_env, make

    for env_id in (we.WRAPPED_ID, we.AUTO_RESET_ID, we.WRAPPED_RESET_ID):
        env = make(env_id, num_envs=2, obs_dim=17)
        with pytest.raises(ValueError, match='need_time_limit_wrapper'):
            check_env(env)
        assert check_env(env, wrappers=True)[:2] == (17, 3)


def test_adapter_modes():
    from omnisafe_b200.adapter.external_adapter import ExternalEnvAdapter

    ad = ExternalEnvAdapter(we.WRAPPED_RESET_ID, 4, 0, _cfgs(), device='cpu')
    assert ad._time_limit == 5 and ad._reset_hook
    ad = ExternalEnvAdapter(we.WRAPPED_ID, 1, 0, _cfgs(), device='cpu')
    assert ad._time_limit == 5 and not ad._reset_hook
    assert ExternalEnvAdapter(we.AUTO_RESET_ID, 1, 0, _cfgs(), device='cpu')._time_limit == 0


def test_refuses_time_limit_without_auto_reset():
    from omnisafe_b200.adapter.external_adapter import ExternalEnvAdapter

    with pytest.raises(NotImplementedError, match='need_auto_reset_wrapper'):
        ExternalEnvAdapter(we.TIME_LIMIT_ONLY_ID, 1, 0, _cfgs(), device='cpu')


def test_refuses_missing_max_episode_steps():
    from omnisafe_b200.adapter.external_adapter import ExternalEnvAdapter

    with pytest.raises(AssertionError, match='You must define max_episode_steps as an integer'):
        ExternalEnvAdapter(we.NO_LIMIT_ID, 1, 0, _cfgs(), device='cpu')


@pytest.mark.parametrize('env_id', [we.WRAPPED_ID, we.AUTO_RESET_ID])
def test_refuses_many_envs_without_reset_hook(env_id):
    from omnisafe_b200.adapter.external_adapter import ExternalEnvAdapter

    with pytest.raises(NotImplementedError, match=r'reset_envs\(mask\).*envs/core\.py'):
        ExternalEnvAdapter(env_id, 4, 0, _cfgs(), device='cpu')


def test_refuses_early_terminated():
    from omnisafe_b200.adapter.early_terminated_adapter import ExternalEarlyTerminatedAdapter

    with pytest.raises(NotImplementedError, match='EarlyTerminated'):
        ExternalEarlyTerminatedAdapter(we.WRAPPED_RESET_ID, 4, 0, _cfgs(), device='cpu')


def test_evaluation_refuses_many_envs_without_reset_hook(tmp_path):
    from test_evaluate_registered_cpu import wide_case
    from omnisafe_b200 import Evaluator

    pi, norm = wide_case(17, 3, seed=1)
    cfg = {'algo': 'PPOLag', 'env_id': we.WRAPPED_ID, 'env_cfgs': {'obs_dim': 17, 'act_dim': 3},
           'algo_cfgs': {'obs_normalize': True}, 'train_cfgs': {'matmul_precision': 'fp32'}}
    os.makedirs(tmp_path / 'torch_save')
    (tmp_path / 'config.json').write_text(json.dumps(cfg))
    torch.save({'pi': {k: torch.as_tensor(v) for k, v in pi.items()},
                'obs_normalizer': {k: torch.as_tensor(v) for k, v in norm.items()}}, tmp_path / 'torch_save' / 'e.pt')
    ev = Evaluator(device='cpu')
    ev.load_saved(str(tmp_path), 'e.pt')
    assert ev._wrapped and ev._time_limit == 1000
    with pytest.raises(NotImplementedError, match=r'reset_envs\(mask\).*envs/core\.py'):
        ev.evaluate(num_episodes=4, num_envs=2)
