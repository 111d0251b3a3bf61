"""The registered-env evaluation oracle (tests/registered_eval_oracle.py) against the reference Evaluator's fixtures at
E = 1 and the synthetic-env oracle at E > 1, and the refusal of the cost rule at E > 1 on an env without
`reset_envs(mask)`."""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import early_envs as ee  # noqa: E402
import external_envs as xe  # noqa: E402
import registered_eval_oracle as reg_oracle  # noqa: E402
from oracle import evaluator as eval_oracle  # noqa: E402
from oracle.synthetic_env import U32, SyntheticBoxEnv  # noqa: E402
from test_evaluate_cpu import load_case  # noqa: E402

F32 = np.float32


class SyntheticReset(SyntheticBoxEnv):
    """The synthetic dynamics with the reset_envs(mask) hook: the masked envs start their next episode."""

    def reset_envs(self, mask):
        mask = np.asarray(mask, bool)
        with np.errstate(over='ignore'):
            self.episode = np.where(mask, self.episode + U32(1), self.episode).astype(U32)
        self.ep_step = np.where(mask, 0, self.ep_step).astype(self.ep_step.dtype)
        self.s = np.where(mask[:, None], self._reset_values(self.episode), self.s).astype(F32)
        return self.s.copy()


def wide_box(E, O, A, tmax):
    env = ee.WideBoxResetOracle(E, O, A, tmax, seed=0)
    env.act_lo, env.act_hi = xe.wide_box_bounds(A)
    return env


def test_single_env_reproduces_reference_fixtures():
    """E = 1, env.reset() after every episode: the reference Evaluator on the synthetic EarlyTerminated case and on the
    registered WideBox (observations up to ~1e3: its fp32 statistics agree to 1e-5)."""
    for name, make_env in (('ppoearly', lambda kw: SyntheticReset(1, seed=0, **kw)),
                           ('widebox', lambda kw: wide_box(1, kw['obs_dim'], kw['act_dim'], kw['max_episode_steps']))):
        g, cfg, pi, norm, saute, cost_limit = load_case(name)
        ret, cost, length, nz, _ = reg_oracle.evaluate(make_env(cfg['env_cfgs']), pi, norm, int(g['num_episodes']),
                                                       float(g['cost_criteria']), saute=saute, cost_limit=cost_limit)
        np.testing.assert_array_equal(length, g['length'])
        np.testing.assert_allclose(ret, g['ret'], rtol=1e-6, atol=1e-6)
        np.testing.assert_allclose(cost, g['cost'], rtol=1e-6, atol=1e-6)
        assert nz.count == int(g['norm_count'])
        tol = 1e-5 if name == 'widebox' else 1e-6
        np.testing.assert_allclose(nz.mean, g['norm_mean'], rtol=tol, atol=tol)
        np.testing.assert_allclose(nz.std, g['norm_std'], rtol=tol, atol=tol)


@pytest.mark.parametrize('E,n', [(4, 11), (7, 40), (64, 300)])
def test_reset_envs_hook_matches_synthetic_oracle(E, n):
    """E > 1 with the cost rule: resetting the cut envs through reset_envs(mask) and pushing their rows as the third
    batch is the synthetic evaluation's in-kernel reset."""
    g, cfg, pi, norm, _, cost_limit = load_case('ppoearly')
    kw, crit = cfg['env_cfgs'], float(g['cost_criteria'])
    ret, cost, length, nz, n_cut = reg_oracle.evaluate(SyntheticReset(E, seed=0, **kw), pi, norm, n, crit,
                                                       cost_limit=cost_limit)
    r, c, ln, nz0 = eval_oracle.evaluate(pi, norm, kw, n, crit, num_envs=E, cost_limit=cost_limit)
    assert n_cut > 0
    np.testing.assert_array_equal(length, ln)
    np.testing.assert_allclose(ret, r, rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(cost, c, rtol=1e-6, atol=1e-6)
    assert nz.count == nz0.count
    np.testing.assert_allclose(nz.mean, nz0.mean, rtol=1e-6, atol=1e-6)


def wide_case(O, A, seed):
    """The GPU test's policy: action 1, which alone decides WideBox's cost sign, is the constant output bias (zero
    weights), so the episode lengths do not depend on the precision's rounding; the other actions use the network."""
    rng = np.random.default_rng(seed)
    pi = {'log_std': np.full(A, -0.5, F32),
          'mean.0.weight': rng.uniform(-0.4, 0.4, (64, O)).astype(F32),
          'mean.0.bias': rng.uniform(-0.1, 0.1, 64).astype(F32),
          'mean.2.weight': rng.uniform(-0.3, 0.3, (64, 64)).astype(F32),
          'mean.2.bias': rng.uniform(-0.1, 0.1, 64).astype(F32),
          'mean.4.weight': rng.uniform(-0.5, 0.5, (A, 64)).astype(F32),
          'mean.4.bias': rng.uniform(-0.1, 0.1, A).astype(F32)}
    pi['mean.4.weight'][1] = 0.0
    pi['mean.4.bias'][1] = F32(0.25)
    mean = rng.uniform(-0.3, 0.3, O).astype(F32)
    std = rng.uniform(0.4, 1.2, O).astype(F32) * (10.0 ** (np.arange(O) % 4)).astype(F32)
    count = 1000
    norm = {'_mean': mean, '_sumsq': (std * std * (count - 1)).astype(F32), '_std': std, '_var': (std * std).astype(F32),
            '_count': np.int64(count), '_clip': np.full(O, 5.0, F32)}
    return pi, norm


WIDE = {'act_dim': 3, 'max_episode_steps': 12}
WIDE_COST_LIMIT = 3.0


@pytest.mark.parametrize('O', [17, 45, 111])
def test_fixture_cuts_episodes_while_env_runs(O):
    """The GPU fixture exercises the hook: at least 20 % of the episodes end by the cost rule while the env still runs."""
    E, A = 64, WIDE['act_dim']
    n = 2 * E
    pi, norm = wide_case(O, A, seed=O)
    _, _, length, _, n_cut = reg_oracle.evaluate(wide_box(E, O, A, WIDE['max_episode_steps']), pi, norm, n, 0.99,
                                                 cost_limit=WIDE_COST_LIMIT)
    assert n_cut >= 0.2 * n, n_cut
    assert (length >= 1).all()


def test_refused_without_reset_envs_hook(tmp_path):
    """E > 1 EarlyTerminated on an env without reset_envs(mask) is refused before anything runs; the message names the
    hook and where it is specified."""
    from omnisafe_b200 import Evaluator
    from omnisafe_b200.envs import CMDP, ENV_REGISTRY, Box, env_register, env_unregister

    added = None
    if ee.SEEDED_WIDE_ID not in ENV_REGISTRY.support_envs():
        added = env_register(ee.reset_envs_cmdps(CMDP, Box)[0])
    try:
        _refusal(tmp_path, Evaluator)
    finally:
        if added is not None:
            env_unregister(added)


def _refusal(tmp_path, Evaluator):
    pi, norm = wide_case(17, 3, seed=1)
    cfg = {'algo': 'PPOEarlyTerminated', 'env_id': ee.SEEDED_WIDE_ID,
           'env_cfgs': {'obs_dim': 17, **WIDE}, 'algo_cfgs': {'obs_normalize': True, 'cost_limit': WIDE_COST_LIMIT},
           'train_cfgs': {'matmul_precision': 'fp32'}}
    os.makedirs(tmp_path / 'torch_save')
    (tmp_path / 'config.json').write_text(json.dumps(cfg))
    torch.save({'pi': {k: torch.as_tensor(v) for k, v in pi.items()},
                'obs_normalizer': {k: torch.as_tensor(v) for k, v in norm.items()}}, tmp_path / 'torch_save' / 'e.pt')
    ev = Evaluator(device='cpu')
    ev.load_saved(str(tmp_path), 'e.pt')
    with pytest.raises(NotImplementedError, match=r'reset_envs\(mask\).*envs/core\.py'):
        ev.evaluate(num_episodes=4, num_envs=2)
