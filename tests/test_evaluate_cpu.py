"""The evaluation oracle (oracle/evaluator.py) against the unmodified reference Evaluator (tests/golden/evaluate_*.npz,
make_golden_evaluate.py), and its E > 1 semantics on their own."""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from oracle import evaluator as eval_oracle  # noqa: E402

from omnisafe_b200.adapter.saute_adapter import per_step_budget  # noqa: E402

CASES = ('ppolag', 'pposaute', 'ppoearly')


def load_case(name):
    g = np.load(os.path.join(HERE, 'golden', f'evaluate_{name}.npz'))
    cfg = json.loads(str(g['config']))
    pi = {k[3:]: g[k] for k in g.files if k.startswith('pi_')}
    norm = {k[5:]: g[k] for k in g.files if k.startswith('norm0')}
    a = cfg['algo_cfgs']
    saute = None
    if 'Saute' in cfg['algo'] or 'Simmer' in cfg['algo']:
        saute = (per_step_budget(a['safety_budget'], a['saute_gamma'], a['max_ep_len']), a['saute_gamma'])
    cost_limit = a['cost_limit'] if 'EarlyTerminated' in cfg['algo'] else None
    return g, cfg, pi, norm, saute, cost_limit


def run_oracle(name, num_envs=1, num_episodes=None):
    g, cfg, pi, norm, saute, cost_limit = load_case(name)
    n = int(g['num_episodes']) if num_episodes is None else num_episodes
    return eval_oracle.evaluate(pi, norm, cfg['env_cfgs'], n, float(g['cost_criteria']), num_envs=num_envs,
                                saute=saute, cost_limit=cost_limit)


@pytest.mark.parametrize('name', CASES)
def test_oracle_matches_reference_evaluator(name):
    g = load_case(name)[0]
    ret, cost, length, norm = run_oracle(name)
    np.testing.assert_array_equal(length, g['length'])
    np.testing.assert_allclose(ret, g['ret'], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(cost, g['cost'], rtol=1e-6, atol=1e-6)
    assert norm.count == int(g['norm_count'])
    np.testing.assert_allclose(norm.mean, g['norm_mean'], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(norm.std, g['norm_std'], rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize('name', CASES)
def test_parallel_envs_play_every_episode(name):
    """E > 1: every episode is played once, in episode order, and the normaliser sees one row per running env and
    step, plus the final and reset rows."""
    n = 11
    ret, cost, length, norm = run_oracle(name, num_envs=4, num_episodes=n)
    g, cfg = load_case(name)[:2]
    assert (length >= 1).all() and (length <= cfg['env_cfgs']['max_episode_steps']).all()
    assert norm.count > int(g['norm0_count']) + length.sum()
    # env e plays episodes e, e + E, ...: its first episode starts from its own first reset
    assert len(set(np.round(ret[:4], 12))) == 4
