"""GPU: `Evaluator` on registered envs at E > 1 -- the cost rule through the env's `reset_envs(mask)` hook
(osb_eval_ext_observe_rst + osb_ext_reset_rows) against the oracle (tests/registered_eval_oracle.py), and graph-safe
envs replaying blocks of steps from a CUDA graph, bit for bit against the eager loop."""
from __future__ import annotations

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
from test_evaluate_gpu import write_run  # noqa: E402
from test_evaluate_registered_cpu import WIDE, WIDE_COST_LIMIT, wide_box, wide_case  # noqa: E402

pytestmark = pytest.mark.gpu
TOL = {'fp32': 1e-4, 'tf32': 5e-3, 'bf16x3': 1e-4}
COUNTED_RESET_ID = 'CountedGraphWideBoxReset-v0'
COUNTED_PLAIN_ID = 'CountedGraphWideBox-v0'


def _counted(cls, env_id):
    """cls under its own id, counting its Python step calls (a replayed step does not call it)."""
    class Counted(cls):
        _support_envs = [env_id]  # noqa: RUF012
        steps = 0

        def step(self, action):
            type(self).steps += 1
            return super().step(action)

    Counted.__name__ = Counted.__qualname__ = 'Counted' + cls.__name__
    return Counted


@pytest.fixture(scope='module', autouse=True)
def _registered():
    from omnisafe_b200.envs import CMDP, ENV_REGISTRY, Box, env_register

    ee.register(CMDP, Box, env_register, ENV_REGISTRY.support_envs())
    if COUNTED_RESET_ID not in ENV_REGISTRY.support_envs():
        WideBox, _, GraphReset = ee.reset_envs_cmdps(CMDP, Box)

        class GraphWideBox(WideBox):
            """Graph-safe WideBox without reset_envs: in-place state, step info always complete."""
            graph_safe = True

            def set_seed(self, seed):
                self._core = ee.GraphWideBoxResetCore(*self._kw, seed=seed, device=self._device)

            def step(self, action):
                nobs, rew, cost, term, trunc, final, fin = self._core.step(torch.as_tensor(action))
                return nobs, rew, cost, term, trunc, {'final_observation': final, '_final_observation': fin}

        env_register(_counted(GraphReset, COUNTED_RESET_ID))
        env_register(_counted(GraphWideBox, COUNTED_PLAIN_ID))


def _evaluator(tmp, env_id, algo, O, precision, pi, norm, obs_normalize=True, **env_cfgs):
    from omnisafe_b200 import Evaluator

    a = {'obs_normalize': obs_normalize}
    if 'EarlyTerminated' in algo:
        a['cost_limit'] = WIDE_COST_LIMIT
    if 'Saute' in algo:
        a.update(safety_budget=3.0, saute_gamma=0.999, max_ep_len=WIDE['max_episode_steps'])
    cfg = {'algo': algo, 'env_id': env_id, 'env_cfgs': {**WIDE, 'obs_dim': O, **env_cfgs}, 'algo_cfgs': a}
    ev = Evaluator()
    ev.load_saved(write_run(tmp, cfg, pi, norm, precision), 'epoch-0.pt')
    return ev


@pytest.mark.parametrize('precision', ['fp32', 'tf32', 'bf16x3'])
@pytest.mark.parametrize('O', [17, 45, 111])
@pytest.mark.parametrize('E', [7, 256, 4096])
def test_cost_rule_through_reset_envs_matches_oracle(cuda, tmp_path, monkeypatch, E, O, precision, capsys):
    """PPOEarlyTerminated on WideBoxReset at E > 1: lengths exact, returns and costs to the precision's tolerance, the
    drifted statistics (with the reset rows as every step's third batch) to the same, relative to each observation
    column's scale (WideBox's column j spans about 10^(j mod 4), and the actions move it by that factor)."""
    monkeypatch.setenv('OSB_NO_GRAPH', '1')
    A, n = WIDE['act_dim'], 2 * E + 3
    pi, norm = wide_case(O, A, seed=O + E)
    ev = _evaluator(tmp_path, ee.RESET_WIDE_ID, 'PPOEarlyTerminated', O, precision, pi, norm)
    rets, costs = ev.evaluate(num_episodes=n, cost_criteria=0.99, num_envs=E)
    capsys.readouterr()
    r, c, ln, nz, n_cut = reg_oracle.evaluate(wide_box(E, O, A, WIDE['max_episode_steps']), pi, norm, n, 0.99,
                                              cost_limit=WIDE_COST_LIMIT)
    assert n_cut >= 0.2 * n
    np.testing.assert_array_equal(ev.episode_lengths, ln)
    tol = TOL[precision]
    np.testing.assert_allclose(rets, r, rtol=tol, atol=tol)
    np.testing.assert_allclose(costs, c, rtol=tol, atol=tol)
    assert int(ev.normalizer.count[0]) == nz.count
    scale = 10.0 ** (np.arange(O) % 4)
    np.testing.assert_array_less(np.abs(ev.normalizer.mean.cpu().numpy() - nz.mean), tol * scale)


@pytest.mark.parametrize('precision', ['fp32', 'tf32', 'bf16x3'])
def test_action_is_predict_bits(cuda, tmp_path, monkeypatch, precision, capsys):
    """One-step episodes without observation normalisation on the hook path: the actions equal
    actor.predict(obs, True) bit for bit, and the returns are the env's rewards for them."""
    from omnisafe_b200.models.actor_critic import ConstraintActorCritic
    from omnisafe_b200.utils.config import Config

    monkeypatch.setenv('OSB_NO_GRAPH', '1')
    O, A, E = 45, WIDE['act_dim'], 300
    pi, norm = wide_case(O, A, seed=5)
    ev = _evaluator(tmp_path, ee.RESET_WIDE_ID, 'PPOEarlyTerminated', O, precision, pi, norm, obs_normalize=False,
                    max_episode_steps=1)
    rets, _ = ev.evaluate(num_episodes=E, num_envs=E)
    capsys.readouterr()
    mc = Config.dict2config({'actor': {'hidden_sizes': [64, 64], 'activation': 'tanh', 'lr': 0.0},
                             'critic': {'hidden_sizes': [64, 64], 'activation': 'tanh', 'lr': 0.0},
                             'actor_type': 'gaussian_learning', 'weight_initialization_mode': 'kaiming_uniform',
                             'linear_lr_decay': False})
    ac = ConstraintActorCritic(O, A, mc, epochs=1)
    ac.precision = {'fp32': 0, 'tf32': 1, 'bf16x3': 2}[precision]
    for k, (off, shape) in ac.layout['actor']['entries'].items():
        ac.theta[off:off + int(np.prod(shape))] = torch.as_tensor(pi[k]).reshape(-1).to(ac.theta)
    core = xe.WideBoxCore(E, O, A, 1, seed=0, device=cuda)
    obs = core.reset()
    act = ac.actor.predict(obs, deterministic=True)
    assert torch.equal(ev.last_actions, act)
    lo, hi = (torch.as_tensor(b).to(cuda) for b in xe.wide_box_bounds(A))
    rew = core.step(lo + (hi - lo) * (act + 1) / 2)[1]
    np.testing.assert_array_equal(np.array(rets), rew.cpu().numpy().astype(np.float64))


def _run(tmp, monkeypatch, graph, env_id, algo, precision, E, n, O=45):
    if graph:
        monkeypatch.delenv('OSB_NO_GRAPH', raising=False)
    else:
        monkeypatch.setenv('OSB_NO_GRAPH', '1')
    from omnisafe_b200.envs.core import ENV_REGISTRY

    cls = ENV_REGISTRY.get_class(env_id)
    On = O + int('Saute' in algo)
    pi, norm = wide_case(On, WIDE['act_dim'], seed=11)
    norm = {k: (v[:O] if np.ndim(v) else v) for k, v in norm.items()}
    ev = _evaluator(tmp, env_id, algo, O, precision, pi, norm)
    cls.steps = 0
    rets, costs = ev.evaluate(num_episodes=n, cost_criteria=0.99, num_envs=E)
    nz = ev.normalizer
    return {'ret': rets, 'cost': costs, 'len': ev.episode_lengths, 'steps': cls.steps,
            'act': ev.last_actions.cpu().numpy(), **{k: getattr(nz, k).cpu().numpy() for k in ('mean', 'sumsq', 'std', 'count')}}


@pytest.mark.parametrize('precision', ['fp32', 'bf16x3'])
@pytest.mark.parametrize('env_id,algo', [(COUNTED_RESET_ID, 'PPOEarlyTerminated'), (COUNTED_RESET_ID, 'PPOLag'),
                                         (COUNTED_RESET_ID, 'PPOSaute'), (COUNTED_PLAIN_ID, 'PPOLag'),
                                         (COUNTED_PLAIN_ID, 'PPOSaute')])
def test_graph_equals_eager_bitwise(cuda, tmp_path, monkeypatch, env_id, algo, precision, capsys):
    """Graph-safe envs at E > 1: the eager warm-up block, the capture and the replays give the eager loop's bits
    (results, statistics, last actions); the env's Python step ran only in the warm-up block and the capture."""
    from omnisafe_b200.evaluator import GRAPH_BLOCK

    E, n = 300, 3000
    eager = _run(tmp_path / 'eager', monkeypatch, False, env_id, algo, precision, E, n)
    graph = _run(tmp_path / 'graph', monkeypatch, True, env_id, algo, precision, E, n)
    capsys.readouterr()
    assert eager['steps'] > 3 * GRAPH_BLOCK            # the evaluation outlasts the warm-up block and one replay
    assert graph['steps'] == 2 * GRAPH_BLOCK
    if 'EarlyTerminated' in algo:
        assert sum(ln < WIDE['max_episode_steps'] for ln in graph['len']) > 0
    for k, v in eager.items():
        if k != 'steps':
            assert np.array_equal(np.asarray(graph[k]), np.asarray(v)), f'{k} differs between graph and eager'


@pytest.mark.parametrize('graph', [False, True])
def test_agent_evaluate_many_envs_after_learn(cuda, tmp_path, monkeypatch, graph, capsys):
    """PPOEarlyTerminated trained on the hook env scores every checkpoint with 64 envs, eager and graph-safe."""
    import omnisafe_b200

    env_id = ee.GRAPH_RESET_WIDE_ID if graph else ee.RESET_WIDE_ID
    if graph:
        monkeypatch.delenv('OSB_NO_GRAPH', raising=False)
    N, T = 64, 32
    cfg = {'seed': 3, 'train_cfgs': {'device': 'cuda', 'vector_env_nums': N, 'total_steps': N * T * 2, 'parallel': 1},
           'algo_cfgs': {'steps_per_epoch': N * T, 'batch_size': 256, 'update_iters': 2, 'cost_limit': 2.0},
           'logger_cfgs': {'log_dir': str(tmp_path), 'save_model_freq': 1, 'window_lens': 100, 'use_tensorboard': False},
           'env_cfgs': {'obs_dim': 45, 'act_dim': 3, 'max_episode_steps': 7}}
    agent = omnisafe_b200.Agent('PPOEarlyTerminated', env_id, custom_cfgs=cfg)
    agent.learn()
    capsys.readouterr()
    agent.evaluate(num_episodes=200, num_envs=64)
    out = capsys.readouterr().out
    assert out.count('Evaluation results:') == 2 and out.count('Episode length:') == 400
    ev = agent._evaluator
    assert len(ev.episode_lengths) == 200 and all(1 <= x <= 7 for x in ev.episode_lengths)


def test_evaluate_between_epochs_changes_nothing(cuda, tmp_path, monkeypatch, capsys):
    """Evaluating a checkpoint with many envs (graph replay and the reset_envs path) between two training epochs leaves
    the next epoch's slabs and parameters bit-identical."""
    import omnisafe_b200

    monkeypatch.delenv('OSB_NO_GRAPH', raising=False)
    N, T = 64, 32
    results = []
    for k, evaluate in enumerate((False, True)):
        cfg = {'seed': 3, 'train_cfgs': {'device': 'cuda', 'vector_env_nums': N, 'total_steps': N * T * 2, 'parallel': 1},
               'algo_cfgs': {'steps_per_epoch': N * T, 'batch_size': 256, 'update_iters': 2, 'cost_limit': 2.0},
               'logger_cfgs': {'log_dir': str(tmp_path / f'run{k}'), 'save_model_freq': 1, 'window_lens': 100,
                               'use_tensorboard': False},
               'env_cfgs': {'obs_dim': 45, 'act_dim': 3, 'max_episode_steps': 7}}
        agent = omnisafe_b200.Agent('PPOEarlyTerminated', ee.GRAPH_RESET_WIDE_ID, custom_cfgs=cfg)
        agent.agent.train_epoch()
        agent.agent._logger.torch_save()
        if evaluate:
            agent.evaluate(num_episodes=100, num_envs=50)
        agent.agent.train_epoch()
        slabs = {key: v.clone() for key, v in agent.agent._buf.data.items() if v is not None}
        results.append((agent.agent._actor_critic.theta.clone(), slabs))
    capsys.readouterr()
    assert torch.equal(results[0][0], results[1][0])
    for key, v in results[0][1].items():
        assert torch.equal(v, results[1][1][key]), key
