"""GPU: registered envs behind TimeLimit and AutoReset -- the wrapper step on the device, the reset of the done envs
through env.reset() (one env, as upstream) or through reset_envs(mask) (any number of envs, graph replay), against the
unmodified reference (golden fixtures), the fused path's golden and the oracle; end to end through Agent, evaluate and
resume."""
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

import external_envs as xe
import wrapper_envs as we
from oracle import actor_critic as oac
from oracle.normalizer import Normalizer as ONormalizer
from oracle.wrapped_external import rollout_epoch_wrapped
from test_external_early_gpu import _compare
from test_external_env_gpu import _check_golden, _model_cfgs

pytestmark = pytest.mark.gpu
TERM, TRUNC = 1, 2


@pytest.fixture(scope='module', autouse=True)
def _registered():
    from omnisafe_b200.envs import CMDP, Box, ENV_REGISTRY, env_register

    xe.register(CMDP, Box, env_register, ENV_REGISTRY.support_envs())
    we.register(CMDP, Box, env_register, ENV_REGISTRY.support_envs())


def _rollout(monkeypatch, dev, env_id, N, T, O, A, seed, theta, eps, precision, epochs, graph=False, window=10,
             **env_cfgs):
    from omnisafe_b200.adapter.external_adapter import ExternalEnvAdapter
    from omnisafe_b200.common.buffer import VectorOnPolicyBuffer
    from omnisafe_b200.models import ConstraintActorCritic

    if graph:
        monkeypatch.delenv('OSB_NO_GRAPH', raising=False)
    else:
        monkeypatch.setenv('OSB_NO_GRAPH', '1')
    cfgs = NS(algo_cfgs=NS(obs_normalize=True, reward_normalize=False, cost_normalize=False),
              logger_cfgs=NS(window_lens=window), env_cfgs=dict(obs_dim=O, act_dim=A, **env_cfgs))
    ad = ExternalEnvAdapter(env_id, N, seed, cfgs, device=dev)
    ad.precision = precision
    agent = ConstraintActorCritic(O, A, _model_cfgs(), epochs=1, device=dev)
    agent.load_flat(theta)
    buf = VectorOnPolicyBuffer(O, A, T, 0.99, 0.95, 0.95, 'gae', 0.0, True, True, num_envs=N, device=dev)
    outs = []
    for e in range(epochs):
        ad.rollout(T, agent, buf, eps=None if eps is None else torch.as_tensor(eps[e]).to(dev))
        torch.cuda.synchronize()
        out = {k: v.cpu().numpy().copy() for k, v in buf.data.items() if v is not None}
        nz = ad._obs_normalizer
        for k in ('mean', 'sumsq', 'std', 'mean1', 'std1', 'count'):
            out['norm_' + k] = getattr(nz, k).cpu().numpy().copy()
        out['ep_ring'], out['ep_meta'] = ad.ep_ring.cpu().numpy().copy(), ad.ep_meta.cpu().numpy().copy()
        outs.append(out)
    return ad, buf, outs


GOLDENS = {'rollout_external_wrappers.npz': we.WRAPPED_ID, 'rollout_external_autoreset.npz': we.AUTO_RESET_ID}


def _golden(golden_dir, fname):
    g = np.load(os.path.join(golden_dir, fname))
    return g, tuple(int(g[k]) for k in ('N', 'T', 'O', 'A', 'epochs_rolled'))


@pytest.mark.parametrize('fname', list(GOLDENS))
@pytest.mark.parametrize('precision,tol', [(0, 2e-5), (2, 2e-5), (1, 5e-3)])
def test_wrappers_golden_reference(cuda, monkeypatch, golden_dir, fname, precision, tol):
    """One env without the hook: the done word read back, env.reset() when set, eager, against two reference epochs."""
    g, (N, T, O, A, E) = _golden(golden_dir, fname)
    ad, buf, outs = _rollout(monkeypatch, cuda, GOLDENS[fname], N, T, O, A, int(g['seed']), g['theta'],
                             g['eps'].reshape(E, T, N, A), precision, E, max_episode_steps=int(g['tmax']))
    assert ad.graph_mode == 'eager' and not ad._reset_hook
    _check_golden(ad, buf, outs[-1], g, tol)


@pytest.mark.parametrize('precision', [0, 2])
def test_wrappers_hook_equals_reset(cuda, monkeypatch, golden_dir, precision):
    """The same run through reset_envs(mask) gives the same bits as through env.reset(), and the reference's values."""
    g, (N, T, O, A, E) = _golden(golden_dir, 'rollout_external_wrappers.npz')
    args = (N, T, O, A, int(g['seed']), g['theta'], g['eps'].reshape(E, T, N, A), precision, E)
    _, _, plain = _rollout(monkeypatch, cuda, we.WRAPPED_ID, *args, max_episode_steps=int(g['tmax']))
    ad, buf, hook = _rollout(monkeypatch, cuda, we.WRAPPED_RESET_ID, *args, max_episode_steps=int(g['tmax']))
    assert ad._reset_hook
    for e in range(E):
        for k in plain[e]:
            assert np.array_equal(plain[e][k], hook[e][k]), f'epoch {e}: {k}'
    _check_golden(ad, buf, hook[-1], g, 2e-5)


def test_wrapped_synthetic_box_reproduces_fused_golden(cuda, monkeypatch, golden_dir):
    """The synthetic dynamics without their own auto-reset, behind TimeLimit / AutoReset with reset_envs, reproduce
    the unmodified PPOLag rollout that the fused synthetic path is checked against (rollout_ppolag.npz)."""
    g = np.load(os.path.join(golden_dir, 'rollout_ppolag.npz'))
    N, T, O, A = int(g['N']), int(g['T']), int(g['O']), int(g['A'])
    ad, buf, outs = _rollout(monkeypatch, cuda, we.WRAPPED_SYNTH_ID, N, T, O, A, int(g['seed']), g['theta'],
                             g['eps'][None], 0, 1, max_episode_steps=int(g['tmax']), term_prob=float(g['term_prob']))
    assert ad._reset_hook and ad._time_limit == int(g['tmax'])
    _check_golden(ad, buf, outs[0], g, 2e-5)


@pytest.mark.timeout(900)
@pytest.mark.parametrize('O', [17, 45, 111])
@pytest.mark.parametrize('N', [7, 256, 4096])
def test_wrappers_hook_vs_oracle(cuda, monkeypatch, N, O):
    """reset_envs with many envs, two epochs, per-env TimeLimit counters: the pushes of oracle/wrapped_external.py."""
    T, A, tmax = 16, 3, 4
    precision = (N + O) % 3
    tol = 5e-3 if precision == 1 else 2e-5
    theta = oac.init_theta(O, A, seed=5)
    eps = np.random.default_rng(N + O).standard_normal((2, T, N, A)).astype(np.float32)
    ad, _, outs = _rollout(monkeypatch, cuda, we.WRAPPED_RESET_ID, N, T, O, A, 11, theta, eps, precision, 2,
                           window=16, max_episode_steps=tmax)
    env, norm, window = we.WrappedBoxOracle(N, O, A, seed=11), ONormalizer((O,)), []
    lo, hi = xe.wide_box_bounds(A)
    both = 0
    for e in range(2):
        ref = rollout_epoch_wrapped(env, norm, theta, T, eps[e], tmax, lo, hi, window=window)
        both += int((((ref['flags'] & TERM) != 0) & ((ref['flags'] & TRUNC) != 0)).sum())
        _compare(outs[e], ref, tol)
    assert both > 0
    np.testing.assert_allclose(outs[-1]['norm_mean'], norm.mean, rtol=tol, atol=tol)
    np.testing.assert_allclose(outs[-1]['norm_std'], norm.std, rtol=tol, atol=tol)
    assert int(outs[-1]['norm_count'][0]) == norm.count
    w = np.array(window[-16:], np.float32)
    meta, ring = outs[-1]['ep_meta'], outs[-1]['ep_ring']
    order = [(int(meta[1]) - int(meta[0]) + i) % 16 for i in range(int(meta[0]))]
    np.testing.assert_allclose(ring[0][order], w[:, 0], rtol=max(tol, 1e-5), atol=max(tol, 1e-5))
    np.testing.assert_allclose(ring[2][order], w[:, 2])


@pytest.mark.parametrize('parity', [False, True])
@pytest.mark.parametrize('N,tmax', [(7, 50), (256, 1), (256, 4)])
def test_wrappers_graph_equals_eager(cuda, monkeypatch, N, tmax, parity):
    """A graph-safe env with reset_envs and no final observation in info: four epochs replayed from the CUDA graph
    equal the eager run bit for bit, and env.reset() runs only at the start of each epoch.  tmax = 1 resets every env
    on every step; at 7 envs and a far limit some steps reset none."""
    T, O, A, E = 16, 45, 3, 4
    theta = oac.init_theta(O, A, seed=6)
    eps = np.random.default_rng(3).standard_normal((E, T, N, A)).astype(np.float32) if parity else None
    ad, _, graph = _rollout(monkeypatch, cuda, we.GRAPH_WRAPPED_ID, N, T, O, A, 5, theta, eps, 2, E, graph=True,
                            max_episode_steps=tmax)
    assert ad.graph_mode == 'graph' and ad.captures == 1 and ad.env._core.resets == E
    _, _, eager = _rollout(monkeypatch, cuda, we.GRAPH_WRAPPED_ID, N, T, O, A, 5, theta, eps, 2, E, graph=False,
                           max_episode_steps=tmax)
    for e in range(E):
        assert graph[e].keys() == eager[e].keys()
        for k in graph[e]:
            assert np.array_equal(graph[e][k], eager[e][k]), f'epoch {e}: {k} differs between graph and eager'
    done = np.stack([o['flags'] for o in graph]) != 0
    if tmax == 1:
        assert done.all()
    if N == 7:
        assert (~done).all(axis=-1).any() and done.any()


def _custom(tmp, N, T=32, epochs=4, algo_cfgs=None, **env):
    return {
        'seed': 3,
        'train_cfgs': {'device': 'cuda', 'vector_env_nums': N, 'total_steps': N * T * epochs, 'parallel': 1},
        'algo_cfgs': {'steps_per_epoch': N * T, 'batch_size': min(256, N * T), 'update_iters': 2,
                      **(algo_cfgs or {})},
        'logger_cfgs': {'log_dir': str(tmp), 'save_model_freq': 2, 'window_lens': 100, 'use_tensorboard': False},
        'env_cfgs': {'obs_dim': 45, 'act_dim': 3, 'max_episode_steps': 7, **env},
    }


def _eval_lengths(E, num_episodes, limit=1000, own_trunc=False):
    """The episode lengths of an evaluation of the wrapped box: its ends depend on its step counter only."""
    gstep, left, out = [0] * E, [(num_episodes - e + E - 1) // E for e in range(E)], {}
    for e in range(E):
        for k in range(left[e]):
            n = 0
            while True:
                g = gstep[e]
                gstep[e] += 1
                n += 1
                term = (e * 7 + g * 13) % 11 == 0 or (e * 3 + g * 5) % 9 == 4
                trunc = (e * 5 + g * 3) % 13 == 4 if own_trunc else n >= limit
                if term or trunc:
                    break
            out[e + k * E] = n
    return [float(out[i]) for i in range(num_episodes)]


@pytest.mark.timeout(900)
@pytest.mark.parametrize('graph', [False, True])
@pytest.mark.parametrize('algo', ['PPOLag', 'FOCOPS', 'CPO'])
def test_agent_learns_on_wrapper_env(cuda, monkeypatch, tmp_path, algo, graph):
    """learn() on a wrapped env, then evaluate(): TimeLimit(1000) discards the env's own truncation, so the episodes end
    at its terminations; E = 64 resets the finished envs through reset_envs (replayed from a graph when graph-safe)."""
    import omnisafe_b200

    if graph:
        monkeypatch.delenv('OSB_NO_GRAPH', raising=False)
        env_id, N = we.GRAPH_WRAPPED_ID, 256
    else:
        monkeypatch.setenv('OSB_NO_GRAPH', '1')
        env_id, N = we.WRAPPED_ID, 1
    agent = omnisafe_b200.Agent(algo, env_id, custom_cfgs=_custom(tmp_path, N, T=64 if N == 1 else 32))
    ep_ret, ep_cost, ep_len = agent.learn()
    assert np.isfinite([ep_ret, ep_cost, ep_len]).all() and 1 <= ep_len <= 7
    ad = agent.agent._env
    assert ad.graph_mode == ('graph' if graph else 'eager')
    assert ad.captures == (1 if graph else 0)
    rows = open(os.path.join(agent.agent.logger.log_dir, 'progress.csv')).read().strip().splitlines()
    assert len(rows) == 1 + 4
    agent.evaluate(num_episodes=3)
    assert agent._evaluator.episode_lengths == _eval_lengths(1, 3)
    if graph:
        agent.evaluate(num_episodes=128, num_envs=64)
        assert agent._evaluator.episode_lengths == _eval_lengths(64, 128)
    else:
        with pytest.raises(NotImplementedError, match='reset_envs'):
            agent.evaluate(num_episodes=128, num_envs=64)


def test_evaluate_graph_equals_eager(cuda, monkeypatch, tmp_path):
    """Evaluation at E = 64 on the graph-safe wrapped env: the graph-replayed blocks equal the eager steps bit for bit."""
    import omnisafe_b200

    monkeypatch.setenv('OSB_NO_GRAPH', '1')
    agent = omnisafe_b200.Agent('PPOLag', we.GRAPH_WRAPPED_ID, custom_cfgs=_custom(tmp_path, 64, epochs=2))
    agent.learn()
    res = {}
    for mode in ('eager', 'graph'):
        if mode == 'graph':
            monkeypatch.delenv('OSB_NO_GRAPH', raising=False)
        agent.evaluate(num_episodes=200, num_envs=64)
        ev = agent._evaluator
        res[mode] = (ev.episode_lengths, ev.last_actions.cpu().numpy(), ev.normalizer.mean.cpu().numpy(),
                     ev.normalizer.std.cpu().numpy())
    assert res['eager'][0] == _eval_lengths(64, 200)
    for a, b in zip(res['eager'], res['graph']):
        assert np.array_equal(np.asarray(a), np.asarray(b))


def test_evaluate_auto_reset_only(cuda, monkeypatch, tmp_path):
    """AutoReset alone: the evaluation keeps the env's own truncation (no TimeLimit), one env reset by env.reset()."""
    import omnisafe_b200

    monkeypatch.setenv('OSB_NO_GRAPH', '1')
    agent = omnisafe_b200.Agent('PPOLag', we.AUTO_RESET_ID, custom_cfgs=_custom(tmp_path, 1, T=64, epochs=2))
    agent.learn()
    agent.evaluate(num_episodes=5)
    assert agent._evaluator.episode_lengths == _eval_lengths(1, 5, own_trunc=True)


@pytest.mark.timeout(900)
@pytest.mark.parametrize('graph', [False, True])
def test_wrappers_resume_bitwise(cuda, monkeypatch, tmp_path, graph):
    """A run resumed from epoch 2 in a fresh process lands on the uninterrupted run's epoch-4 state, checkpoint and
    progress.csv rows, bit for bit: one env through env.reset() (eager), or 256 envs through reset_envs (replayed)."""
    import test_resume_gpu as tr
    import wrapper_resume_worker as wrw

    wrw.register_envs()
    monkeypatch.setattr(tr, 'WORKER', os.path.join(tr.ROOT, 'tests', 'wrapper_resume_worker.py'))
    env = dict(os.environ)
    if graph:
        monkeypatch.delenv('OSB_NO_GRAPH', raising=False)
        env.pop('OSB_NO_GRAPH', None)
        env_id, N = wrw.GRAPH_WRAPPED_RESUME_ID, 256
    else:
        monkeypatch.setenv('OSB_NO_GRAPH', '1')
        env['OSB_NO_GRAPH'] = '1'
        env_id, N = wrw.WRAPPED_RESUME_ID, 1
    info = tr._train_and_resume(tmp_path, 'PPOLag', env_id, _custom(tmp_path, N, T=64 if N == 1 else 32), env=env)
    assert info['graph_mode'] == ('graph' if graph else 'eager')
    assert info['captures'] == ([0, 1] if graph else [0, 0])
