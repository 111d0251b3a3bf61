"""GPU: PPOEarlyTerminated / TRPOEarlyTerminated on registered envs -- the cost-limit rule in the observe kernel, the
reset of the cut envs through env.reset() (one env, as upstream) or through the optional reset_envs(mask) hook (any
number of envs, graph replay), against the unmodified reference (golden fixtures) and the oracle; end to end through
Agent, evaluate and resume."""
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

import early_envs as ee
import external_envs as xe
from oracle import actor_critic as oac
from oracle.early_external import rollout_epoch_early
from oracle.normalizer import Normalizer as ONormalizer
from test_external_env_gpu import _check_golden, _model_cfgs

pytestmark = pytest.mark.gpu
TERM, TRUNC = 1, 2


@pytest.fixture(scope='module', autouse=True)
def _registered():
    from omnisafe_b200.envs import CMDP, Box, ENV_REGISTRY, env_register

    xe.register(CMDP, Box, env_register, ENV_REGISTRY.support_envs())
    ee.register(CMDP, Box, env_register, ENV_REGISTRY.support_envs())


def _rollout(monkeypatch, dev, env_id, N, T, O, A, seed, theta, eps, precision, cost_limit, epochs, graph=False,
             window=10, **env_cfgs):
    from omnisafe_b200.adapter.early_terminated_adapter import ExternalEarlyTerminatedAdapter
    from omnisafe_b200.common.buffer import VectorOnPolicyBuffer
    from omnisafe_b200.models import ConstraintActorCritic

    if graph:
        monkeypatch.delenv('OSB_NO_GRAPH', raising=False)
    else:
        monkeypatch.setenv('OSB_NO_GRAPH', '1')
    cfgs = NS(algo_cfgs=NS(obs_normalize=True, reward_normalize=False, cost_normalize=False, cost_limit=cost_limit),
              logger_cfgs=NS(window_lens=window), env_cfgs=dict(obs_dim=O, act_dim=A, **env_cfgs))
    ad = ExternalEarlyTerminatedAdapter(env_id, N, seed, cfgs, device=dev)
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
        out['cost_logger'] = ad._cost_logger.cpu().numpy().copy()
        outs.append(out)
    return ad, buf, outs


def _golden(golden_dir):
    g = np.load(os.path.join(golden_dir, 'rollout_external_early.npz'))
    dims = tuple(int(g[k]) for k in ('N', 'T', 'O', 'A', 'epochs_rolled'))
    return g, dims


@pytest.mark.parametrize('precision,tol', [(0, 2e-5), (2, 2e-5), (1, 5e-3)])
def test_early_golden_reference(cuda, monkeypatch, golden_dir, precision, tol):
    """One WideBox env without the hook: env.reset() after a trigger, eager, against two reference epochs."""
    g, (N, T, O, A, E) = _golden(golden_dir)
    ad, buf, outs = _rollout(monkeypatch, cuda, xe.WIDE_BOX_ID, N, T, O, A, int(g['seed']), g['theta'],
                             g['eps'].reshape(E, T, N, A), precision, float(g['cost_limit']), E,
                             max_episode_steps=int(g['tmax']))
    assert ad.graph_mode == 'eager' and not ad._hook
    sl = outs[-1]
    trig = g['slab_reward'][:, 0] == 0
    flags = sl['flags'][:, 0]
    assert ((flags & TERM) != 0)[trig & ~g['env_term'][-1]].all()
    _check_golden(ad, buf, sl, g, tol)


@pytest.mark.parametrize('precision', [0, 2])
def test_early_golden_hook_equals_reset(cuda, monkeypatch, golden_dir, precision):
    """The same run through reset_envs(mask) gives the same bits as through env.reset(), and the reference's values."""
    g, (N, T, O, A, E) = _golden(golden_dir)
    args = (N, T, O, A, int(g['seed']), g['theta'], g['eps'].reshape(E, T, N, A), precision, float(g['cost_limit']), E)
    _, _, plain = _rollout(monkeypatch, cuda, xe.WIDE_BOX_ID, *args, max_episode_steps=int(g['tmax']))
    ad, buf, hook = _rollout(monkeypatch, cuda, ee.RESET_WIDE_ID, *args, max_episode_steps=int(g['tmax']))
    assert ad._hook
    for e in range(E):
        for k in plain[e]:
            assert np.array_equal(plain[e][k], hook[e][k]), f'epoch {e}: {k}'
    _check_golden(ad, buf, hook[-1], g, 2e-5)


def test_early_synthetic_box_reproduces_fused_golden(cuda, monkeypatch, golden_dir):
    """The synthetic dynamics as a single registered env reproduce the unmodified PPOEarlyTerminated rollout that the
    fused synthetic path is checked against (rollout_ppoearly.npz)."""
    g = np.load(os.path.join(golden_dir, 'rollout_ppoearly.npz'))
    N, T, O, A = int(g['N']), int(g['T']), int(g['O']), int(g['A'])
    ad, buf, outs = _rollout(monkeypatch, cuda, xe.ORACLE_BOX_ID, N, T, O, A, int(g['seed']), g['theta'],
                             g['eps'][None], 0, float(g['algo_cost_limit']), 1, max_episode_steps=int(g['tmax']),
                             term_prob=float(g['term_prob']))
    assert (g['slab_reward'] == 0).sum() >= 10
    _check_golden(ad, buf, outs[0], g, 2e-5)


def _compare(sl, ref, tol=2e-5):
    t = dict(rtol=tol, atol=tol)
    for a, b in (('obs', 'obs'), ('act', 'act'), ('reward', 'rew'), ('value_r', 'val_r'), ('value_c', 'val_c')):
        np.testing.assert_allclose(sl[a], ref[b], err_msg=a, **t)
    np.testing.assert_allclose(sl['logp'], ref['logp'], rtol=tol, atol=5e-5)
    assert np.array_equal(sl['cost'], ref['cost'])
    assert np.array_equal(sl['flags'], ref['flags'])
    ends = ref['flags'] != 0
    ends[-1, :] = True
    need = ends & ((ref['flags'] & TERM) == 0)
    np.testing.assert_allclose(sl['boot_r'][need], ref['boot_r'][need], **t)
    np.testing.assert_allclose(sl['boot_c'][need], ref['boot_c'][need], **t)


@pytest.mark.timeout(900)
@pytest.mark.parametrize('N,O,precision,limit', [(7, 17, 0, 0.5), (256, 45, 2, 1.5), (4096, 111, 2, 0.5),
                                                 (4096, 45, 1, 1.5)])
def test_early_hook_vs_oracle(cuda, monkeypatch, N, O, precision, limit):
    """reset_envs with many envs: B1 / B2 / B3 pushes of oracle/early_external.py, two epochs, accumulators carried.
    A limit below 1 cuts every step with a cost (back-to-back triggers); 1.5 carries the accumulator across steps."""
    T, A, tmax = 16, 3, 5
    tol = 5e-3 if precision == 1 else 2e-5
    theta = oac.init_theta(O, A, seed=5)
    eps = np.random.default_rng(N + O).standard_normal((2, T, N, A)).astype(np.float32)
    ad, _, outs = _rollout(monkeypatch, cuda, ee.RESET_WIDE_ID, N, T, O, A, 11, theta, eps, precision, limit, 2,
                           window=16, max_episode_steps=tmax)
    env, norm, window = ee.WideBoxResetOracle(N, O, A, tmax, seed=11), ONormalizer((O,)), []
    early = {'cost_limit': limit, 'acc': np.zeros(N, np.float32)}
    lo, hi = xe.wide_box_bounds(A)
    both = b2b = 0
    for e in range(2):
        ref = rollout_epoch_early(env, norm, theta, T, eps[e], early, lo, hi, window=window)
        trig = early['trig']
        both += int((trig & ((ref['flags'] & TRUNC) != 0)).sum())
        b2b += int((trig[1:] & trig[:-1]).sum())
        _compare(outs[e], ref, tol)
        assert np.array_equal(outs[e]['cost_logger'], early['acc'])
    assert both > 0, both
    assert b2b > 0 if limit < 1 else (early['acc'] > 0).any(), b2b
    np.testing.assert_allclose(outs[-1]['norm_mean'], norm.mean, rtol=tol, atol=tol)
    np.testing.assert_allclose(outs[-1]['norm_std'], norm.std, rtol=tol, atol=tol)
    assert int(outs[-1]['norm_count'][0]) == norm.count
    w = np.array(window[-16:], np.float32)
    meta, ring = outs[-1]['ep_meta'], outs[-1]['ep_ring']
    order = [(int(meta[1]) - int(meta[0]) + i) % 16 for i in range(int(meta[0]))]
    np.testing.assert_allclose(ring[0][order], w[:, 0], rtol=max(tol, 1e-5), atol=max(tol, 1e-5))
    np.testing.assert_allclose(ring[2][order], w[:, 2])


@pytest.mark.parametrize('parity', [False, True])
@pytest.mark.parametrize('precision', [0, 2])
def test_early_graph_equals_eager(cuda, monkeypatch, precision, parity):
    """A graph-safe env with reset_envs: four epochs replayed from the CUDA graph equal the eager run bit for bit, and
    env.reset() runs only at the start of each epoch (never inside the captured steps)."""
    N, T, O, A, E = 256, 16, 45, 3, 4
    theta = oac.init_theta(O, A, seed=6)
    eps = np.random.default_rng(3).standard_normal((E, T, N, A)).astype(np.float32) if parity else None
    kw = dict(max_episode_steps=5)
    ad, _, graph = _rollout(monkeypatch, cuda, ee.GRAPH_RESET_WIDE_ID, N, T, O, A, 5, theta, eps, precision, 1.5, E,
                            graph=True, **kw)
    assert ad.graph_mode == 'graph' and ad.captures == 1 and ad.env._core.resets == E
    _, _, eager = _rollout(monkeypatch, cuda, ee.GRAPH_RESET_WIDE_ID, N, T, O, A, 5, theta, eps, precision, 1.5, E,
                           graph=False, **kw)
    for e in range(E):
        assert graph[e].keys() == eager[e].keys()
        for k in graph[e]:
            assert np.array_equal(graph[e][k], eager[e][k]), f'epoch {e}: {k} differs between graph and eager'
    assert (graph[-1]['reward'] == 0).sum() > N


def test_graph_safe_env_without_hook_runs_eagerly(cuda, monkeypatch):
    from test_external_graph_gpu import GRAPH_WIDE_ID, _graph_envs
    from omnisafe_b200.envs import CMDP, Box, ENV_REGISTRY, env_register

    if GRAPH_WIDE_ID not in ENV_REGISTRY.support_envs():
        for cls in _graph_envs(CMDP, Box):
            env_register(cls)
    O, A, T = 45, 3, 16
    ad, _, outs = _rollout(monkeypatch, cuda, GRAPH_WIDE_ID, 1, T, O, A, 2, oac.init_theta(O, A, seed=2), None, 2,
                           1.5, 3, graph=True, max_episode_steps=5)
    assert ad.graph_mode == 'eager' and ad.captures == 0 and 'reset_envs' in ad._why_eager


def _custom(tmp, N, T=32, epochs=4, algo_cfgs=None, **env):
    return {
        'seed': 3,
        'train_cfgs': {'device': 'cuda', 'vector_env_nums': N, 'total_steps': N * T * epochs, 'parallel': 1},
        'algo_cfgs': {'steps_per_epoch': N * T, 'batch_size': min(256, N * T), 'update_iters': 2, 'cost_limit': 2.0,
                      **(algo_cfgs or {})},
        'logger_cfgs': {'log_dir': str(tmp), 'save_model_freq': 2, 'window_lens': 100, 'use_tensorboard': False},
        'env_cfgs': {'obs_dim': 45, 'act_dim': 3, 'max_episode_steps': 7, **env},
    }


@pytest.mark.timeout(900)
@pytest.mark.parametrize('graph', [False, True])
@pytest.mark.parametrize('algo', ['PPOEarlyTerminated', 'TRPOEarlyTerminated'])
def test_agent_early_learns_on_registered_env(cuda, monkeypatch, tmp_path, algo, graph):
    import omnisafe_b200

    if graph:
        monkeypatch.delenv('OSB_NO_GRAPH', raising=False)
        env_id, N = ee.GRAPH_RESET_WIDE_ID, 256
    else:
        env_id, N = ee.SEEDED_WIDE_ID, 1
    agent = omnisafe_b200.Agent(algo, env_id, custom_cfgs=_custom(tmp_path, N, T=64 if N == 1 else 32,
                                                                  algo_cfgs={'cost_normalize': True}))
    ep_ret, ep_cost, ep_len = agent.learn()
    assert np.isfinite([ep_ret, ep_cost, ep_len]).all() and 1 <= ep_len <= 7
    ad = agent.agent._env
    assert ad.graph_mode == ('graph' if graph else 'eager')
    assert ad.captures == (1 if graph else 0)
    rows = open(os.path.join(agent.agent.logger.log_dir, 'progress.csv')).read().strip().splitlines()
    assert len(rows) == 1 + 4
    vals = [float(v) for v in rows[-1].split(',') if v not in ('', 'nan')]
    assert np.isfinite(vals).all()
    agent.evaluate(num_episodes=2)
    ev = agent._evaluator
    assert len(ev.episode_lengths) == 2 and all(1 <= n <= 7 for n in ev.episode_lengths)


@pytest.mark.timeout(900)
@pytest.mark.parametrize('graph', [False, True])
def test_early_resume_bitwise(cuda, monkeypatch, tmp_path, graph):
    """A run resumed from epoch 2 in a fresh process lands on the uninterrupted run's epoch-4 state, checkpoint and
    progress.csv rows, bit for bit: one env through env.reset() (eager), or 256 envs through reset_envs (replayed)."""
    import early_resume_worker as erw
    import resume_worker as rw
    import test_resume_gpu as tr

    erw.register_envs()
    monkeypatch.setattr(tr, 'WORKER', os.path.join(tr.ROOT, 'tests', 'early_resume_worker.py'))
    env = dict(os.environ)
    if graph:
        monkeypatch.delenv('OSB_NO_GRAPH', raising=False)
        env.pop('OSB_NO_GRAPH', None)
        env_id, N = erw.GRAPH_RESET_ID, 256
    else:
        monkeypatch.setenv('OSB_NO_GRAPH', '1')
        env['OSB_NO_GRAPH'] = '1'
        env_id, N = rw.WIDE_ID, 1
    info = tr._train_and_resume(tmp_path, 'PPOEarlyTerminated', env_id, _custom(tmp_path, N, T=64 if N == 1 else 32),
                                env=env)
    assert info['graph_mode'] == ('graph' if graph else 'eager')
    assert info['captures'] == ([0, 1] if graph else [0, 0])
