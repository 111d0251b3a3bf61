"""GPU: CUDA-graph replay of the external-env rollout for envs that declare `graph_safe`.

The graph-safe envs here keep the arithmetic of tests/external_envs.py::WideBoxCore and of the TorchBox dynamics of
tools/external_env_bench.py bit for bit; only their state updates are in place and their step info always carries the
final observation.  Epoch 0 of an adapter runs eagerly, epoch 1 captures and replays, later epochs replay."""
import os

import numpy as np
import pytest
import torch

import external_envs as xe
from oracle import actor_critic as oac
from test_external_env_gpu import _cfgs, _check_golden, _custom, _model_cfgs

pytestmark = pytest.mark.gpu

GRAPH_WIDE_ID = 'GraphWideBox-v0'
GRAPH_TORCH_ID = 'GraphTorchBox-v0'
M32 = 0xFFFFFFFF


class GraphWideBoxCore(xe.WideBoxCore):
    """WideBoxCore with its state written in place (a replay reads what the previous one wrote)."""

    def reset(self):
        self.episode += 1
        self.ep_step.zero_()
        self.s.copy_(self._reset_values(self.episode))
        return self.s

    def step(self, a):
        a = a.to(self.dev, torch.float32).reshape(self.N, self.A)
        sn = self.s * 0.9 + (a[:, self.idx] * 0.05) * self.scale
        reward = a[:, 0] * 0.5 - sn[:, 0] * 0.001
        cost = (sn[:, 1 % self.O] > 0).to(torch.float32)
        term = ((self.gid * 7 + self.gstep * 13) % 11) == 0
        trunc = (self.ep_step + 1) >= self.tmax
        fin = term | trunc
        self.gstep += 1
        self.episode.copy_(torch.where(fin, self.episode + 1, self.episode))
        self.s.copy_(torch.where(fin[:, None], self._reset_values(self.episode), sn))
        self.ep_step.copy_(torch.where(fin, torch.zeros_like(self.ep_step), self.ep_step + 1))
        return self.s.clone(), reward, cost, term, trunc, sn, fin


def _mix(x):
    x = x ^ (x >> 16)
    x = (x * 0x7FEB352D) & M32
    x = x ^ (x >> 15)
    x = (x * 0x846CA68B) & M32
    return x ^ (x >> 16)


def _graph_envs(CMDP, Box):
    WideBox = xe.wide_box_cmdp(CMDP, Box)

    class GraphWideBox(WideBox):
        _support_envs = [GRAPH_WIDE_ID]  # noqa: RUF012
        graph_safe = True

        def set_seed(self, seed):
            self._core = GraphWideBoxCore(*self._kw, seed=seed, device=self._device)

        def step(self, action):
            nobs, rew, cost, term, trunc, final, fin = self._core.step(torch.as_tensor(action))
            return nobs, rew, cost, term, trunc, {'final_observation': final, '_final_observation': fin}

    class GraphTorchBox(CMDP):
        """The TorchBox dynamics (synthetic env in PyTorch: hash resets, clipped linear step, time-limit truncation)."""
        _support_envs = [GRAPH_TORCH_ID]  # noqa: RUF012
        need_auto_reset_wrapper = need_time_limit_wrapper = need_evaluation = False
        graph_safe = True

        def __init__(self, env_id, num_envs=1, device='cuda', obs_dim=60, act_dim=8, max_episode_steps=64, **_):
            super().__init__(env_id)
            self._num_envs, self._device = num_envs, torch.device(device)
            dev = self._device
            self._observation_space, self._action_space = Box(-10.0, 10.0, (obs_dim,)), Box(-1.0, 1.0, (act_dim,))
            self.tmax, self.seed = max_episode_steps, 0
            self.j = torch.arange(obs_dim, device=dev)
            self.idx = self.j % act_dim
            self.bias = 0.02 * (((7 * self.j + 3) % 5) - 2).to(torch.float32)
            self.gid = torch.arange(num_envs, device=dev)
            self.episode = torch.zeros(num_envs, dtype=torch.int64, device=dev)
            self.ep_step = torch.zeros(num_envs, dtype=torch.int64, device=dev)
            self.s = torch.zeros(num_envs, obs_dim, device=dev)

        def _reset_values(self, episode):
            h = _mix(self.seed ^ ((self.gid[:, None] * 0x9E3779B1) & M32))
            h = _mix(h ^ ((episode[:, None] * 0x85EBCA77) & M32))
            h = _mix(h ^ ((self.j[None, :] * 0xC2B2AE3D) & M32))
            return (h >> 8).to(torch.float32) * (1.0 / 8388608.0) - 1.0

        def set_seed(self, seed):
            self.seed = int(seed) & M32

        def reset(self, seed=None, options=None):
            self.episode += 1
            self.ep_step.zero_()
            self.s.copy_(self._reset_values(self.episode))
            return self.s, {}

        def step(self, action):
            a = action.clamp(-1.0, 1.0)
            sn = (0.95 * self.s + 0.1 * a[:, self.idx] + self.bias).clamp(-10.0, 10.0)
            reward = 1.0 - (sn * sn).mean(1)
            cost = (sn[:, 0] > 0.0).to(torch.float32)
            trunc = (self.ep_step + 1) >= self.tmax
            term = torch.zeros_like(trunc)
            self.episode.copy_(torch.where(trunc, self.episode + 1, self.episode))
            self.s.copy_(torch.where(trunc[:, None], self._reset_values(self.episode), sn))
            self.ep_step.copy_(torch.where(trunc, torch.zeros_like(self.ep_step), self.ep_step + 1))
            return self.s, reward, cost, term, trunc, {'final_observation': sn, '_final_observation': trunc}

        def close(self):
            pass

    return GraphWideBox, GraphTorchBox


@pytest.fixture(scope='module', autouse=True)
def _registered():
    from omnisafe_b200.envs import CMDP, Box, ENV_REGISTRY, env_register

    xe.register(CMDP, Box, env_register, ENV_REGISTRY.support_envs())
    if GRAPH_WIDE_ID not in ENV_REGISTRY.support_envs():
        for cls in _graph_envs(CMDP, Box):
            env_register(cls)


def _state(ad, buf) -> dict:
    """Every slab, the normaliser state and the episode window, as host arrays."""
    out = {k: v.cpu().numpy().copy() for k, v in buf.data.items() if v is not None}
    nz = ad._obs_normalizer
    for k in ('mean', 'sumsq', 'std', 'mean1', 'std1', 'count'):
        out['norm_' + k] = getattr(nz, k).cpu().numpy().copy()
    out['ep_ring'], out['ep_meta'] = ad.ep_ring.cpu().numpy().copy(), ad.ep_meta.cpu().numpy().copy()
    out['window_sums'] = ad.window_sums.cpu().numpy().copy()
    return out


def _adapter(monkeypatch, dev, env_id, N, T, O, A, seed, theta, precision, graph, **env_cfgs):
    from omnisafe_b200.adapter.external_adapter import ExternalEnvAdapter
    from omnisafe_b200.common.buffer import VectorOnPolicyBuffer
    from omnisafe_b200.models import ConstraintActorCritic

    if graph:
        monkeypatch.delenv('OSB_NO_GRAPH', raising=False)
    else:
        monkeypatch.setenv('OSB_NO_GRAPH', '1')
    ad = ExternalEnvAdapter(env_id, N, seed, _cfgs(True, 10, False, obs_dim=O, act_dim=A, **env_cfgs), device=dev)
    ad.precision = precision
    agent = ConstraintActorCritic(O, A, _model_cfgs(), epochs=1, device=dev)
    agent.load_flat(theta)
    buf = VectorOnPolicyBuffer(O, A, T, 0.99, 0.95, 0.95, 'gae', 0.0, True, True, num_envs=N, device=dev)
    assert ad.graph_mode == ('graph' if graph and ad.env.graph_safe else 'eager')
    return ad, agent, buf


def _run(monkeypatch, dev, env_id, N, T, O, A, seed, theta, eps, precision, epochs, graph, new_buffer_at=None,
         **env_cfgs):
    from omnisafe_b200.common.buffer import VectorOnPolicyBuffer

    ad, agent, buf = _adapter(monkeypatch, dev, env_id, N, T, O, A, seed, theta, precision, graph, **env_cfgs)
    outs = []
    for e in range(epochs):
        if e == new_buffer_at:
            buf = VectorOnPolicyBuffer(O, A, T, 0.99, 0.95, 0.95, 'gae', 0.0, True, True, num_envs=N, device=dev)
        ad.rollout(T, agent, buf, eps=None if eps is None else torch.as_tensor(eps[e]).to(dev))
        torch.cuda.synchronize()
        outs.append(_state(ad, buf))
    return ad, buf, outs


def _assert_same(a, b):
    for e, (x, y) in enumerate(zip(a, b)):
        assert x.keys() == y.keys()
        for k in x:
            assert np.array_equal(x[k], y[k]), f'epoch {e}: {k} differs between graph and eager'


@pytest.mark.parametrize('precision,tol', [(0, 2e-5), (2, 2e-5), (1, 5e-3)])
def test_graph_wide_box_golden(cuda, monkeypatch, golden_dir, precision, tol):
    """Two epochs of the unmodified reference (rollout_external.npz); epoch 1 is the first replay of the graph."""
    g = np.load(os.path.join(golden_dir, 'rollout_external.npz'))
    N, T, O, A, E = int(g['N']), int(g['T']), int(g['O']), int(g['A']), int(g['epochs_rolled'])
    assert E == 2
    ad, agent, buf = _adapter(monkeypatch, cuda, GRAPH_WIDE_ID, N, T, O, A, int(g['seed']), g['theta'], precision,
                              True, max_episode_steps=int(g['tmax']))
    eps = g['eps'].reshape(E, T, N, A)
    for e in range(E):
        ad.rollout(T, agent, buf, eps=torch.as_tensor(eps[e]).to(cuda))
    torch.cuda.synchronize()
    assert ad.captures == 1
    sl = {k: v.cpu().numpy() for k, v in buf.data.items() if v is not None}
    _check_golden(ad, buf, sl, g, tol)


@pytest.mark.parametrize('parity', [False, True])
@pytest.mark.parametrize('precision', [0, 2])
def test_graph_equals_eager_bitwise(cuda, monkeypatch, precision, parity):
    """N = 256, O = 45, four epochs: every slab, epfin, the normaliser and the episode ring are the same bits."""
    N, T, O, A, E = 256, 16, 45, 3, 4
    theta = oac.init_theta(O, A, seed=6)
    eps = np.random.default_rng(3).standard_normal((E, T, N, A)).astype(np.float32) if parity else None
    kw = dict(max_episode_steps=7)
    ad, _, graph = _run(monkeypatch, cuda, GRAPH_WIDE_ID, N, T, O, A, 5, theta, eps, precision, E, True, **kw)
    _, _, eager = _run(monkeypatch, cuda, GRAPH_WIDE_ID, N, T, O, A, 5, theta, eps, precision, E, False, **kw)
    assert ad.captures == 1
    assert graph[-1]['ep_meta'][0] > 0 and (graph[-1]['flags'] & 1).any() and (graph[-1]['flags'] & 2).any()
    _assert_same(graph, eager)


@pytest.mark.timeout(900)
@pytest.mark.parametrize('precision', [0, 2])
def test_graph_equals_eager_headline(cuda, monkeypatch, precision):
    """The graph-safe TorchBox at 4096 envs x T = 128 (the benchmark's shape), Philox noise, two epochs."""
    N, T, O, A = 4096, 128, 60, 8
    theta = oac.init_theta(O, A, seed=3)
    ad, _, graph = _run(monkeypatch, cuda, GRAPH_TORCH_ID, N, T, O, A, 9, theta, None, precision, 2, True,
                        max_episode_steps=64)
    _, _, eager = _run(monkeypatch, cuda, GRAPH_TORCH_ID, N, T, O, A, 9, theta, None, precision, 2, False,
                       max_episode_steps=64)
    assert ad.captures == 1 and (graph[1]['flags'] & 2).any()
    _assert_same(graph, eager)


def test_philox_advances_across_replays(cuda, monkeypatch):
    N, T, O, A = 256, 16, 45, 3
    theta = oac.init_theta(O, A, seed=1)
    ad, _, o1 = _run(monkeypatch, cuda, GRAPH_WIDE_ID, N, T, O, A, 4, theta, None, 2, 4, True)
    _, _, o2 = _run(monkeypatch, cuda, GRAPH_WIDE_ID, N, T, O, A, 4, theta, None, 2, 4, True)
    assert ad.captures == 1
    for e in (1, 2, 3):                                   # replays
        assert not np.array_equal(o1[e]['act'], o1[e - 1]['act']), e
    _assert_same(o1, o2)
    assert int(ad._epoch_dev.item()) == 4                 # the captured advance ran once per replay


def test_new_buffer_recaptures(cuda, monkeypatch):
    """A new VectorOnPolicyBuffer moves every slab: the adapter captures again instead of replaying stale pointers."""
    N, T, O, A, E = 256, 16, 45, 3, 4
    theta = oac.init_theta(O, A, seed=8)
    ad, _, graph = _run(monkeypatch, cuda, GRAPH_WIDE_ID, N, T, O, A, 2, theta, None, 2, E, True, new_buffer_at=2)
    _, _, eager = _run(monkeypatch, cuda, GRAPH_WIDE_ID, N, T, O, A, 2, theta, None, 2, E, False, new_buffer_at=2)
    assert ad.captures == 2
    _assert_same(graph, eager)


def test_env_without_graph_safe_is_never_captured(cuda, monkeypatch):
    N, T, O, A = 64, 8, 45, 3
    ad, _, _ = _run(monkeypatch, cuda, xe.WIDE_BOX_ID, N, T, O, A, 2, oac.init_theta(O, A, seed=2), None, 2, 3, True)
    assert ad.graph_mode == 'eager' and ad.captures == 0 and ad._graph is None


def test_nonfinite_observation_in_graph_mode_raises_once(cuda, monkeypatch):
    from omnisafe_b200._lib import OsbError

    N, T, O, A = 32, 8, 45, 3
    ad, agent, buf = _adapter(monkeypatch, cuda, GRAPH_WIDE_ID, N, T, O, A, 1, oac.init_theta(O, A, seed=2), 0, True)
    core = ad.env._core
    poison = torch.zeros(N, O, dtype=torch.bool, device=cuda)
    step, calls = core.step, []

    def poisoned_step(a):
        out = list(step(a))
        calls.append(1)
        out[0] = torch.where(poison, float('nan'), out[0])     # the mask is read on the device at every replay
        return tuple(out)

    core.step = poisoned_step
    ad.rollout(T, agent, buf)                                   # eager
    ad.rollout(T, agent, buf)                                   # capture + first replay
    assert len(calls) == 2 * T and ad.captures == 1
    poison[5, 7] = True
    with pytest.raises(OsbError, match='non-finite observation'):
        ad.rollout(T, agent, buf)
    assert len(calls) == 2 * T                                  # the env's Python ran at capture only
    poison.zero_()
    ad.rollout(T, agent, buf)                                   # raised once: the flag was cleared
    assert ad.captures == 1


@pytest.mark.parametrize('algo', ['PPOLag', 'CPO'])
def test_agent_trains_in_graph_mode(cuda, monkeypatch, tmp_path, algo):
    import omnisafe_b200
    from omnisafe_b200.common.normalizer import Normalizer

    monkeypatch.delenv('OSB_NO_GRAPH', raising=False)
    agent = omnisafe_b200.Agent(algo, GRAPH_WIDE_ID, custom_cfgs=_custom(tmp_path, epochs=3))
    ep_ret, ep_cost, ep_len = agent.learn()
    assert np.isfinite([ep_ret, ep_cost, ep_len]).all() and 1 <= ep_len <= 7
    ad = agent.agent._env
    assert ad.graph_mode == 'graph' and ad.captures == 1
    log_dir = agent.agent.logger.log_dir
    rows = open(os.path.join(log_dir, 'progress.csv')).read().strip().splitlines()
    assert len(rows) == 1 + 3
    vals = [float(v) for v in rows[-1].split(',') if v not in ('', 'nan')]
    assert np.isfinite(vals).all()
    ckpt = torch.load(os.path.join(log_dir, 'torch_save', 'epoch-3.pt'), weights_only=False)
    assert ckpt['pi']['mean.0.weight'].shape == (64, 45)
    nz = Normalizer((45,), device=cuda)
    nz.load_state_dict(ckpt['obs_normalizer'])
    np.testing.assert_allclose(nz.mean.cpu().numpy(), ad._obs_normalizer.mean.cpu().numpy())
