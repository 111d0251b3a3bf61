"""GPU: rollout on user-registered CMDPs (env.step in PyTorch, act / observe kernels around it) vs the unmodified
reference (golden fixtures), vs the oracle, and vs the fused synthetic path; end to end through Agent."""
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

import external_envs as xe
from oracle import actor_critic as oac
from oracle import rollout as orollout
from oracle.normalizer import Normalizer as ONormalizer

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _registered():
    from omnisafe_b200.envs import CMDP, Box, ENV_REGISTRY, env_register

    xe.register(CMDP, Box, env_register, ENV_REGISTRY.support_envs())


def _cfgs(obs_normalize=True, window=100, rc_normalize=False, **env_cfgs):
    return NS(algo_cfgs=NS(obs_normalize=obs_normalize, reward_normalize=rc_normalize, cost_normalize=rc_normalize),
              logger_cfgs=NS(window_lens=window), env_cfgs=env_cfgs)


def _model_cfgs():
    net = NS(hidden_sizes=[64, 64], activation='tanh', lr=3e-4)
    return NS(actor=net, critic=net, actor_type='gaussian_learning', linear_lr_decay=True,
              weight_initialization_mode='kaiming_uniform')


def _ext_rollout(dev, env_id, N, T, O, A, seed, theta, eps, precision=0, window=100, epochs=1, rc_normalize=False,
                 obs_normalize=True, **env_cfgs):
    from omnisafe_b200.adapter.external_adapter import ExternalEnvAdapter
    from omnisafe_b200.common.buffer import VectorOnPolicyBuffer
    from omnisafe_b200.models import ConstraintActorCritic

    cfgs = _cfgs(obs_normalize, window, rc_normalize, obs_dim=O, act_dim=A, **env_cfgs)
    ad = ExternalEnvAdapter(env_id, N, seed, cfgs, device=dev)
    ad.precision = precision
    agent = ConstraintActorCritic(O, A, _model_cfgs(), epochs=1, device=dev)
    agent.load_flat(theta)
    buf = VectorOnPolicyBuffer(O, A, T, 0.99, 0.95, 0.95, 'gae', 0.0, True, True, num_envs=N, device=dev)
    outs = []
    for e in range(epochs):
        ad.rollout(T, agent, buf, eps=None if eps is None else torch.as_tensor(eps[e]).to(dev))
        torch.cuda.synchronize()
        outs.append({k: v.cpu().numpy().copy() for k, v in buf.data.items() if v is not None})
    return ad, buf, outs


def _window(ad, W):
    meta, ring = ad.ep_meta.cpu().numpy(), ad.ep_ring.cpu().numpy()
    cnt, head = int(meta[0]), int(meta[1])
    order = [(head - cnt + i) % W for i in range(cnt)]
    return ring[:, order]


def _check_golden(ad, buf, sl, g, tol, W=10):
    t = dict(rtol=tol, atol=tol)
    np.testing.assert_allclose(sl['obs'], g['slab_obs'], **t)
    np.testing.assert_allclose(sl['act'], g['slab_act'], **t)
    np.testing.assert_allclose(sl['reward'], g['slab_reward'], **t)
    assert np.array_equal(sl['cost'], g['slab_cost'])
    np.testing.assert_allclose(sl['value_r'], g['slab_value_r'], **t)
    np.testing.assert_allclose(sl['value_c'], g['slab_value_c'], **t)
    np.testing.assert_allclose(sl['logp'], g['slab_logp'], rtol=tol, atol=max(tol, 5e-5) if tol < 1e-3 else 2e-2)
    nz = ad._obs_normalizer
    np.testing.assert_allclose(nz.mean.cpu().numpy(), g['norm_mean'], **t)      # tf32: the trajectory itself moves by 5e-3
    np.testing.assert_allclose(nz.std.cpu().numpy(), g['norm_std'], **t)
    assert int(nz.count[0]) == int(g['norm_count'])
    buf.finish_paths()
    torch.cuda.synchronize()
    ta = dict(rtol=1e-4, atol=5e-5) if tol < 1e-3 else dict(rtol=2e-2, atol=2e-2)
    np.testing.assert_allclose(buf.data['adv_r'].cpu().numpy(), g['slab_adv_r'], **ta)
    np.testing.assert_allclose(buf.data['adv_c'].cpu().numpy(), g['slab_adv_c'], **ta)
    np.testing.assert_allclose(buf.data['target_value_r'].cpu().numpy(), g['slab_target_value_r'], **ta)
    ring = _window(ad, W)
    assert ring.shape[1] == len(g['win_ret'])
    np.testing.assert_allclose(ring[0], g['win_ret'], rtol=max(tol, 1e-5), atol=max(tol, 1e-5))
    np.testing.assert_allclose(ring[1], g['win_cost'])
    np.testing.assert_allclose(ring[2], g['win_len'])


@pytest.mark.parametrize('precision', [0, 2])
def test_external_synthetic_golden_reference(cuda, golden_dir, precision):
    """The synthetic env as a user CMDP (CUDA tensors) through the external path reproduces the unmodified reference."""
    g = np.load(os.path.join(golden_dir, 'rollout_ppolag.npz'))
    N, T, O, A = int(g['N']), int(g['T']), int(g['O']), int(g['A'])
    ad, buf, outs = _ext_rollout(cuda, xe.ORACLE_BOX_ID, N, T, O, A, int(g['seed']), g['theta'], g['eps'][None],
                                 precision, window=10, max_episode_steps=int(g['tmax']), term_prob=float(g['term_prob']))
    _check_golden(ad, buf, outs[0], g, 2e-5)


def test_external_reward_cost_normalize_golden(cuda, golden_dir):
    g = np.load(os.path.join(golden_dir, 'rollout_pdo.npz'))
    N, T, O, A, E = int(g['N']), int(g['T']), int(g['O']), int(g['A']), int(g['epochs_rolled'])
    ad, buf, outs = _ext_rollout(cuda, xe.ORACLE_BOX_ID, N, T, O, A, int(g['seed']), g['theta'],
                                 g['eps'].reshape(E, T, N, A), 0, window=10, epochs=E, rc_normalize=True,
                                 max_episode_steps=int(g['tmax']), term_prob=float(g['term_prob']))
    sl = outs[-1]
    np.testing.assert_allclose(sl['obs'], g['slab_obs'], rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(sl['reward'], g['slab_reward'], rtol=5e-5, atol=5e-5)
    np.testing.assert_allclose(sl['cost'], g['slab_cost'], rtol=5e-5, atol=5e-5)
    rn, cn = ad.save()['reward_normalizer'], ad.save()['cost_normalizer']
    np.testing.assert_allclose([float(rn.mean), float(rn.std), float(cn.mean), float(cn.std)],
                               [g['rnorm_mean'], g['rnorm_std'], g['cnorm_mean'], g['cnorm_std']], rtol=2e-5)
    buf.finish_paths()
    torch.cuda.synchronize()
    np.testing.assert_allclose(buf.data['adv_r'].cpu().numpy(), g['slab_adv_r'], rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(buf.data['adv_c'].cpu().numpy(), g['slab_adv_c'], rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize('precision,tol', [(0, 2e-5), (2, 2e-5), (1, 5e-3)])
def test_external_wide_box_golden(cuda, golden_dir, precision, tol):
    """Asymmetric action box, |obs| up to ~1e3, terminated and truncated in one step, O = 45: two epochs of the
    unmodified reference (tests/golden/make_golden_external.py)."""
    g = np.load(os.path.join(golden_dir, 'rollout_external.npz'))
    N, T, O, A, E = int(g['N']), int(g['T']), int(g['O']), int(g['A']), int(g['epochs_rolled'])
    ad, buf, outs = _ext_rollout(cuda, xe.WIDE_BOX_ID, N, T, O, A, int(g['seed']), g['theta'],
                                 g['eps'].reshape(E, T, N, A), precision, window=10, epochs=E,
                                 max_episode_steps=int(g['tmax']))
    _check_golden(ad, buf, outs[-1], g, tol)


def _compare(sl, ref, tol=2e-5):
    t = dict(rtol=tol, atol=tol)
    for a, b in (('obs', 'obs'), ('act', 'act'), ('reward', 'rew'), ('value_r', 'val_r'), ('value_c', 'val_c')):
        np.testing.assert_allclose(sl[a], ref[b], err_msg=a, **t)
    np.testing.assert_allclose(sl['logp'], ref['logp'], rtol=tol, atol=5e-5)
    assert np.array_equal(sl['cost'], ref['cost'])
    assert np.array_equal(sl['flags'], ref['flags'])
    ends = ref['flags'] != 0
    ends[-1, :] = True
    need = ends & ((ref['flags'] & 1) == 0)
    np.testing.assert_allclose(sl['boot_r'][need], ref['boot_r'][need], **t)
    np.testing.assert_allclose(sl['boot_c'][need], ref['boot_c'][need], **t)


@pytest.mark.parametrize('N,T,O,A,tmax,precision', [
    (1, 20, 17, 3, 5, 0),         # a single env: unbatched tensors
    (50, 16, 60, 4, 6, 2),        # ragged tiles, bf16x3
    (40, 12, 111, 8, 7, 2),       # O > 64: bf16x3 falls back to the fp32 tiles
    (33, 6, 376, 5, 3, 0),        # Humanoid-like obs dim
])
def test_external_vs_oracle(cuda, monkeypatch, N, T, O, A, tmax, precision):
    """oracle/rollout.py with the env's action bounds, two epochs with state carried over."""
    rng = np.random.default_rng(N + O)
    theta = oac.init_theta(O, A, seed=5)
    eps = rng.standard_normal((2, T, N, A)).astype(np.float32)
    ad, buf, outs = _ext_rollout(cuda, xe.WIDE_BOX_ID, N, T, O, A, 11, theta, eps, precision, window=16, epochs=2,
                                 max_episode_steps=tmax)
    lo, hi = xe.wide_box_bounds(A)
    scale = orollout.action_scale
    monkeypatch.setattr(orollout, 'action_scale', lambda act: scale(act, lo, hi))
    env, norm, window = xe.WideBoxOracle(N, O, A, tmax, seed=11), ONormalizer((O,)), []
    for e in range(2):
        ref = orollout.rollout_epoch(env, norm, theta, T, eps[e], window=window)
        _compare(outs[e], ref)
    w = np.array(window[-16:], np.float32)
    ring = _window(ad, 16)
    np.testing.assert_allclose(ring[0], w[:, 0], rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(ring[2], w[:, 2])
    np.testing.assert_allclose(ad._obs_normalizer.mean.cpu().numpy(), norm.mean, rtol=2e-5, atol=2e-5)


@pytest.mark.timeout(900)
@pytest.mark.parametrize('precision', [0, 2])
def test_external_matches_fused_headline(cuda, precision):
    """The synthetic dynamics through the external path = the fused kernel, at 4096 envs x T = 128, same seed / eps."""
    from omnisafe_b200.adapter.onpolicy_adapter import OnPolicyAdapter
    from omnisafe_b200.common.buffer import VectorOnPolicyBuffer
    from omnisafe_b200.models import ConstraintActorCritic

    N, T, O, A = 4096, 128, 60, 8
    env_cfgs = dict(max_episode_steps=64, term_prob=0.01)
    theta = oac.init_theta(O, A, seed=3)
    eps = np.random.default_rng(7).standard_normal((1, T, N, A)).astype(np.float32)
    _, _, ext = _ext_rollout(cuda, xe.ORACLE_BOX_ID, N, T, O, A, 9, theta, eps, precision, **env_cfgs)
    ad = OnPolicyAdapter('SyntheticBox-v0', N, 9, _cfgs(obs_dim=O, act_dim=A, **env_cfgs), device=cuda)
    ad.precision = precision
    agent = ConstraintActorCritic(O, A, _model_cfgs(), epochs=1, device=cuda)
    agent.load_flat(theta)
    buf = VectorOnPolicyBuffer(O, A, T, 0.99, 0.95, 0.95, 'gae', 0.0, True, True, num_envs=N, device=cuda)
    ad.rollout(T, agent, buf, eps=torch.as_tensor(eps[0]).to(cuda))
    a, b = ext[0], {k: v.cpu().numpy() for k, v in buf.data.items() if v is not None}
    assert (b['flags'] & 1).any() and (b['flags'] & 2).any()
    for k in ('obs', 'act', 'logp', 'reward', 'value_r', 'value_c', 'boot_r', 'boot_c'):
        np.testing.assert_allclose(a[k], b[k], rtol=2e-5, atol=2e-5, err_msg=k)
    for k in ('flags', 'cost'):
        assert np.array_equal(a[k], b[k]), k
    done = b['flags'] != 0
    np.testing.assert_allclose(a['epfin'][:, done], b['epfin'][:, done], rtol=2e-5, atol=2e-5)


def _custom(tmp, N=64, T=32, epochs=2, **algo):
    return {
        'seed': 3,
        'train_cfgs': {'device': 'cuda', 'vector_env_nums': N, 'total_steps': N * T * epochs, 'parallel': 1},
        'algo_cfgs': {'steps_per_epoch': N * T, 'batch_size': 256, 'update_iters': 3, **algo},
        'logger_cfgs': {'log_dir': str(tmp), 'save_model_freq': 1, 'window_lens': 100, 'use_tensorboard': False},
        'env_cfgs': {'obs_dim': 45, 'act_dim': 3, 'max_episode_steps': 7},
    }


@pytest.mark.parametrize('algo', ['PPOLag', 'CPO', 'FOCOPS'])
def test_agent_learns_on_registered_env(cuda, tmp_path, algo):
    import omnisafe_b200
    from omnisafe_b200.common.normalizer import Normalizer

    agent = omnisafe_b200.Agent(algo, xe.WIDE_BOX_ID, custom_cfgs=_custom(tmp_path))
    ep_ret, ep_cost, ep_len = agent.learn()
    assert np.isfinite([ep_ret, ep_cost, ep_len]).all() and 1 <= ep_len <= 7
    log_dir = agent.agent.logger.log_dir
    rows = open(os.path.join(log_dir, 'progress.csv')).read().strip().splitlines()
    assert len(rows) == 1 + 2
    vals = [float(v) for v in rows[-1].split(',') if v not in ('', 'nan')]
    assert np.isfinite(vals).all()
    ckpt = torch.load(os.path.join(log_dir, 'torch_save', 'epoch-2.pt'), weights_only=False)
    assert ckpt['pi']['mean.0.weight'].shape == (64, 45)
    assert set(ckpt['obs_normalizer']) == {'_mean', '_sumsq', '_var', '_std', '_count', '_clip'}
    nz = Normalizer((45,), device=cuda)
    nz.load_state_dict(ckpt['obs_normalizer'])
    np.testing.assert_allclose(nz.mean.cpu().numpy(), agent.agent._env._obs_normalizer.mean.cpu().numpy())
    assert float(nz.mean.abs().max()) > 10.0              # the raw observations reach ~1e3
    actor = torch.nn.Module()                             # the reference GaussianLearningActor's parameter layout
    actor.mean = torch.nn.Sequential(torch.nn.Linear(45, 64), torch.nn.Tanh(), torch.nn.Linear(64, 64), torch.nn.Tanh(),
                                     torch.nn.Linear(64, 3))
    actor.log_std = torch.nn.Parameter(torch.zeros(3))
    actor.load_state_dict(ckpt['pi'])
    assert torch.isfinite(actor.mean(torch.randn(4, 45))).all()


def test_philox_fast_mode_deterministic(cuda):
    O, A, N, T = 45, 3, 256, 16
    theta = oac.init_theta(O, A, seed=1)
    _, _, o1 = _ext_rollout(cuda, xe.WIDE_BOX_ID, N, T, O, A, 4, theta, None, 2, epochs=2)
    _, _, o2 = _ext_rollout(cuda, xe.WIDE_BOX_ID, N, T, O, A, 4, theta, None, 2, epochs=2)
    for e in range(2):
        assert np.array_equal(o1[e]['act'], o2[e]['act']) and np.array_equal(o1[e]['obs'], o2[e]['obs'])
    assert not np.array_equal(o1[0]['act'], o1[1]['act'])


def test_nan_observation_raises_at_epoch_end(cuda):
    from omnisafe_b200._lib import OsbError
    from omnisafe_b200.adapter.external_adapter import ExternalEnvAdapter
    from omnisafe_b200.common.buffer import VectorOnPolicyBuffer
    from omnisafe_b200.models import ConstraintActorCritic

    O, A, N, T = 45, 3, 32, 8
    ad = ExternalEnvAdapter(xe.WIDE_BOX_ID, N, 1, _cfgs(obs_dim=O, act_dim=A), device=cuda)
    agent = ConstraintActorCritic(O, A, _model_cfgs(), epochs=1, device=cuda)
    agent.load_flat(oac.init_theta(O, A, seed=2))
    buf = VectorOnPolicyBuffer(O, A, T, 0.99, 0.95, 0.95, 'gae', 0.0, True, True, num_envs=N, device=cuda)
    step, calls = ad.env.step, []

    def bad_step(action):
        out = list(step(action))
        calls.append(1)
        if len(calls) == 3:
            out[0] = out[0].clone()
            out[0][5, 7] = float('nan')
        return tuple(out)

    ad.env.step = bad_step
    with pytest.raises(OsbError, match='non-finite observation'):
        ad.rollout(T, agent, buf)
    assert len(calls) == T                  # raised once, at the end of the epoch


def test_saute_family_refuses_external_env(cuda, tmp_path):
    import omnisafe_b200

    for algo in ('PPOSaute', 'PPOSimmerPID', 'PPOEarlyTerminated'):
        cfg = _custom(tmp_path)
        with pytest.raises(NotImplementedError):
            omnisafe_b200.Agent(algo, xe.WIDE_BOX_ID, custom_cfgs=cfg)
