"""GPU parity: fused rollout-step kernel (env + ObsNormalize + 3 MLP forwards + sample + append)
vs the oracle and vs the golden fixture produced by the unmodified reference."""
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from oracle import actor_critic as oac
from oracle import rollout as orollout
from oracle.normalizer import Normalizer as ONormalizer
from oracle.synthetic_env import SyntheticBoxEnv as OEnv

pytestmark = pytest.mark.gpu


def _cfgs(obs_normalize=True, window=100, rc_normalize=False, **env_cfgs):
    return NS(algo_cfgs=NS(obs_normalize=obs_normalize, reward_normalize=rc_normalize, cost_normalize=rc_normalize),
              logger_cfgs=NS(window_lens=window), env_cfgs=env_cfgs)


def _model_cfgs():
    net = NS(hidden_sizes=[64, 64], activation='tanh', lr=3e-4)
    return NS(actor=net, critic=net, actor_type='gaussian_learning', linear_lr_decay=True,
              weight_initialization_mode='kaiming_uniform')


def _gpu_rollout(dev, N, T, O, A, seed, theta, eps, tmax, term_prob, obs_normalize=True, window=100, epochs=1,
                 rc_normalize=False, precision=0):
    from omnisafe_b200.adapter.onpolicy_adapter import OnPolicyAdapter
    from omnisafe_b200.common.buffer import VectorOnPolicyBuffer
    from omnisafe_b200.models import ConstraintActorCritic

    cfgs = _cfgs(obs_normalize, window, rc_normalize, obs_dim=O, act_dim=A, max_episode_steps=tmax, term_prob=term_prob)
    ad = OnPolicyAdapter('SyntheticBox-v0', N, seed, cfgs, device=dev)
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


def _compare(sl_gpu, sl_ref, tol=2e-5):
    t = dict(rtol=tol, atol=tol)
    np.testing.assert_allclose(sl_gpu['obs'], sl_ref['obs'], **t)
    np.testing.assert_allclose(sl_gpu['act'], sl_ref['act'], **t)      # identical eps -> same actions
    np.testing.assert_allclose(sl_gpu['reward'], sl_ref['rew'], **t)
    assert (sl_gpu['cost'] != sl_ref['cost']).mean() < 1e-3
    np.testing.assert_allclose(sl_gpu['value_r'], sl_ref['val_r'], **t)
    np.testing.assert_allclose(sl_gpu['value_c'], sl_ref['val_c'], **t)
    np.testing.assert_allclose(sl_gpu['logp'], sl_ref['logp'], rtol=tol, atol=5e-5)
    assert np.array_equal(sl_gpu['flags'], sl_ref['flags'])
    ends = (sl_ref['flags'] != 0)
    ends[-1, :] = True
    need = ends & ((sl_ref['flags'] & 1) == 0)
    np.testing.assert_allclose(sl_gpu['boot_r'][need], sl_ref['boot_r'][need], **t)
    np.testing.assert_allclose(sl_gpu['boot_c'][need], sl_ref['boot_c'][need], **t)


@pytest.mark.parametrize('precision', [0, 2])      # exact fp32 FMA tiles / split-bf16 tensor-core tiles: same bar
def test_rollout_golden_reference(cuda, golden_dir, precision):
    """Same seed / params / noise as the unmodified reference run -> same slabs."""
    g = np.load(os.path.join(golden_dir, 'rollout_ppolag.npz'))
    N, T, O, A = int(g['N']), int(g['T']), int(g['O']), int(g['A'])
    ad, buf, outs = _gpu_rollout(cuda, N, T, O, A, int(g['seed']), g['theta'], g['eps'][None],
                                 int(g['tmax']), float(g['term_prob']), window=10, precision=precision)
    sl = outs[0]
    t = dict(rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(sl['obs'], g['slab_obs'], **t)
    np.testing.assert_allclose(sl['act'], g['slab_act'], **t)
    np.testing.assert_allclose(sl['reward'], g['slab_reward'], **t)
    assert np.array_equal(sl['cost'], g['slab_cost'])
    np.testing.assert_allclose(sl['value_r'], g['slab_value_r'], **t)
    np.testing.assert_allclose(sl['logp'], g['slab_logp'], rtol=2e-5, atol=5e-5)
    nz = ad._obs_normalizer
    np.testing.assert_allclose(nz.mean.cpu().numpy(), g['norm_mean'], **t)
    np.testing.assert_allclose(nz.std.cpu().numpy(), g['norm_std'], **t)
    assert int(nz.count[0]) == int(g['norm_count'])
    buf.finish_paths()
    torch.cuda.synchronize()
    np.testing.assert_allclose(buf.data['adv_r'].cpu().numpy(), g['slab_adv_r'], rtol=1e-4, atol=5e-5)
    np.testing.assert_allclose(buf.data['adv_c'].cpu().numpy(), g['slab_adv_c'], rtol=1e-4, atol=5e-5)
    np.testing.assert_allclose(buf.data['target_value_r'].cpu().numpy(), g['slab_target_value_r'], rtol=1e-4, atol=5e-5)
    # Logger window (deque maxlen 10) of finished episodes
    meta = ad.ep_meta.cpu().numpy()
    ring = ad.ep_ring.cpu().numpy()
    cnt, head = int(meta[0]), int(meta[1])
    assert cnt == len(g['win_ret'])
    order = [(head - cnt + i) % 10 for i in range(cnt)]
    np.testing.assert_allclose(ring[0][order], g['win_ret'], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(ring[1][order], g['win_cost'])
    np.testing.assert_allclose(ring[2][order], g['win_len'])
    ws = ad.window_sums.cpu().numpy()
    np.testing.assert_allclose(ws[1] / ws[3], g['win_cost'].mean(), rtol=1e-6)


def test_rollout_reward_cost_normalize_golden(cuda, golden_dir):
    """RewardNormalize / CostNormalize (wrapper.py:L280-423) as the slab post-pass vs two epochs of the
    unmodified reference with PDO's defaults (normalisers on); then GAE on the normalised slabs."""
    g = np.load(os.path.join(golden_dir, 'rollout_pdo.npz'))
    N, T, O, A, E = int(g['N']), int(g['T']), int(g['O']), int(g['A']), int(g['epochs_rolled'])
    ad, buf, outs = _gpu_rollout(cuda, N, T, O, A, int(g['seed']), g['theta'], g['eps'].reshape(E, T, N, A),
                                 int(g['tmax']), float(g['term_prob']), window=10, epochs=E, rc_normalize=True)
    sl = outs[-1]
    t = dict(rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(sl['obs'], g['slab_obs'], **t)
    np.testing.assert_allclose(sl['reward'], g['slab_reward'], rtol=5e-5, atol=5e-5)
    np.testing.assert_allclose(sl['cost'], g['slab_cost'], rtol=5e-5, atol=5e-5)
    rn, cn = ad.save()['reward_normalizer'], ad.save()['cost_normalizer']
    np.testing.assert_allclose([float(rn.mean), float(rn.std), float(cn.mean), float(cn.std)],
                               [g['rnorm_mean'], g['rnorm_std'], g['cnorm_mean'], g['cnorm_std']], rtol=2e-5)
    assert int(rn.count[0]) == int(g['rnorm_count']) and int(cn.count[0]) == int(g['cnorm_count'])
    assert set(rn.state_dict()) == {'_mean', '_sumsq', '_var', '_std', '_count', '_clip'}
    buf.finish_paths()
    torch.cuda.synchronize()
    np.testing.assert_allclose(buf.data['adv_r'].cpu().numpy(), g['slab_adv_r'], rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(buf.data['adv_c'].cpu().numpy(), g['slab_adv_c'], rtol=1e-4, atol=1e-4)
    # episode statistics stay raw (info['original_reward'], onpolicy_adapter.py:L141-146)
    meta, ring = ad.ep_meta.cpu().numpy(), ad.ep_ring.cpu().numpy()
    cnt, head = int(meta[0]), int(meta[1])
    order = [(head - cnt + i) % 10 for i in range(cnt)]
    np.testing.assert_allclose(ring[0][order], g['win_ret'], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(ring[1][order], g['win_cost'])


def test_scalar_normalizer_large_rows(cuda):
    """Slab post-pass vs the oracle Normalizer(()) at a headline-sized row (N = 4096) over several epochs."""
    from omnisafe_b200.common.normalizer import ScalarNormalizer
    from oracle.normalizer import Normalizer as ONorm
    from oracle.rollout import normalize_rows

    rng = np.random.default_rng(4)
    sn, on = ScalarNormalizer(5.0, cuda), ONorm(())
    for e in range(3):
        x = (rng.standard_normal((16, 4096)) * (1 + e) + 0.3 * e).astype(np.float32)
        want = normalize_rows(on, x)
        got = torch.as_tensor(x).to(cuda)
        sn.normalize_rows_(got)
        np.testing.assert_allclose(got.cpu().numpy(), want, rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose([float(sn.mean), float(sn.std)], [on.mean, on.std], rtol=1e-5)
    assert int(sn.count[0]) == on.count
    one = ScalarNormalizer(5.0, cuda)      # N == 1: count <= 1 after the first push -> passthrough
    y = torch.tensor([[2.0], [4.0], [9.0]], device=cuda)
    o1 = ONorm(())
    want = normalize_rows(o1, np.array([[2.0], [4.0], [9.0]], np.float32))
    one.normalize_rows_(y)
    np.testing.assert_allclose(y.cpu().numpy(), want, rtol=1e-6)


@pytest.mark.parametrize('N,T,O,A,tmax,term_prob,norm', [
    (64, 40, 60, 8, 16, 0.0, True),
    (50, 33, 60, 8, 7, 0.05, True),       # ragged tile (N % 32 != 0), terminations + truncations
    (32, 20, 17, 6, 5, 0.1, False),       # no ObsNormalize
    (40, 12, 111, 8, 6, 0.03, True),      # obs dim > 64: two layer-1 chunks
    (33, 6, 376, 8, 3, 0.0, True),        # Humanoid-like obs dim: six chunks
])
def test_rollout_vs_oracle(cuda, N, T, O, A, tmax, term_prob, norm):
    rng = np.random.default_rng(N * 7 + T)
    theta = oac.init_theta(O, A, seed=3)
    epochs = 2
    eps = rng.standard_normal((epochs, T, N, A)).astype(np.float32)
    ad, buf, outs = _gpu_rollout(cuda, N, T, O, A, 9, theta, eps, tmax, term_prob, obs_normalize=norm,
                                 window=16, epochs=epochs)
    env = OEnv(N, O, A, max_episode_steps=tmax, seed=9, term_prob=term_prob)
    onorm = ONormalizer((O,))
    window = []
    for e in range(epochs):   # state (normaliser, episode counters, window) carries across epochs
        ref = orollout.rollout_epoch(env, onorm, theta, T, eps[e], obs_normalize=norm, window=window)
        _compare(outs[e], ref)
    w = np.array(window[-16:], np.float32)
    meta = ad.ep_meta.cpu().numpy(); ring = ad.ep_ring.cpu().numpy()
    cnt, head = int(meta[0]), int(meta[1])
    assert cnt == len(w)
    order = [(head - cnt + i) % 16 for i in range(cnt)]
    np.testing.assert_allclose(ring[0][order], w[:, 0], rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(ring[1][order], w[:, 1])
    np.testing.assert_allclose(ring[2][order], w[:, 2])


def test_rollout_philox_fast_mode(cuda):
    """Fast mode (in-kernel Philox noise): actions are mu + sigma*eps with eps ~ N(0,1) and the
    stored log-prob is consistent with the stored action; deterministic under a fixed seed."""
    N, T, O, A = 4096, 8, 60, 8
    theta = oac.init_theta(O, A, seed=1)
    _, _, o1 = _gpu_rollout(cuda, N, T, O, A, 4, theta, None, 64, 0.0)
    _, _, o2 = _gpu_rollout(cuda, N, T, O, A, 4, theta, None, 64, 0.0)
    assert np.array_equal(o1[0]['act'], o2[0]['act'])
    sl = o1[0]
    nets = oac.unflatten(torch.as_tensor(theta), O, A)
    obs = torch.as_tensor(sl['obs'])
    with torch.no_grad():
        dist = oac.actor_dist(nets['actor'], obs)
        z = ((torch.as_tensor(sl['act']) - dist.loc) / dist.scale).numpy()
        logp = dist.log_prob(torch.as_tensor(sl['act'])).sum(-1).numpy()
    np.testing.assert_allclose(sl['logp'], logp, rtol=1e-4, atol=1e-3)
    assert abs(z.mean()) < 0.01 and abs(z.std() - 1.0) < 0.01
    assert abs(np.corrcoef(z[0, :, 0], z[1, :, 0])[0, 1]) < 0.05


@pytest.mark.timeout(180)
@pytest.mark.parametrize('N,T,tmax,term_prob', [(256, 24, 8, 0.0), (200, 20, 6, 0.05)])
def test_rollout_tensor_core_mode(cuda, N, T, tmax, term_prob):
    """matmul_precision = tf32 (wgmma tiles of 128 envs): same trajectory as the oracle up to the
    TF32 rounding of the three layer GEMMs (tolerance 5e-3 on values / actions, stated here); the
    env / normaliser / bookkeeping arithmetic is unchanged."""
    from omnisafe_b200.adapter.onpolicy_adapter import OnPolicyAdapter
    from omnisafe_b200.common.buffer import VectorOnPolicyBuffer
    from omnisafe_b200.models import ConstraintActorCritic

    O, A = 60, 8
    rng = np.random.default_rng(N + T)
    theta = oac.init_theta(O, A, seed=3)
    eps = rng.standard_normal((T, N, A)).astype(np.float32)
    cfgs = _cfgs(True, 16, obs_dim=O, act_dim=A, max_episode_steps=tmax, term_prob=term_prob)
    ad = OnPolicyAdapter('SyntheticBox-v0', N, 9, cfgs, device=cuda)
    ad.precision = 1
    agent = ConstraintActorCritic(O, A, _model_cfgs(), epochs=1, device=cuda)
    agent.load_flat(theta)
    buf = VectorOnPolicyBuffer(O, A, T, 0.99, 0.95, 0.95, 'gae', 0.0, True, True, num_envs=N, device=cuda)
    ad.rollout(T, agent, buf, eps=torch.as_tensor(eps).to(cuda))
    torch.cuda.synchronize()
    sl = {k: v.cpu().numpy() for k, v in buf.data.items() if v is not None}
    ref = orollout.rollout_epoch(OEnv(N, O, A, max_episode_steps=tmax, seed=9, term_prob=term_prob),
                                 ONormalizer((O,)), theta, T, eps)
    assert np.array_equal(sl['flags'], ref['flags'])
    tol = dict(rtol=5e-3, atol=5e-3)
    np.testing.assert_allclose(sl['obs'], ref['obs'], **tol)
    np.testing.assert_allclose(sl['act'], ref['act'], **tol)
    np.testing.assert_allclose(sl['value_r'], ref['val_r'], **tol)
    np.testing.assert_allclose(sl['value_c'], ref['val_c'], **tol)
    np.testing.assert_allclose(sl['reward'], ref['rew'], **tol)
    np.testing.assert_allclose(sl['logp'], ref['logp'], rtol=5e-3, atol=2e-2)
    assert (sl['cost'] != ref['cost']).mean() < 5e-3
    need = ((ref['flags'] != 0) | (np.arange(T)[:, None] == T - 1)) & ((ref['flags'] & 1) == 0)
    np.testing.assert_allclose(sl['boot_r'][need], ref['boot_r'][need], **tol)


@pytest.mark.timeout(600)
@pytest.mark.parametrize('N,T,tmax,term_prob,precision', [(256, 24, 8, 0.0, 2), (200, 20, 6, 0.05, 2), (100, 33, 7, 0.02, 2),
                                                          (4096, 128, 64, 0.0, 0), (4096, 128, 64, 0.0, 2),
                                                          (6000, 8, 6, 0.02, 2)])
def test_rollout_vs_oracle_bf16x3_and_headline(cuda, N, T, tmax, term_prob, precision):
    """matmul_precision = bf16x3 (bf16 wgmma, three bf16 pieces per fp32 operand) is held to the bar of the exact
    fp32 tiles -- 2e-5 on every slab vs the oracle (the tf32 tiles get 5e-3) -- and both modes are checked at the headline
    size of the bench workload (4096 envs x 128 steps, obs 60 / act 8).  N = 6000 is more CTAs (tiles x 3 networks) than
    the GPU has SMs, so the epoch runs as one tensor-core launch per step instead of the persistent kernel."""
    if N > 4096:
        assert -(-N // 128) * 3 > torch.cuda.get_device_properties(cuda).multi_processor_count
    O, A = 60, 8
    rng = np.random.default_rng(N + T)
    theta = oac.init_theta(O, A, seed=3)
    eps = rng.standard_normal((1, T, N, A)).astype(np.float32)
    ad, buf, outs = _gpu_rollout(cuda, N, T, O, A, 9, theta, eps, tmax, term_prob, window=16, precision=precision)
    ref = orollout.rollout_epoch(OEnv(N, O, A, max_episode_steps=tmax, seed=9, term_prob=term_prob),
                                 ONormalizer((O,)), theta, T, eps[0])
    _compare(outs[0], ref, tol=2e-5)
