"""GPU end-to-end: the omnisafe-style Agent entry point, full training epochs, CPO update parity with
the unmodified reference (golden), checkpoint format."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
# the class goldens run on the exact fp32 tiles and on the split-bf16 tiles (the SyntheticBox-v0 default), same bars
PRECISIONS = ['fp32', 'bf16x3']


def _custom(tmp, N=64, T=32, epochs=3, **algo):
    return {
        'seed': 3,
        'train_cfgs': {'device': 'cuda', 'vector_env_nums': N, 'total_steps': N * T * epochs, 'parallel': 1},
        'algo_cfgs': {'steps_per_epoch': N * T, 'batch_size': 256, 'update_iters': 3, **algo},
        'logger_cfgs': {'log_dir': str(tmp), 'save_model_freq': 2, 'window_lens': 100, 'use_tensorboard': False},
        'env_cfgs': {'obs_dim': 60, 'act_dim': 8, 'max_episode_steps': 16},
    }


@pytest.mark.parametrize('algo', ['PPOLag', 'TRPOLag', 'CPO', 'FOCOPS', 'PPO', 'TRPO', 'RCPO', 'NaturalPG', 'PolicyGradient',
                                  'PCPO', 'CPPOPID', 'TRPOPID', 'OnCRPO', 'PDO', 'IPO', 'P3O'])
def test_agent_trains_and_logs(cuda, tmp_path, algo):
    import omnisafe_b200

    agent = omnisafe_b200.Agent(algo, 'SyntheticBox-v0', custom_cfgs=_custom(tmp_path))
    ep_ret, ep_cost, ep_len = agent.learn()
    assert np.isfinite([ep_ret, ep_cost, ep_len]).all() and ep_len == 16
    log_dir = agent.agent.logger.log_dir
    rows = open(os.path.join(log_dir, 'progress.csv')).read().strip().splitlines()
    assert len(rows) == 1 + 3 and 'Time/FPS' in rows[0] and 'Metrics/EpCost' in rows[0]
    assert os.path.exists(os.path.join(log_dir, 'config.json'))
    ckpt = torch.load(os.path.join(log_dir, 'torch_save', 'epoch-3.pt'), weights_only=False)
    # reference checkpoint format: {'pi': actor.state_dict(), 'obs_normalizer': Normalizer.state_dict()}
    assert set(ckpt['pi']) == {'log_std', 'mean.0.weight', 'mean.0.bias', 'mean.2.weight', 'mean.2.bias',
                               'mean.4.weight', 'mean.4.bias'}
    assert ckpt['pi']['mean.0.weight'].shape == (64, 60)
    assert set(ckpt['obs_normalizer']) == {'_mean', '_sumsq', '_var', '_std', '_count', '_clip'}
    theta = agent.agent._actor_critic.theta
    assert torch.isfinite(theta).all()


def test_ppolag_learning_signal(cuda, tmp_path):
    """A few epochs of PPO-Lag on the synthetic env must raise the return (sanity of the whole
    rollout -> GAE -> update loop, not a parity claim)."""
    import omnisafe_b200

    cfg = _custom(tmp_path, N=256, T=64, epochs=12)
    cfg['algo_cfgs'].update({'update_iters': 8, 'batch_size': 2048})
    cfg['model_cfgs'] = {'actor': {'lr': 1e-3}, 'critic': {'lr': 1e-3}}
    agent = omnisafe_b200.Agent('PPOLag', 'SyntheticBox-v0', custom_cfgs=cfg)
    agent.learn()
    rows = open(os.path.join(agent.agent.logger.log_dir, 'progress.csv')).read().strip().splitlines()
    hdr = rows[0].split(',')
    ret = [float(r.split(',')[hdr.index('Metrics/EpRet')]) for r in rows[1:]]
    print('EpRet per epoch:', ret)
    assert ret[-1] > ret[0] + 0.05, ret


@pytest.mark.parametrize('name,fname', [('CPO', 'update_cpo.npz'), ('PCPO', 'update_pcpo.npz')])
@pytest.mark.parametrize('prec', PRECISIONS)
def test_cpo_update_golden(cuda, tmp_path, golden_dir, name, fname, prec):
    """CPO._update / PCPO._update of the unmodified reference vs ours on identical data: same case
    analysis, same step, same parameters afterwards, on the fp32 and the split-bf16 tiles."""
    import omnisafe_b200

    g = np.load(os.path.join(golden_dir, fname))
    N, T, O, A = int(g['N']), int(g['T']), int(g['O']), int(g['A'])
    cfg = {
        'seed': int(g['seed']) if 'seed' in g.files else 7,
        'train_cfgs': {'device': 'cuda', 'vector_env_nums': N, 'total_steps': N * T * 2, 'matmul_precision': prec},
        'algo_cfgs': {'steps_per_epoch': N * T, 'batch_size': 32, 'update_iters': 2, 'cost_limit': float(g['cost_limit'])},
        'logger_cfgs': {'log_dir': str(tmp_path), 'window_lens': 10, 'use_tensorboard': False},
        'env_cfgs': {'obs_dim': O, 'act_dim': A, 'max_episode_steps': 8, 'term_prob': 0.05},
    }
    algo = omnisafe_b200.Agent(name, 'SyntheticBox-v0', custom_cfgs=cfg).agent
    assert algo._engine.precision == {'fp32': 0, 'bf16x3': 2}[prec]
    algo._actor_critic.load_flat(g['theta0'])
    data = {k[5:]: g[k] for k in g.files if k.startswith('data_')}

    def tm(x):
        x = np.asarray(x, np.float32)
        return torch.as_tensor(x.reshape(N, T, *x.shape[1:]).swapaxes(0, 1).copy()).to(cuda)

    for k in ('obs', 'act', 'logp', 'adv_r', 'adv_c', 'target_value_r', 'target_value_c'):
        algo._buf.data[k].copy_(tm(data[k]))
    algo._buf.adv_moments.copy_(torch.tensor([0.0, 1.0, 0.0, 1.0]))
    algo._env.window_sums.copy_(torch.tensor([0.0, float(g['ep_cost']) * 10, 0.0, 10.0], dtype=torch.float64))
    rows = lambda k: ((k % T) * N + (k // T)).astype(np.int32)   # noqa: E731
    perms = torch.as_tensor(np.stack([rows(p.astype(np.int64)) for p in g['perms'][::2]])).to(cuda)
    algo._update(perm=perms)
    torch.cuda.synchronize()
    m = algo._misc
    assert int(m['Misc/OptimCase']) == int(g['misc_OptimCase'][-1])
    assert int(m['Misc/AcceptanceStep']) == int(g['misc_AcceptanceStep'][-1])
    for key in ('xHx', 'q', 'r', 's', 'A', 'B', 'Nu_star', 'Lambda_star', 'Alpha', 'gradient_norm',
                'cost_gradient_norm', 'H_inv_g', 'FinalStepNorm'):
        np.testing.assert_allclose(m[f'Misc/{key}'], g[f'misc_{key}'][-1], rtol=5e-3, atol=1e-5, err_msg=key)
    np.testing.assert_allclose(float(algo._engine.kl_state[0]), g['kl'][-1], rtol=5e-3, atol=1e-6)
    got, want = algo._actor_critic.theta.cpu().numpy(), g['theta1']
    # Adam normalises every step to ~lr, so a parameter whose gradient is at rounding level can differ
    # by a few lr (1e-3) between two correct fp32 implementations: allow < 0.1 % such elements.
    bad = ~np.isclose(got, want, rtol=2e-3, atol=2e-5)
    assert bad.mean() < 1e-3 and np.abs(got - want).max() < 5e-3, (bad.sum(), np.abs(got - want).max())


def test_pid_lagrange_kernel_golden(cuda, golden_dir):
    """osb_pid_lagrange_update vs the reference PIDLagrangian over the recorded cost sequences: the
    fp64 penalty bit-for-bit, the fp32 multiplier the kernels read = its rounding."""
    from omnisafe_b200.common.pid_lagrange import PIDLagrangian

    g = np.load(os.path.join(golden_dir, 'pid_lagrange.npz'))
    keys = ('pid_kp', 'pid_ki', 'pid_kd', 'pid_d_delay', 'pid_delta_p_ema_alpha', 'pid_delta_d_ema_alpha',
            'sum_norm', 'diff_norm', 'penalty_max', 'lagrangian_multiplier_init', 'cost_limit')
    for i in range(int(g['n_cfgs'])):
        pid = PIDLagrangian(**{k: g[f'cfg_{i}_{k}'].item() for k in keys}, device=cuda)
        pens, lams = [], []
        for c in g['costs']:
            ws = torch.tensor([0.0, float(c) * 8.0, 0.0, 8.0], dtype=torch.float64, device=cuda)
            pid.pid_update(ws)
            pens.append(pid.pid_state[3].clone())
            lams.append(pid.state[0].clone())
        pens = torch.stack(pens).cpu().numpy()
        lams = torch.stack(lams).cpu().numpy()
        np.testing.assert_array_equal(pens, g[f'lam_{i}'])
        np.testing.assert_array_equal(lams, g[f'lam_{i}'].astype(np.float32))
        assert int(pid.nan_flag) == 0
    empty = torch.zeros(4, dtype=torch.float64, device=cuda)
    pid.pid_update(empty)
    assert int(pid.nan_flag) == 1


@pytest.mark.parametrize('fname', ['update_trpolag.npz', 'update_oncrpo.npz', 'update_rcpo.npz'])
@pytest.mark.parametrize('prec', PRECISIONS)
def test_trpo_family_update_golden(cuda, tmp_path, golden_dir, fname, prec):
    """TRPOLag._update / OnCRPO._update (cost-surrogate branch) / RCPO._update (plain natural step) of the
    unmodified reference vs ours on identical data: same natural direction, same accepted line-search step,
    same parameters afterwards."""
    import omnisafe_b200

    g = np.load(os.path.join(golden_dir, fname))
    name = str(g['name'])
    N, T, O, A = int(g['N']), int(g['T']), int(g['O']), int(g['A'])
    extra = {k[6:]: float(g[k]) for k in g.files if k.startswith('extra_')}
    cfg = {
        'seed': int(g['seed']),
        'train_cfgs': {'device': 'cuda', 'vector_env_nums': N, 'total_steps': N * T * 2, 'matmul_precision': prec},
        'algo_cfgs': {'steps_per_epoch': N * T, 'batch_size': 32, 'update_iters': 2, **extra},
        'logger_cfgs': {'log_dir': str(tmp_path), 'window_lens': 10, 'use_tensorboard': False},
        'env_cfgs': {'obs_dim': O, 'act_dim': A, 'max_episode_steps': 8, 'term_prob': 0.05},
    }
    lag = {k[9:]: float(g[k]) for k in g.files if k.startswith('lagrange_')}
    if lag:
        cfg['lagrange_cfgs'] = lag
    algo = omnisafe_b200.Agent(name, 'SyntheticBox-v0', custom_cfgs=cfg).agent
    assert algo._engine.precision == {'fp32': 0, 'bf16x3': 2}[prec]
    algo._actor_critic.load_flat(g['theta0'])
    data = {k[5:]: g[k] for k in g.files if k.startswith('data_')}

    def tm(x):
        x = np.asarray(x, np.float32)
        return torch.as_tensor(x.reshape(N, T, *x.shape[1:]).swapaxes(0, 1).copy()).to(cuda)

    for k in ('obs', 'act', 'logp', 'adv_r', 'adv_c', 'target_value_r', 'target_value_c'):
        algo._buf.data[k].copy_(tm(data[k]))
    algo._buf.adv_moments.copy_(torch.tensor([0.0, 1.0, 0.0, 1.0]))
    algo._env.window_sums.copy_(torch.tensor([0.0, float(g['ep_cost']) * 10, 0.0, 10.0], dtype=torch.float64))
    rows = lambda k: ((k % T) * N + (k // T)).astype(np.int32)   # noqa: E731
    perms = torch.as_tensor(np.stack([rows(p.astype(np.int64)) for p in g['perms'][::2]])).to(cuda)
    algo._update(perm=perms)
    torch.cuda.synchronize()
    m = algo._misc
    for key in ('xHx', 'Alpha', 'gradient_norm', 'H_inv_g', 'FinalStepNorm'):
        np.testing.assert_allclose(m[f'Misc/{key}'], g[f'misc_{key}'][-1], rtol=5e-3, atol=1e-5, err_msg=key)
    if name != 'RCPO':      # the NaturalPG family takes the natural step as is: no acceptance step, no KL logged
        assert int(m['Misc/AcceptanceStep']) == int(g['misc_AcceptanceStep'][-1])
        np.testing.assert_allclose(float(algo._engine.kl_state[0]), g['kl'][-1], rtol=5e-3, atol=1e-6)
    if hasattr(algo, '_lagrange'):
        np.testing.assert_allclose(float(algo._lagrange.lagrangian_multiplier), float(g['lam1']), rtol=1e-4, atol=1e-6)
    got, want = algo._actor_critic.theta.cpu().numpy(), g['theta1']
    bad = ~np.isclose(got, want, rtol=2e-3, atol=2e-5)
    assert bad.mean() < 1e-3 and np.abs(got - want).max() < 5e-3, (bad.sum(), np.abs(got - want).max())


@pytest.mark.parametrize('fname', ['update_ipo.npz', 'update_cppopid.npz', 'update_pdo.npz'])
@pytest.mark.parametrize('prec', PRECISIONS)
def test_first_order_family_update_golden(cuda, tmp_path, golden_dir, fname, prec):
    """IPO._update / CPPOPID._update / PDO._update of the unmodified reference vs ours on identical data:
    the class derives the same penalty / multiplier from Jc and the fused update lands on the same parameters."""
    import omnisafe_b200

    g = np.load(os.path.join(golden_dir, fname))
    name = str(g['name'])
    N, T, O, A = int(g['N']), int(g['T']), int(g['O']), int(g['A'])
    cfg = {
        'seed': int(g['seed']),
        'train_cfgs': {'device': 'cuda', 'vector_env_nums': N, 'total_steps': N * T * 2, 'matmul_precision': prec},
        'algo_cfgs': {'steps_per_epoch': N * T, 'batch_size': 32, 'update_iters': 2,
                      **{k[6:]: float(g[k]) for k in g.files if k.startswith('extra_')}},
        'logger_cfgs': {'log_dir': str(tmp_path), 'window_lens': 10, 'use_tensorboard': False},
        'env_cfgs': {'obs_dim': O, 'act_dim': A, 'max_episode_steps': 8, 'term_prob': 0.05},
    }
    lag = {k[9:]: float(g[k]) for k in g.files if k.startswith('lagrange_')}
    if lag:
        cfg['lagrange_cfgs'] = lag
    algo = omnisafe_b200.Agent(name, 'SyntheticBox-v0', custom_cfgs=cfg).agent
    assert algo._engine.precision == {'fp32': 0, 'bf16x3': 2}[prec]
    algo._actor_critic.load_flat(g['theta0'])
    data = {k[5:]: g[k] for k in g.files if k.startswith('data_')}

    def tm(x):
        x = np.asarray(x, np.float32)
        return torch.as_tensor(x.reshape(N, T, *x.shape[1:]).swapaxes(0, 1).copy()).to(cuda)

    for k in ('obs', 'act', 'logp', 'adv_r', 'adv_c', 'target_value_r', 'target_value_c'):
        algo._buf.data[k].copy_(tm(data[k]))
    algo._buf.adv_moments.copy_(torch.tensor([0.0, 1.0, 0.0, 1.0]))
    algo._env.window_sums.copy_(torch.tensor([0.0, float(g['ep_cost']) * 10, 0.0, 10.0], dtype=torch.float64))
    rows = lambda k: ((k % T) * N + (k // T)).astype(np.int32)   # noqa: E731
    perms = torch.as_tensor(np.stack([rows(p.astype(np.int64)) for p in g['perms'][::2]])).to(cuda)
    algo._update(perm=perms)
    torch.cuda.synchronize()
    lam = algo._penalty if name == 'IPO' else float(algo._lagrange.lagrangian_multiplier)
    np.testing.assert_allclose(lam, float(g['lam1']), rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(float(algo._engine.kl_state[0]), g['kl'][-1], rtol=2e-3, atol=1e-6)
    got, want = algo._actor_critic.theta.cpu().numpy(), g['theta1']
    # Adam normalises every step to ~lr = 3e-4: parameters whose gradient sits at rounding level may differ by a
    # few lr between two correct fp32 implementations (12 steps here); allow < 0.5 % such elements, none beyond 2e-3
    bad = ~np.isclose(got, want, rtol=2e-4, atol=2e-6)
    assert bad.mean() < 5e-3 and np.abs(got - want).max() < 2e-3, (bad.sum(), np.abs(got - want).max())
