"""GPU: actor objectives written in PyTorch on the kernel update path.

- the supplied-dmu backward (osb_actor_dmu_backward) against float64 autograd of the actor MLP;
- a subclass whose hooks return super()'s reproduces the goldens of the unmodified reference (first-order and natural
  families), i.e. the PyTorch path and the fused path of the same class agree within the golden bars;
- objectives the kernels do not have, against a float64 restatement of PolicyGradient._update;
- whole runs through Agent (synthetic and registered env), evaluation and a bit-exact resume;
- a subclass that overrides nothing stays on the fused path, bit for bit.
"""
import math
import os

import numpy as np
import pytest
import torch
from torch.distributions import Normal
from torch.nn.utils.clip_grad import clip_grad_norm_

from oracle import actor_critic as oac

pytestmark = pytest.mark.gpu
PREC = {'fp32': 0, 'tf32': 1, 'bf16x3': 2}


def _subclass(base_name, *hooks):
    """A user subclass of a library class whose hooks return what super() returns."""
    from omnisafe_b200.algorithms import registry

    base = registry.get(base_name)
    body = {}
    if '_loss_pi' in hooks:
        body['_loss_pi'] = lambda self, obs, act, logp, adv: super(cls, self)._loss_pi(obs, act, logp, adv)
    if '_loss_pi_cost' in hooks:
        body['_loss_pi_cost'] = lambda self, obs, act, logp, adv_c: super(cls, self)._loss_pi_cost(obs, act, logp, adv_c)
    if '_compute_adv_surrogate' in hooks:
        body['_compute_adv_surrogate'] = lambda self, r, c: super(cls, self)._compute_adv_surrogate(r, c)
    cls = type(f'User{base_name}', (base,), body)
    return cls


def _agent(monkeypatch, tmp, name, cls, cfg, env_id='SyntheticBox-v0'):
    """omnisafe_b200.Agent(name, ...) building `cls` in place of the library class."""
    import omnisafe_b200
    from omnisafe_b200.algorithms import registry

    if cls is not None:
        monkeypatch.setitem(registry._classes, name, cls)
    return omnisafe_b200.Agent(name, env_id, custom_cfgs=cfg)


def _golden_cfg(tmp, g, prec, algo_extra=None, lagrange=None):
    N, T, O, A = int(g['N']), int(g['T']), int(g['O']), int(g['A'])
    cfg = {
        'seed': int(g['seed']) if 'seed' in g.files else 7,
        'train_cfgs': {'device': 'cuda', 'vector_env_nums': N, 'total_steps': N * T * 2, 'matmul_precision': prec},
        'algo_cfgs': {'steps_per_epoch': N * T, 'batch_size': int(g['batch_size']) if 'batch_size' in g.files else 32,
                      'update_iters': int(g['update_iters']) if 'update_iters' in g.files else 2, **(algo_extra or {})},
        'logger_cfgs': {'log_dir': str(tmp), 'window_lens': 10, 'use_tensorboard': False},
        'env_cfgs': {'obs_dim': O, 'act_dim': A, 'max_episode_steps': 8, 'term_prob': 0.05},
    }
    if lagrange:
        cfg['lagrange_cfgs'] = lagrange
    return cfg


def _load_golden_batch(algo, g, jc):
    N, T = int(g['N']), int(g['T'])
    data = {k[5:]: g[k] for k in g.files if k.startswith('data_')}

    def tm(x):
        x = np.asarray(x, np.float32)
        return torch.as_tensor(x.reshape(N, T, *x.shape[1:]).swapaxes(0, 1).copy()).cuda()

    algo._actor_critic.load_flat(g['theta0'])
    for k in ('obs', 'act', 'logp', 'adv_r', 'adv_c', 'target_value_r', 'target_value_c'):
        algo._buf.data[k].copy_(tm(data[k]))
    algo._buf.adv_moments.copy_(torch.tensor([0.0, 1.0, 0.0, 1.0]))
    algo._env.window_sums.copy_(torch.tensor([0.0, jc * 10, 0.0, 10.0], dtype=torch.float64))
    rows = lambda k: ((k % T) * N + (k // T)).astype(np.int32)   # noqa: E731
    return torch.as_tensor(np.stack([rows(p.astype(np.int64)) for p in g['perms'][::2]])).cuda()


def _assert_theta(got, want, prec, rtol, atol, frac, amax):
    if prec == 'tf32':      # the tf32 tiles' bar (test_update_tc_gpu.py): 5e-3-level arithmetic
        rtol, atol, frac, amax = 2e-2, 2e-3, 2e-2, 2e-2
    bad = ~np.isclose(got, want, rtol=rtol, atol=atol)
    assert bad.mean() < frac and np.abs(got - want).max() < amax, (bad.sum(), np.abs(got - want).max())


# ---- the supplied-dmu backward ---------------------------------------------------------------------------------------
@pytest.mark.parametrize('prec', list(PREC))
@pytest.mark.parametrize('O', [17, 64, 65, 376])
@pytest.mark.parametrize('A', [1, 8, 16])
def test_dmu_backward_vs_autograd(cuda, prec, O, A):
    from omnisafe_b200._lib import current_stream, lib, ptr

    rng = np.random.default_rng(O * 31 + A)
    B = 777
    theta = oac.init_theta(O, A, seed=O + A)
    Pa = oac.layout(O, A)['actor']['size']
    th = torch.as_tensor(theta[:Pa]).cuda()
    th[:A] = torch.as_tensor(rng.uniform(-0.5, 0.5, A).astype(np.float32)).cuda()
    obs = torch.as_tensor(rng.standard_normal((B, O)).astype(np.float32)).cuda()
    dmu = torch.as_tensor(rng.standard_normal((B, A)).astype(np.float32)).cuda()
    p = PREC[prec]
    nb = lib().osb_actor_dmu_grid_blocks(B, O, p)
    gpart = torch.zeros(nb * Pa, dtype=torch.float32, device=cuda)
    stats = torch.zeros(nb * 24, dtype=torch.float32, device=cuda)
    got = torch.zeros(Pa, dtype=torch.float32, device=cuda)
    lib().osb_actor_dmu_backward(ptr(th), O, A, ptr(obs), ptr(dmu), B, p, ptr(gpart), ptr(stats), current_stream())
    lib().osb_reduce_partials(ptr(gpart), nb, Pa, Pa, 1.0, 0, 0.0, ptr(got), current_stream())
    th64 = th.double().requires_grad_(True)
    params = oac.unflatten(torch.cat([th64, torch.zeros(oac.layout(O, A)['total'] - Pa, dtype=torch.float64,
                                                         device=cuda)]), O, A)['actor']
    (oac.mlp(params, obs.double()) * dmu.double()).sum().backward()
    want = th64.grad.cpu().numpy()
    got = got.cpu().numpy()
    assert np.all(got[:A] == 0.0)
    tol = 2e-2 if prec == 'tf32' else 2e-4
    scale = np.abs(want).max()
    np.testing.assert_allclose(got, want, rtol=tol, atol=tol * scale)


# ---- goldens of the unmodified reference through the PyTorch path -------------------------------------------------------
@pytest.mark.parametrize('prec', list(PREC))
@pytest.mark.parametrize('fname,name', [('update_ppolag.npz', 'PPOLag'), ('update_focops.npz', 'FOCOPS'),
                                        ('update_p3o.npz', 'P3O')])
def test_first_order_golden_through_torch_loss(cuda, tmp_path, golden_dir, monkeypatch, fname, name, prec):
    g = dict(np.load(os.path.join(golden_dir, fname)))
    if 'N' not in g:
        g.update(N=np.array(8), T=np.array(24), O=np.array(12), A=np.array(3))
    g = _NpzView(g)
    extra, lag, jc = {}, None, float(g['Jc'])
    if name in ('PPOLag', 'FOCOPS'):
        lag = {'cost_limit': float(g['cost_limit']), 'lagrangian_multiplier_init': float(g['lam0']),
               'lambda_lr': float(g['lambda_lr'])}
        if 'upper_bound' in g.files:
            lag['lagrangian_upper_bound'] = float(g['upper_bound'])
    if name == 'FOCOPS':
        extra = {'focops_lam': float(g['focops_lam']), 'focops_eta': float(g['focops_eta'])}
    if name == 'P3O':
        extra = {'kappa': float(g['kappa']), 'cost_limit': float(g['cost_limit'])}
    cfg = _golden_cfg(tmp_path, g, prec, extra, lag)
    algo = _agent(monkeypatch, tmp_path, name, _subclass(name, '_loss_pi'), cfg).agent
    assert algo._torch_hooks and algo._engine.precision == PREC[prec]
    perms = _load_golden_batch(algo, g, jc)
    algo._update(perm=perms)
    torch.cuda.synchronize()
    if lag:
        np.testing.assert_allclose(float(algo._lagrange.lagrangian_multiplier), float(g['lam1']), rtol=1e-4, atol=1e-6)
    kl_tol = 2e-2 if prec == 'tf32' else 2e-3
    np.testing.assert_allclose(float(algo._engine.kl_state[0]), g['kl'][-1], rtol=kl_tol, atol=1e-6)
    _assert_theta(algo._actor_critic.theta.cpu().numpy(), g['theta1'], prec, 2e-4, 2e-6, 1e-3, 2e-3)
    st = algo._loss_stats.means()
    np.testing.assert_allclose(st['Loss/Loss_pi'], g['loss_pi'].mean(), rtol=5e-2 if prec == 'tf32' else 2e-3,
                               atol=1e-5)
    if name == 'P3O':
        np.testing.assert_allclose(st['Loss/Loss_pi_cost'], g['loss_pi_cost'].mean(), rtol=2e-2, atol=1e-5)


class _NpzView(dict):
    @property
    def files(self):
        return list(self)


@pytest.mark.parametrize('prec', list(PREC))
def test_logged_loss_pi_kernel_equals_torch_loss(cuda, tmp_path, golden_dir, monkeypatch, prec):
    """Loss/Loss_pi of one PPOLag update at entropy_coef 0.01 and a trained log_std is the same on the kernel path and
    through super()._loss_pi: the per-minibatch loss after loss -= entropy_coef * entropy.mean() (base/ppo.py:L76-84)."""
    g = _NpzView(np.load(os.path.join(golden_dir, 'update_ppolag.npz')))
    g.update(N=np.array(8), T=np.array(24), O=np.array(12), A=np.array(3))
    theta0 = np.array(g['theta0'], np.float32)
    theta0[:3] = oac.trained_log_std(3)
    g['theta0'] = theta0
    lag = {'cost_limit': float(g['cost_limit']), 'lagrangian_multiplier_init': float(g['lam0']),
           'lambda_lr': float(g['lambda_lr'])}
    logged = []
    for tag, cls in (('kernel', None), ('torch', _subclass('PPOLag', '_loss_pi'))):
        cfg = _golden_cfg(tmp_path / tag, g, prec, {'entropy_coef': 0.01}, lag)
        algo = _agent(monkeypatch, tmp_path, 'PPOLag', cls, cfg).agent
        assert bool(algo._torch_hooks) == (cls is not None)
        perms = _load_golden_batch(algo, g, float(g['Jc']))
        algo._update(perm=perms)
        torch.cuda.synchronize()
        if cls is None:
            ts = algo._engine.train_stats.view(3, 8).tolist()
            logged.append((ts[0][0] + ts[0][4]) / ts[0][3])      # as the epoch log forms Loss/Loss_pi
        else:
            logged.append(float(algo._loss_stats.means()['Loss/Loss_pi']))
    print(f'[{prec}] Loss/Loss_pi kernel {logged[0]:.7f}, super()._loss_pi {logged[1]:.7f}')
    np.testing.assert_allclose(logged[0], logged[1], rtol=5e-2 if prec == 'tf32' else 2e-3, atol=1e-5)


@pytest.mark.parametrize('prec', list(PREC))
@pytest.mark.parametrize('fname', ['update_trpolag.npz', 'update_cpo.npz', 'update_pcpo.npz'])
def test_natural_golden_through_torch_loss(cuda, tmp_path, golden_dir, monkeypatch, fname, prec):
    g = np.load(os.path.join(golden_dir, fname))
    name = str(g['name']) if 'name' in g.files else {'update_cpo.npz': 'CPO', 'update_pcpo.npz': 'PCPO'}[fname]
    extra = {k[6:]: float(g[k]) for k in g.files if k.startswith('extra_')}
    if 'cost_limit' in g.files:
        extra['cost_limit'] = float(g['cost_limit'])
    lag = {k[9:]: float(g[k]) for k in g.files if k.startswith('lagrange_')}
    cfg = _golden_cfg(tmp_path, g, prec, extra, lag)
    cfg['algo_cfgs'].update(batch_size=32, update_iters=2)
    hooks = ('_loss_pi', '_loss_pi_cost') if name in ('CPO', 'PCPO') else ('_loss_pi',)
    algo = _agent(monkeypatch, tmp_path, name, _subclass(name, *hooks), cfg).agent
    assert algo._torch_hooks
    perms = _load_golden_batch(algo, g, float(g['ep_cost']))
    algo._update(perm=perms)
    torch.cuda.synchronize()
    m = algo._misc
    tol = 5e-2 if prec == 'tf32' else 5e-3
    for key in ('xHx', 'Alpha', 'gradient_norm', 'H_inv_g', 'FinalStepNorm'):
        np.testing.assert_allclose(m[f'Misc/{key}'], g[f'misc_{key}'][-1], rtol=tol, atol=1e-5, err_msg=key)
    assert int(m['Misc/AcceptanceStep']) == int(g['misc_AcceptanceStep'][-1])
    if name in ('CPO', 'PCPO'):
        assert int(m['Misc/OptimCase']) == int(g['misc_OptimCase'][-1])
        np.testing.assert_allclose(m['Misc/cost_gradient_norm'], g['misc_cost_gradient_norm'][-1], rtol=tol, atol=1e-5)
    np.testing.assert_allclose(float(algo._engine.kl_state[0]), g['kl'][-1], rtol=tol, atol=1e-6)
    _assert_theta(algo._actor_critic.theta.cpu().numpy(), g['theta1'], prec, 2e-3, 2e-5, 1e-3, 5e-3)


# ---- new objectives against a float64 restatement of PolicyGradient._update ------------------------------------------
def _ppo_kl_penalty(cls):
    def _loss_pi(self, obs, act, logp, adv):
        clipped = super(cls_, self)._loss_pi(obs, act, logp, adv)
        self._actor_critic.actor(obs)
        log_ratio = self._actor_critic.actor.log_prob(act) - logp
        return clipped + 0.5 * (torch.exp(log_ratio) - 1 - log_ratio).mean()    # KL(old || new), k3 estimate
    cls_ = type('PPOKLPenalty', (cls,), {'_loss_pi': _loss_pi})
    return cls_


def _cost_surrogate(cls):
    cls_ = type('PPOCostSurrogate', (cls,), {'_compute_adv_surrogate': lambda self, r, c: r - 2.0 * c})
    return cls_


def _ref_loss(kind, p, obs, act, logp, adv_r, adv_c, clip):
    d = oac.actor_dist(p, obs)
    log_ratio = d.log_prob(act).sum(-1) - logp
    ratio = torch.exp(log_ratio)
    adv = adv_r if kind == 'kl' else adv_r - 2.0 * adv_c
    loss = -torch.min(ratio * adv, torch.clamp(ratio, 1 - clip, 1 + clip) * adv).mean()
    if kind == 'kl':
        loss = loss + 0.5 * (ratio - 1 - log_ratio).mean()
    return loss


def _ref_update(theta, data, orders, kind, *, batch_size, clip, lr, max_grad_norm, critic_norm_coef, O, A):
    """PolicyGradient._update in float64: per minibatch the reward critic, the cost critic, then the actor; each
    clip_grad_norm_ + Adam."""
    th = torch.as_tensor(theta, dtype=torch.float64, device='cuda').clone()
    nets = oac.unflatten(th, O, A)
    params = {n: [v.clone().requires_grad_(True) for v in nets[n].values()] for n in nets}
    names = {n: list(nets[n]) for n in nets}
    opt = {n: torch.optim.Adam(params[n], lr=lr) for n in nets}
    d = {k: torch.as_tensor(v, dtype=torch.float64, device='cuda') for k, v in data.items()}

    def pd(n):
        return dict(zip(names[n], params[n]))

    def step(n, loss):
        opt[n].zero_grad()
        loss.backward()
        clip_grad_norm_(params[n], max_grad_norm)
        opt[n].step()

    for order in orders:
        for s in range(0, len(order), batch_size):
            idx = order[s:s + batch_size]
            obs = d['obs'][idx]
            for n, tgt in (('reward_critic', 'target_value_r'), ('cost_critic', 'target_value_c')):
                loss = torch.nn.functional.mse_loss(oac.critic_value(pd(n), obs), d[tgt][idx])
                loss = loss + sum(p_.pow(2).sum() for p_ in params[n]) * critic_norm_coef
                step(n, loss)
            step('actor', _ref_loss(kind, pd('actor'), obs, d['act'][idx], d['logp'][idx], d['adv_r'][idx],
                                    d['adv_c'][idx], clip))
    return torch.cat([p_.detach().reshape(-1) for n in ('actor', 'reward_critic', 'cost_critic') for p_ in params[n]])


@pytest.mark.parametrize('prec', list(PREC))
@pytest.mark.parametrize('O', [60, 111])
@pytest.mark.parametrize('kind', ['kl', 'surrogate'])
def test_new_objective_vs_float64(cuda, tmp_path, monkeypatch, kind, O, prec):
    from omnisafe_b200.algorithms import registry

    N, T, A = 1024, 64, 8
    B = N * T
    cls = (_ppo_kl_penalty if kind == 'kl' else _cost_surrogate)(registry.get('PPO'))
    cfg = {
        'seed': 3,
        'train_cfgs': {'device': 'cuda', 'vector_env_nums': N, 'total_steps': B, 'matmul_precision': prec},
        'algo_cfgs': {'steps_per_epoch': B, 'batch_size': 8192, 'update_iters': 2, 'use_cost': True,
                      'max_grad_norm': 0.05, 'kl_early_stop': False},
        'logger_cfgs': {'log_dir': str(tmp_path), 'window_lens': 10, 'use_tensorboard': False},
        'env_cfgs': {'obs_dim': O, 'act_dim': A, 'max_episode_steps': 16},
        'model_cfgs': {'actor': {'lr': 1e-3}, 'critic': {'lr': 1e-3}},
    }
    algo = _agent(monkeypatch, tmp_path, 'PPO', cls, cfg).agent
    assert algo._torch_hooks
    rng = np.random.default_rng(O)
    theta = oac.init_theta(O, A, seed=11)
    obs = rng.standard_normal((B, O)).astype(np.float32)
    eps = rng.standard_normal((B, A)).astype(np.float32)
    act, _, _, logp = oac.step(theta, obs, eps, O, A)
    logp = (logp + 0.3 * rng.standard_normal(B)).astype(np.float32)
    raw = {'obs': obs, 'act': act, 'logp': logp, 'adv_r': rng.standard_normal(B).astype(np.float32),
           'adv_c': rng.standard_normal(B).astype(np.float32),
           'target_value_r': rng.standard_normal(B).astype(np.float32),
           'target_value_c': rng.standard_normal(B).astype(np.float32)}
    moments = np.array([0.3, 1.7, -0.2, 1.0], np.float32)
    algo._actor_critic.load_flat(theta)
    for k, v in raw.items():         # slab row r holds sample r
        algo._buf.data[k].copy_(torch.as_tensor(v.reshape(T, N, *v.shape[1:])).cuda())
    algo._buf.adv_moments.copy_(torch.as_tensor(moments))
    orders = [rng.permutation(B) for _ in range(2)]
    algo._update(perm=torch.as_tensor(np.stack(orders).astype(np.int32)).cuda())
    torch.cuda.synchronize()
    ref_data = dict(raw, adv_r=(raw['adv_r'] - moments[0]) / moments[1], adv_c=raw['adv_c'] - moments[2])
    want = _ref_update(theta, ref_data, orders, kind, batch_size=8192, clip=0.2, lr=1e-3, max_grad_norm=0.05,
                       critic_norm_coef=0.001, O=O, A=A).cpu().numpy()
    got = algo._actor_critic.theta.cpu().numpy()
    # Adam moves every parameter by ~lr per step: compare the parameter change, relative to lr * steps
    steps = 2 * math.ceil(B / 8192)
    err = np.abs(got - want) / (1e-3 * steps)
    tol = 0.25 if prec == 'tf32' else 0.02
    assert np.quantile(err, 0.999) < tol and err.max() < 10 * tol, (np.quantile(err, 0.999), err.max())


def test_new_objective_through_trpo_line_search(cuda, tmp_path, monkeypatch):
    """TRPO on the custom surrogate adv_r - 2 adv_c: natural direction and line search on the PyTorch loss against
    float64 autograd of the same objective (gradient), and the accepted step keeps KL <= target_kl."""
    from omnisafe_b200.algorithms import registry

    N, T, O, A = 256, 32, 60, 8
    B = N * T
    cls = type('TRPOCostSurrogate', (registry.get('TRPO'),), {'_compute_adv_surrogate': lambda self, r, c: r - 2.0 * c})
    cfg = {'seed': 3, 'train_cfgs': {'device': 'cuda', 'vector_env_nums': N, 'total_steps': B, 'matmul_precision': 'fp32'},
           'algo_cfgs': {'steps_per_epoch': B, 'batch_size': 1024, 'update_iters': 1},
           'logger_cfgs': {'log_dir': str(tmp_path), 'window_lens': 10, 'use_tensorboard': False},
           'env_cfgs': {'obs_dim': O, 'act_dim': A, 'max_episode_steps': 16}}
    algo = _agent(monkeypatch, tmp_path, 'TRPO', cls, cfg).agent
    rng = np.random.default_rng(5)
    theta = oac.init_theta(O, A, seed=4)
    obs = rng.standard_normal((B, O)).astype(np.float32)
    act, _, _, logp = oac.step(theta, obs, rng.standard_normal((B, A)).astype(np.float32), O, A)
    adv_r, adv_c = rng.standard_normal(B).astype(np.float32), rng.standard_normal(B).astype(np.float32)
    algo._actor_critic.load_flat(theta)
    for k, v in {'obs': obs, 'act': act, 'logp': logp, 'adv_r': adv_r, 'adv_c': adv_c}.items():
        algo._buf.data[k].copy_(torch.as_tensor(v.reshape(T, N, *v.shape[1:])).cuda())
    algo._buf.adv_moments.copy_(torch.tensor([0.0, 1.0, 0.0, 1.0]))
    algo._update()
    torch.cuda.synchronize()
    Pa = algo._engine.Pa
    th = torch.as_tensor(theta[:Pa], dtype=torch.float64).cuda().requires_grad_(True)
    p = oac.unflatten(torch.cat([th, torch.zeros(len(theta) - Pa, dtype=torch.float64, device=cuda)]), O, A)['actor']
    t64 = lambda x: torch.as_tensor(x, dtype=torch.float64).cuda()   # noqa: E731
    d = oac.actor_dist(p, t64(obs))
    loss = -(torch.exp(d.log_prob(t64(act)).sum(-1) - t64(logp)) * (t64(adv_r) - 2 * t64(adv_c))).mean()
    loss.backward()
    np.testing.assert_allclose(algo._misc['Misc/gradient_norm'], float(th.grad.norm()), rtol=1e-3)
    assert 1 <= int(algo._misc['Misc/AcceptanceStep']) <= 15
    assert 0 < float(algo._engine.kl_state[0]) <= algo._cfgs.algo_cfgs.target_kl
    with torch.no_grad():
        new = torch.as_tensor(algo._actor_critic.theta[:Pa].cpu().numpy(), dtype=torch.float64).cuda()
        p2 = oac.unflatten(torch.cat([new, torch.zeros(len(theta) - Pa, dtype=torch.float64, device=cuda)]), O, A)['actor']
        loss2 = -(torch.exp(oac.actor_dist(p2, t64(obs)).log_prob(t64(act)).sum(-1) - t64(logp))
                  * (t64(adv_r) - 2 * t64(adv_c))).mean()
    assert float(loss2) < float(loss.detach())


# ---- whole runs ---------------------------------------------------------------------------------------------------------
def _e2e_cfg(tmp, env_cfgs):
    return {'seed': 5, 'train_cfgs': {'device': 'cuda', 'vector_env_nums': 64, 'total_steps': 64 * 32 * 4},
            'algo_cfgs': {'steps_per_epoch': 64 * 32, 'batch_size': 512, 'update_iters': 2},
            'logger_cfgs': {'log_dir': str(tmp), 'save_model_freq': 2, 'window_lens': 100, 'use_tensorboard': False},
            'env_cfgs': env_cfgs}


@pytest.mark.parametrize('env', ['synthetic', 'registered'])
@pytest.mark.parametrize('name', ['PPOLag', 'CPO'])
def test_agent_trains_evaluates_and_resumes(cuda, tmp_path, monkeypatch, name, env):
    """4 epochs with the training state saved every 2, finite progress.csv, evaluate(), and a resume from epoch 2 that
    lands on the same bits.  The registered env is the WideBox CMDP with state hooks (tests/resume_worker.py) for the
    run and its evaluable form (tests/eval_envs.py) for evaluate(), which builds the env without set_seed."""
    import omnisafe_b200

    synthetic = {'obs_dim': 60, 'act_dim': 8, 'max_episode_steps': 16, 'term_prob': 0.02}
    if env == 'registered':
        import eval_envs
        import resume_worker as rw
        from omnisafe_b200.envs import CMDP, Box, ENV_REGISTRY, env_register
        rw.register_envs()
        eval_envs.register(CMDP, Box, env_register, ENV_REGISTRY.support_envs())
        env_id, eval_id, env_cfgs = rw.WIDE_ID, eval_envs.WIDE_BOX_EVAL_ID, {}
    else:
        env_id, eval_id, env_cfgs = 'SyntheticBox-v0', 'SyntheticBox-v0', synthetic
    cls = _subclass(name, '_loss_pi')
    agent = _agent(monkeypatch, tmp_path / 'run', name, cls, _e2e_cfg(tmp_path / 'run', env_cfgs), env_id)
    assert type(agent.agent) is cls
    agent.learn(save_state_freq=2)
    log_dir = agent.agent.logger.log_dir
    rows = open(os.path.join(log_dir, 'progress.csv')).read().strip().splitlines()
    assert len(rows) == 5
    hdr = rows[0].split(',')
    for r in rows[1:]:
        vals = dict(zip(hdr, r.split(',')))
        for k in ('Loss/Loss_pi', 'Train/PolicyRatio', 'Train/KL', 'Metrics/EpRet', 'Loss/Loss_reward_critic'):
            assert math.isfinite(float(vals[k])), (k, vals[k])
    theta_b = agent.agent._actor_critic.theta.clone()
    resumed = omnisafe_b200.Agent.resume(os.path.join(log_dir, 'train_state', 'epoch-2'))
    assert type(resumed.agent) is cls
    resumed.learn()
    assert torch.equal(resumed.agent._actor_critic.theta, theta_b)
    if eval_id == env_id:
        agent.evaluate(num_episodes=2)
    else:
        cfg = _e2e_cfg(tmp_path / 'eval', env_cfgs)
        cfg['train_cfgs']['total_steps'] = 64 * 32
        ev = _agent(monkeypatch, tmp_path / 'eval', name, cls, cfg, eval_id)
        ev.learn()
        ev.evaluate(num_episodes=2)


@pytest.mark.parametrize('name', ['PPOLag', 'TRPOLag'])
def test_subclass_without_overrides_stays_fused(cuda, tmp_path, monkeypatch, name):
    import omnisafe_b200

    cfg = _e2e_cfg(tmp_path / 'a', {'obs_dim': 60, 'act_dim': 8, 'max_episode_steps': 16, 'term_prob': 0.02})
    base = omnisafe_b200.Agent(name, 'SyntheticBox-v0', custom_cfgs=cfg)
    base.learn()
    from omnisafe_b200.algorithms import registry
    cls = type(f'Plain{name}', (registry.get(name),), {})
    cfg = _e2e_cfg(tmp_path / 'b', {'obs_dim': 60, 'act_dim': 8, 'max_episode_steps': 16, 'term_prob': 0.02})
    sub = _agent(monkeypatch, tmp_path, name, cls, cfg)
    assert not sub.agent._torch_hooks
    sub.learn()
    assert torch.equal(base.agent._actor_critic.theta, sub.agent._actor_critic.theta)


def test_torch_path_follows_the_fused_sample_order(cuda, tmp_path, monkeypatch):
    """Without a supplied permutation the PyTorch path draws the kernels' Feistel order: one epoch of a PPOLag
    subclass returning super()'s loss lands where the fused PPOLag does (fp32 tiles)."""
    import omnisafe_b200

    env_cfgs = {'obs_dim': 60, 'act_dim': 8, 'max_episode_steps': 16, 'term_prob': 0.02}
    runs = []
    for tag, cls in (('fused', None), ('torch', _subclass('PPOLag', '_loss_pi'))):
        cfg = _e2e_cfg(tmp_path / tag, env_cfgs)
        cfg['train_cfgs'].update(total_steps=64 * 32, matmul_precision='fp32')
        ag = _agent(monkeypatch, tmp_path, 'PPOLag', cls, cfg) if cls else omnisafe_b200.Agent(
            'PPOLag', 'SyntheticBox-v0', custom_cfgs=cfg)
        ag.learn()
        runs.append(ag.agent._actor_critic.theta.cpu().numpy())
    bad = ~np.isclose(runs[1], runs[0], rtol=2e-4, atol=2e-6)
    assert bad.mean() < 1e-3 and np.abs(runs[1] - runs[0]).max() < 2e-3, (bad.sum(), np.abs(runs[1] - runs[0]).max())
