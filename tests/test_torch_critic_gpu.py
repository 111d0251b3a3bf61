"""GPU: critic updates written in PyTorch on the kernel update path.

- the supplied-dV backward (osb_critic_dv_backward) against float64 autograd of the critic MLP, both critics, every
  precision, and the forward a hook sees against the update kernels' critic forward, bit for bit;
- a subclass whose critic hooks call super() ends `_update` where the stepwise kernel path does (first-order and
  natural families, Saute);
- losses the kernels do not have (Huber, PPO value clipping) against a float64 restatement of PolicyGradient._update,
  with the actor on its kernel step or on its own hook, clipping active;
- whole runs through Agent (synthetic and registered env), evaluation and a bit-exact resume, progress.csv included.
"""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch.nn.utils.clip_grad import clip_grad_norm_

from oracle import actor_critic as oac

pytestmark = pytest.mark.gpu
PREC = {'fp32': 0, 'tf32': 1, 'bf16x3': 2}
HOOKS = ('_update_reward_critic', '_update_cost_critic')
NAMES = {1: 'reward_critic', 2: 'cost_critic'}


def _tiles(prec, O):
    return 2 if prec == 'bf16x3' and O <= 64 else (1 if prec == 'tf32' and O <= 512 else 0)


def _dv_backward(th, O, A, net, obs, dv, p, value=None):
    from omnisafe_b200._lib import current_stream, lib, ptr

    B, P = obs.shape[0], th.numel()
    nb = lib().osb_critic_dv_grid_blocks(B, O, p)
    gpart = torch.zeros(nb * P, dtype=torch.float32, device='cuda')
    stats = torch.zeros(nb * 24, dtype=torch.float32, device='cuda')
    lib().osb_critic_dv_backward(ptr(th), O, A, net, ptr(obs), ptr(dv), ptr(value), B, p, ptr(gpart), ptr(stats),
                                 current_stream())
    return gpart.view(nb, P)


# ---- the supplied-dV backward ----------------------------------------------------------------------------------------
@pytest.mark.parametrize('prec', list(PREC))
@pytest.mark.parametrize('O', [17, 60, 64, 65, 376])
@pytest.mark.parametrize('B', [1, 777, 16384])
@pytest.mark.parametrize('net', [1, 2])
def test_dv_backward_vs_autograd(cuda, prec, O, B, net):
    A = 3 if net == 1 else 16         # the critic segment's offset moves with the actor's size
    rng = np.random.default_rng(O * 31 + B + net)
    theta = oac.init_theta(O, A, seed=O + net)
    lay = oac.layout(O, A)[NAMES[net]]
    th = torch.as_tensor(theta).cuda()
    obs = torch.as_tensor(rng.standard_normal((B, O)).astype(np.float32)).cuda()
    dv = torch.as_tensor(rng.standard_normal(B).astype(np.float32)).cuda()
    value = torch.empty(B, dtype=torch.float32, device='cuda')
    part = _dv_backward(th, O, A, net, obs, dv, PREC[prec], value)
    s, n = lay['start'], lay['size']
    outside = torch.cat([part[:, :s], part[:, s + n:]], 1)
    assert torch.count_nonzero(outside) == 0, 'only the critic segment is written'
    got = part[:, s:s + n].double().sum(0).cpu().numpy()
    th64 = th.double().requires_grad_(True)
    params = oac.unflatten(th64, O, A)[NAMES[net]]
    (oac.critic_value(params, obs.double()) * dv.double()).sum().backward()
    want = th64.grad[s:s + n].cpu().numpy()
    tol = 2e-2 if prec == 'tf32' else 2e-4
    np.testing.assert_allclose(got, want, rtol=tol, atol=tol * np.abs(want).max())
    v64 = oac.critic_value(params, obs.double()).detach()
    np.testing.assert_allclose(value.cpu().numpy(), v64.cpu().numpy(), rtol=tol, atol=tol * float(v64.abs().max()))


@pytest.mark.parametrize('prec', list(PREC))
@pytest.mark.parametrize('O', [17, 60, 64, 65, 376])
@pytest.mark.parametrize('net', [1, 2])
def test_hook_forward_has_the_update_kernels_bits(cuda, prec, O, net):
    """The MSE step through the hook's forward (the dV entry with dV = 0, as TrainingCritic runs it) and the dV
    backward gives the update kernel's critic partials bit for bit: the same V per row, the same tiles and CTAs."""
    from omnisafe_b200._lib import current_stream, lib, ptr

    A, B = 8, 3001
    p = PREC[prec]
    rng = np.random.default_rng(O + 7 * net)
    th = torch.as_tensor(oac.init_theta(O, A, seed=O)).cuda()
    P = th.numel()
    obs = torch.as_tensor(rng.standard_normal((B, O)).astype(np.float32)).cuda()
    tv = torch.as_tensor(rng.standard_normal(B).astype(np.float32)).cuda()
    z = lambda *s: torch.zeros(*s, dtype=torch.float32, device='cuda')   # noqa: E731
    act, logp, adv, mu_old, logstd_old = z(B, A), z(B), z(B), z(B, A), z(A)
    moments = torch.tensor([0.0, 1.0, 0.0, 1.0], device='cuda')
    perm = torch.arange(B, dtype=torch.int32, device='cuda')
    tiles = _tiles(prec, O)
    grad_fn = {0: lib().osb_minibatch_grad, 1: lib().osb_minibatch_grad_tc, 2: lib().osb_minibatch_grad_x3}[tiles]
    nb = lib().osb_tc_grid_blocks(B, 1 << net) if tiles else lib().osb_update_grid_blocks(B)
    gpart, stats = z(nb * P), z(nb * 24)
    grad_fn(ptr(th), O, A, ptr(obs), ptr(act), ptr(logp), ptr(adv), ptr(adv), ptr(tv), ptr(tv), ptr(mu_old),
            ptr(moments), ptr(perm), B, 0, 0, B, 1, 0.0, 0.0, 1.0, 0.0, 0, ptr(logstd_old), 1 << net, ptr(gpart),
            ptr(stats), 0, current_stream())
    v = z(B)
    _dv_backward(th, O, A, net, obs, z(B), p, v)
    inv_b = torch.tensor(1.0, device='cuda') / torch.tensor(float(B), device='cuda')
    dv = (2.0 * (v - tv)) * inv_b                      # d mse / d v as the update kernels form it
    part = _dv_backward(th, O, A, net, obs, dv, p)
    assert part.shape[0] == nb
    lay = oac.layout(O, A)[NAMES[net]]
    s, n = lay['start'], lay['size']
    want = gpart.view(nb, P)[:, s:s + n]
    assert torch.equal(part[:, s:s + n], want), (part[:, s:s + n] - want).abs().max()


# ---- algorithms built on synthetic data ------------------------------------------------------------------------------
def _cfg(tmp, prec, algo_extra=None, N=256, T=32, O=60, A=8):
    return {
        'seed': 3,
        'train_cfgs': {'device': 'cuda', 'vector_env_nums': N, 'total_steps': N * T, 'matmul_precision': prec},
        'algo_cfgs': {'steps_per_epoch': N * T, 'batch_size': 1024, 'update_iters': 2, 'kl_early_stop': False,
                      **(algo_extra or {})},
        'logger_cfgs': {'log_dir': str(tmp), 'window_lens': 10, 'use_tensorboard': False},
        'env_cfgs': {'obs_dim': O, 'act_dim': A, 'max_episode_steps': 16},
    }


def _agent(monkeypatch, name, cls, cfg, env_id='SyntheticBox-v0'):
    import omnisafe_b200
    from omnisafe_b200.algorithms import registry

    if cls is not None:
        monkeypatch.setitem(registry._classes, name, cls)
    return omnisafe_b200.Agent(name, env_id, custom_cfgs=cfg)


def _fill(algo, seed):
    """Random rollout data in the slab (slab row r holds sample r); returns it as float32 numpy."""
    O, A = algo._env.obs_dim, algo._env.act_dim
    T, N = algo._buf.T, algo._buf.N
    B = T * N
    rng = np.random.default_rng(seed)
    theta = algo._actor_critic.theta.cpu().numpy()
    obs = rng.standard_normal((B, O)).astype(np.float32)
    act, _, _, logp = oac.step(theta, obs, rng.standard_normal((B, A)).astype(np.float32), O, A)
    raw = {'obs': obs, 'act': act, 'logp': (logp + 0.3 * rng.standard_normal(B)).astype(np.float32),
           'adv_r': rng.standard_normal(B).astype(np.float32), 'adv_c': rng.standard_normal(B).astype(np.float32),
           'target_value_r': rng.standard_normal(B).astype(np.float32),
           'target_value_c': rng.standard_normal(B).astype(np.float32)}
    for k, v in raw.items():
        algo._buf.data[k].copy_(torch.as_tensor(v.reshape(T, N, *v.shape[1:])).cuda())
    algo._buf.adv_moments.copy_(torch.tensor([0.0, 1.0, 0.0, 1.0]))
    algo._env.window_sums.copy_(torch.tensor([0.0, 30.0, 0.0, 10.0], dtype=torch.float64))
    return raw


def _super_subclass(base, *hooks):
    body = {}
    if '_update_reward_critic' in hooks:
        body['_update_reward_critic'] = lambda self, o, t: super(cls, self)._update_reward_critic(o, t)
    if '_update_cost_critic' in hooks:
        body['_update_cost_critic'] = lambda self, o, t: super(cls, self)._update_cost_critic(o, t)
    if '_loss_pi' in hooks:
        body['_loss_pi'] = lambda self, o, a, lp, adv: super(cls, self)._loss_pi(o, a, lp, adv)
    cls = type(f'User{base.__name__}', (base,), body)
    return cls


def _assert_theta(got, want, prec, rtol=2e-4, atol=2e-6, frac=1e-3, amax=2e-3):
    if prec == 'tf32':      # the tf32 tiles' bar (test_update_tc_gpu.py): 5e-3-level arithmetic
        rtol, atol, frac, amax = 2e-2, 2e-3, 2e-2, 2e-2
    bad = ~np.isclose(got, want, rtol=rtol, atol=atol)
    assert bad.mean() < frac and np.abs(got - want).max() < amax, (bad.sum(), np.abs(got - want).max())


@pytest.mark.parametrize('prec', list(PREC))
@pytest.mark.parametrize('name', ['PPOLag', 'FOCOPS', 'CPO', 'PPOSaute'])
def test_super_hooks_reproduce_the_stepwise_kernel_path(cuda, tmp_path, monkeypatch, name, prec):
    from omnisafe_b200.algorithms import registry

    B, runs = 256 * 32, {}
    orders = np.stack([np.random.default_rng(1).permutation(B) for _ in range(2)]).astype(np.int32)
    for tag in ('kernel', 'hook'):
        with monkeypatch.context() as m:
            m.setenv('OSB_X3_NO_FUSE', '1')          # the stepwise kernel path in every precision
            cls = _super_subclass(registry.get(name), *HOOKS) if tag == 'hook' else None
            algo = _agent(m, name, cls, _cfg(tmp_path / tag, prec, {'use_cost': True})).agent
            assert sorted(algo._critic_hooks) == (sorted(HOOKS) if cls else [])
            _fill(algo, 9)
            theta0 = algo._actor_critic.theta.clone()
            algo._update(perm=torch.as_tensor(orders).cuda())
            torch.cuda.synchronize()
            ac = algo._actor_critic
            runs[tag] = [t.cpu().numpy() for t in (ac.theta, ac.adam_m, ac.adam_step)]
            if tag == 'hook':
                stats = algo._loss_stats.means()
    (th_k, m_k, step_k), (th_h, m_h, step_h) = runs['kernel'], runs['hook']
    assert np.array_equal(step_k, step_h)
    Pa = algo._engine.Pa
    assert not np.array_equal(th_h[Pa:], theta0[Pa:].cpu().numpy()), 'the critics trained'
    _assert_theta(th_h, th_k, prec)
    scale = np.abs(m_k).max()
    _assert_theta(m_h / scale, m_k / scale, prec, 1e-3, 1e-4, 1e-2, 1e-2)
    for key in ('Loss/Loss_reward_critic', 'Loss/Loss_cost_critic'):
        assert math.isfinite(stats[key]) and stats[key] > 0, (key, stats)


# ---- losses the kernels do not have, against float64 ------------------------------------------------------------------
DELTA, VCLIP, COEF, MAXN, LR = 0.5, 0.2, 0.001, 0.05, 1e-3


def _critic_loss64(kind, p, obs, tgt, p_old):
    v = oac.critic_value(p, obs)
    if kind == 'huber':
        loss = F.huber_loss(v, tgt, delta=DELTA)
    elif kind == 'vclip':
        v_old = oac.critic_value(p_old, obs)
        v_clip = v_old + (v - v_old).clamp(-VCLIP, VCLIP)
        loss = 0.5 * torch.max((v - tgt) ** 2, (v_clip - tgt) ** 2).mean()
    else:
        loss = F.mse_loss(v, tgt)
    return loss + sum(t.pow(2).sum() for t in p.values()) * COEF


def _hook(kind, which):
    """A user's critic hook: upstream's method body with the loss replaced."""
    def hook(self, obs, target):
        ac = self._actor_critic
        critic, opt = getattr(ac, which), getattr(ac, f'{which}_optimizer')
        opt.zero_grad()
        value = critic(obs)[0]
        if kind == 'huber':
            loss = F.huber_loss(value, target, delta=DELTA)
        else:      # PPO value clipping around the values of the critic the update started from
            v_old = oac.critic_value(self._critics_old[which], obs)
            v_clip = v_old + (value - v_old).clamp(-VCLIP, VCLIP)
            loss = 0.5 * torch.max((value - target) ** 2, (v_clip - target) ** 2).mean()
        for param in critic.parameters():
            loss = loss + param.pow(2).sum() * COEF
        loss.backward()
        clip_grad_norm_(critic.parameters(), MAXN)
        from omnisafe_b200.utils import distributed
        distributed.avg_grads(critic)
        opt.step()
        self._logger.store({f'Loss/Loss_{which}': loss.mean().item()})
    return hook


def _ref_update64(theta, data, orders, kinds, *, batch_size, clip, O, A):
    """PolicyGradient._update in float64: per minibatch the reward critic, the cost critic, then the PPO actor; each
    clip_grad_norm_ + Adam.  kinds: net -> 'huber' / 'vclip' / 'mse'."""
    th = torch.as_tensor(theta, dtype=torch.float64, device='cuda').clone()
    nets = oac.unflatten(th, O, A)
    old = {n: {k: v.clone() for k, v in nets[n].items()} for n in nets}
    params = {n: {k: v.clone().requires_grad_(True) for k, v in nets[n].items()} for n in nets}
    opt = {n: torch.optim.Adam(list(params[n].values()), lr=LR) for n in nets}
    d = {k: torch.as_tensor(v, dtype=torch.float64, device='cuda') for k, v in data.items()}

    def step(n, loss):
        opt[n].zero_grad()
        loss.backward()
        clip_grad_norm_(list(params[n].values()), MAXN)
        opt[n].step()

    for order in orders:
        for s in range(0, len(order), batch_size):
            idx = torch.as_tensor(order[s:s + batch_size], device='cuda')
            obs = d['obs'][idx]
            for n, tgt in (('reward_critic', 'target_value_r'), ('cost_critic', 'target_value_c')):
                step(n, _critic_loss64(kinds[n], params[n], obs, d[tgt][idx], old[n]))
            dist = oac.actor_dist(params['actor'], obs)
            ratio = torch.exp(dist.log_prob(d['act'][idx]).sum(-1) - d['logp'][idx])
            adv = d['adv_r'][idx]
            step('actor', -torch.min(ratio * adv, torch.clamp(ratio, 1 - clip, 1 + clip) * adv).mean())
    return torch.cat([p.detach().reshape(-1) for n in ('actor', 'reward_critic', 'cost_critic')
                      for p in params[n].values()])


@pytest.mark.parametrize('prec', list(PREC))
@pytest.mark.parametrize('actor', ['kernel', 'hook'])
@pytest.mark.parametrize('case', ['huber_reward', 'huber_cost', 'huber_both', 'vclip_both'])
def test_new_critic_loss_vs_float64(cuda, tmp_path, monkeypatch, case, actor, prec):
    from omnisafe_b200.algorithms import registry

    kind, which = case.split('_')
    nets = {'reward': ['reward_critic'], 'cost': ['cost_critic'], 'both': ['reward_critic', 'cost_critic']}[which]
    base = registry.get('PPO')
    body = {f'_update_{n}': _hook(kind, n) for n in nets}
    if kind == 'vclip':       # the critics the update starts from: what the rollout's values came from
        def _update(self, *args, **kwargs):
            self._critics_old = oac.unflatten(self._actor_critic.theta.clone(), self._env.obs_dim, self._env.act_dim)
            return base._update(self, *args, **kwargs)
        body['_update'] = _update
    if actor == 'hook':
        body['_loss_pi'] = lambda self, o, a, lp, adv: base._loss_pi(self, o, a, lp, adv)
    cls = type('UserPPO', (base,), body)
    cfg = _cfg(tmp_path, prec, {'use_cost': True, 'max_grad_norm': MAXN, 'entropy_coef': 0.0,
                                'critic_norm_coef': COEF, 'use_critic_norm': True})
    cfg['model_cfgs'] = {'actor': {'lr': LR}, 'critic': {'lr': LR}}
    algo = _agent(monkeypatch, 'PPO', cls, cfg).agent
    assert sorted(algo._critic_hooks) == sorted(f'_update_{n}' for n in nets)
    assert bool(algo._actor_hooks) == (actor == 'hook')
    raw = _fill(algo, 4)
    O, A = algo._env.obs_dim, algo._env.act_dim
    B = raw['obs'].shape[0]
    theta = algo._actor_critic.theta.cpu().numpy()
    orders = [np.random.default_rng(s).permutation(B) for s in range(2)]
    algo._update(perm=torch.as_tensor(np.stack(orders).astype(np.int32)).cuda())
    torch.cuda.synchronize()
    kinds = {n: (kind if n in nets else 'mse') for n in ('reward_critic', 'cost_critic')}
    want = _ref_update64(theta, raw, orders, kinds, batch_size=1024, clip=algo._cfgs.algo_cfgs.clip, O=O,
                         A=A).cpu().numpy()
    got = algo._actor_critic.theta.cpu().numpy()
    steps = 2 * math.ceil(B / 1024)
    err = np.abs(got - want) / (LR * steps)
    tol = 0.25 if prec == 'tf32' else 0.02
    assert np.quantile(err, 0.999) < tol and err.max() < 10 * tol, (np.quantile(err, 0.999), err.max())
    # clipping was active: the first critic gradient of the float64 loop is above MAXN (Huber's is bounded)
    p = oac.unflatten(torch.as_tensor(theta, dtype=torch.float64, device='cuda'), O, A)['reward_critic']
    p = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    idx = torch.as_tensor(orders[0][:1024], device='cuda')
    d = {k: torch.as_tensor(raw[k], dtype=torch.float64, device='cuda')[idx] for k in ('obs', 'target_value_r')}
    _critic_loss64(kinds['reward_critic'], p, d['obs'], d['target_value_r'], p).backward()
    assert float(torch.cat([v.grad.reshape(-1) for v in p.values()]).norm()) > 1.2 * MAXN
    st = algo._loss_stats.means()
    for n in nets:
        assert math.isfinite(st[f'Loss/Loss_{n}'])


# ---- whole runs ---------------------------------------------------------------------------------------------------------
def _e2e_cfg(tmp, env_cfgs):
    return {'seed': 5, 'train_cfgs': {'device': 'cuda', 'vector_env_nums': 64, 'total_steps': 64 * 32 * 4},
            'algo_cfgs': {'steps_per_epoch': 64 * 32, 'batch_size': 512, 'update_iters': 2},
            'logger_cfgs': {'log_dir': str(tmp), 'save_model_freq': 2, 'window_lens': 100, 'use_tensorboard': False},
            'env_cfgs': env_cfgs}


@pytest.mark.parametrize('env', ['synthetic', 'registered'])
@pytest.mark.parametrize('name', ['PPOLag', 'CPO'])
def test_agent_trains_evaluates_and_resumes(cuda, tmp_path, monkeypatch, name, env):
    """4 epochs with a Huber reward critic and the library's cost critic through super(), the training state saved
    every 2; a resume from epoch 2 of a copy of the run stopped there lands on the same bits, progress.csv included
    (but Time/*); evaluate().  The registered env is the graph-safe WideBox CMDP (replayed as a CUDA graph)."""
    import omnisafe_b200
    from omnisafe_b200.algorithms import registry
    from test_resume_gpu import _rows, _stopped_copy

    synthetic = {'obs_dim': 60, 'act_dim': 8, 'max_episode_steps': 16, 'term_prob': 0.02}
    if env == 'registered':
        import eval_envs
        import resume_worker as rw
        from omnisafe_b200.envs import CMDP, Box, ENV_REGISTRY, env_register
        rw.register_envs()
        eval_envs.register(CMDP, Box, env_register, ENV_REGISTRY.support_envs())
        env_id, eval_id, env_cfgs = rw.GRAPH_WIDE_ID, eval_envs.WIDE_BOX_EVAL_ID, {}
    else:
        env_id, eval_id, env_cfgs = 'SyntheticBox-v0', 'SyntheticBox-v0', synthetic
    base = registry.get(name)
    cls = type(f'User{name}', (base,), {
        '_update_reward_critic': _hook('huber', 'reward_critic'),
        '_update_cost_critic': lambda self, o, t: base._update_cost_critic(self, o, t)})
    agent = _agent(monkeypatch, name, cls, _e2e_cfg(tmp_path / 'run', env_cfgs), env_id)
    assert type(agent.agent) is cls
    agent.learn(save_state_freq=2)
    if env == 'registered':
        assert agent.agent._env.graph_mode == 'graph'
    log_dir = agent.agent.logger.log_dir
    rows = _rows(log_dir)
    assert len(rows) == 5
    for r in rows[1:]:
        vals = dict(zip(rows[0], r))
        for k in ('Loss/Loss_pi', 'Loss/Loss_reward_critic', 'Loss/Loss_cost_critic', 'Train/KL', 'Metrics/EpRet'):
            assert math.isfinite(float(vals[k])), (k, vals[k])
    theta_b = agent.agent._actor_critic.theta.clone()
    copy = _stopped_copy(log_dir, str(tmp_path / 'stopped'))
    resumed = omnisafe_b200.Agent.resume(os.path.join(copy, 'train_state', 'epoch-2'))
    assert type(resumed.agent) is cls
    resumed.learn()
    assert torch.equal(resumed.agent._actor_critic.theta, theta_b)
    rb, rc = _rows(log_dir), _rows(resumed.agent.logger.log_dir)
    keep = [i for i, key in enumerate(rb[0]) if not key.startswith('Time/')]
    assert rc[0] == rb[0] and len(rc) == 5
    for e in (2, 3):
        assert [rb[1 + e][i] for i in keep] == [rc[1 + e][i] for i in keep], f'progress.csv row of epoch {e + 1}'
    if eval_id == env_id:
        agent.evaluate(num_episodes=2)
    else:
        cfg = _e2e_cfg(tmp_path / 'eval', env_cfgs)
        cfg['train_cfgs']['total_steps'] = 64 * 32
        ev = _agent(monkeypatch, name, cls, cfg, eval_id)
        ev.learn()
        ev.evaluate(num_episodes=2)
