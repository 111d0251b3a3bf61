"""GPU: hidden widths below 64, run as zero-padded 64-wide networks (models/actor_critic.py ParamMap).

- goldens of the unmodified reference with actor [24, 40] and critic [8, 64] (make_golden_hidden.py): a rollout epoch,
  PPOLag._update, CPO's Fisher-vector product and CG, and CPO._update (case analysis, line search, parameters), at the
  bars of the 64-wide golden tests;
- after two epochs of Agent.learn every padded coordinate of theta, adam_m and adam_v is +0 (fp32, tf32, bf16x3; synthetic
  and registered env; a subclass training through `_loss_pi` and a critic hook);
- a narrow model and its zero-padded 64-wide twin give the same bits: training (slabs, parameters, Adam state), step /
  predict / critics and Evaluator.evaluate on the synthetic and a registered env;
- a narrow run resumed from epoch 2 lands on the uninterrupted run's bits, and its checkpoints hold upstream's shapes.
"""
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
PREC = {'fp32': 0, 'tf32': 1, 'bf16x3': 2}
ACTOR, CRITIC = [24, 40], [8, 64]


def _model_cfgs(actor=ACTOR, critic=CRITIC, lr_actor=3e-4, lr_critic=3e-4):
    return NS(actor=NS(hidden_sizes=list(actor), activation='tanh', lr=lr_actor),
              critic=NS(hidden_sizes=list(critic), activation='tanh', lr=lr_critic),
              actor_type='gaussian_learning', linear_lr_decay=False, weight_initialization_mode='kaiming_uniform')


def _golden(golden_dir, name):
    from omnisafe_b200.models import ParamMap

    g = np.load(os.path.join(golden_dir, f'{name}_hidden.npz'))
    O, A = (int(g['O']), int(g['A'])) if 'O' in g.files else (12, 3)     # update_ppolag: make_golden.py's 12 x 3
    pmap = ParamMap(O, A, [int(x) for x in g['actor_hidden']], [int(x) for x in g['critic_hidden']])
    for key in ('theta', 'theta0', 'theta1'):      # the reference's flat order of the narrow networks
        assert key not in g.files or g[key].shape == (pmap.ref['total'],), (key, g[key].shape)
    return g, pmap, O, A


def _pads(pmap, dev='cpu'):
    mask = torch.ones(pmap.kernel['total'], dtype=torch.bool, device=dev)
    for net in ('actor', 'reward_critic', 'cost_critic'):
        for v in pmap.views(mask, net).values():
            v.fill_(False)
    return mask


def _assert_pads_zero(pmap, **vecs):
    pads = _pads(pmap)
    for name, v in vecs.items():
        bits = v.detach().cpu()[pads].view(torch.int32)
        assert int(bits.numel()) > 0 and not bits.any(), f'{name}: {int((bits != 0).sum())} padded coordinates not +0'


# ---- goldens of the unmodified reference ------------------------------------------------------------------------------
@pytest.mark.parametrize('precision', [0, 2])      # the 64-wide rollout golden's precisions and bar
def test_rollout_golden_reference(cuda, golden_dir, precision):
    from test_rollout_gpu import _cfgs

    from omnisafe_b200.adapter.onpolicy_adapter import OnPolicyAdapter
    from omnisafe_b200.common.buffer import VectorOnPolicyBuffer
    from omnisafe_b200.models import ConstraintActorCritic

    g, pmap, O, A = _golden(golden_dir, 'rollout_ppolag')
    N, T = int(g['N']), int(g['T'])
    cfgs = _cfgs(True, 10, False, obs_dim=O, act_dim=A, max_episode_steps=int(g['tmax']), term_prob=float(g['term_prob']))
    ad = OnPolicyAdapter('SyntheticBox-v0', N, int(g['seed']), cfgs, device=cuda)
    ad.precision = precision
    agent = ConstraintActorCritic(O, A, _model_cfgs(), epochs=1, device=cuda)
    agent.load_flat(pmap.to_kernel(g['theta']))
    buf = VectorOnPolicyBuffer(O, A, T, 0.99, 0.95, 0.95, 'gae', 0.0, True, True, num_envs=N, device=cuda)
    ad.rollout(T, agent, buf, eps=torch.as_tensor(g['eps']).to(cuda))
    torch.cuda.synchronize()
    sl = {k: v.cpu().numpy() for k, v in buf.data.items() if v is not None}
    t = dict(rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(sl['obs'], g['slab_obs'], **t)
    np.testing.assert_allclose(sl['act'], g['slab_act'], **t)
    np.testing.assert_allclose(sl['reward'], g['slab_reward'], **t)
    assert np.array_equal(sl['cost'], g['slab_cost'])
    np.testing.assert_allclose(sl['value_r'], g['slab_value_r'], **t)
    np.testing.assert_allclose(sl['value_c'], g['slab_value_c'], **t)
    np.testing.assert_allclose(sl['logp'], g['slab_logp'], rtol=2e-5, atol=5e-5)
    nz = ad._obs_normalizer
    np.testing.assert_allclose(nz.mean.cpu().numpy(), g['norm_mean'], **t)
    np.testing.assert_allclose(nz.std.cpu().numpy(), g['norm_std'], **t)
    buf.finish_paths()
    torch.cuda.synchronize()
    np.testing.assert_allclose(buf.data['adv_r'].cpu().numpy(), g['slab_adv_r'], rtol=1e-4, atol=5e-5)
    np.testing.assert_allclose(buf.data['adv_c'].cpu().numpy(), g['slab_adv_c'], rtol=1e-4, atol=5e-5)
    np.testing.assert_allclose(buf.data['target_value_r'].cpu().numpy(), g['slab_target_value_r'], rtol=1e-4, atol=5e-5)


def _setup(dev, g, pmap, O, A, lr_actor=3e-4, lr_critic=3e-4):
    """test_update_gpu._setup with the narrow model: the golden's initial parameters and its env-major data."""
    from omnisafe_b200.algorithms.engine import UpdateEngine
    from omnisafe_b200.common.buffer import VectorOnPolicyBuffer
    from omnisafe_b200.models import ConstraintActorCritic

    N, T = 8, 24
    data = {k[5:]: g[k] for k in g.files if k.startswith('data_')}
    agent = ConstraintActorCritic(O, A, _model_cfgs(lr_actor=lr_actor, lr_critic=lr_critic), epochs=1, device=dev)
    assert agent.param_map.ref == pmap.ref
    agent.load_flat(pmap.to_kernel(g['theta0']))
    buf = VectorOnPolicyBuffer(O, A, T, 0.99, 0.95, 0.95, 'gae', 0.0, True, True, num_envs=N, device=dev)
    for k in ('obs', 'act', 'logp', 'adv_r', 'adv_c', 'target_value_r', 'target_value_c'):
        x = np.asarray(data[k], np.float32)
        buf.data[k].copy_(torch.as_tensor(x.reshape(N, T, *x.shape[1:]).swapaxes(0, 1).copy()).to(dev))
    buf.adv_moments.copy_(torch.tensor([0.0, 1.0, 0.0, 1.0]))     # the data holds standardised advantages
    return data, agent, buf, UpdateEngine(agent, buf)


def test_ppolag_update_epoch_golden(cuda, golden_dir):
    from test_update_gpu import _rows

    from omnisafe_b200.common.lagrange import Lagrange

    g, pmap, O, A = _golden(golden_dir, 'update_ppolag')
    N, T = 8, 24
    data, agent, buf, eng = _setup(cuda, g, pmap, O, A)
    lag = Lagrange(float(g['cost_limit']), float(g['lam0']), float(g['lambda_lr']), device=cuda)
    lag.update_lagrange_multiplier(torch.tensor([0.0, float(g['Jc']) * 10, 0.0, 10.0], dtype=torch.float64, device=cuda))
    perms = torch.as_tensor(np.stack([_rows(p_, N, T) for p_ in g['perms'][::2]])).to(cuda)
    eng.ppo_epoch(loss_kind=0, lagrange=lag.state, net_mask=7, batch_size=int(g['batch_size']),
                  update_iters=int(g['update_iters']), clip=0.2, entropy_coef=0.0, critic_norm_coef=0.001,
                  max_grad_norm=40.0, lr_actor=3e-4, lr_critic=3e-4, target_kl=0.02, kl_early_stop=True, perm=perms)
    torch.cuda.synchronize()
    got, want = pmap.to_ref(agent.theta.cpu()).numpy(), g['theta1']
    bad = ~np.isclose(got, want, rtol=2e-4, atol=2e-6)
    assert bad.mean() < 1e-3 and np.abs(got - want).max() < 2e-3, (bad.sum(), np.abs(got - want).max())
    _assert_pads_zero(pmap, theta=agent.theta, adam_m=agent.adam_m, adam_v=agent.adam_v)
    kls = eng.kl_state.cpu().numpy()
    np.testing.assert_allclose(kls[0], g['kl'][-1], rtol=2e-3, atol=1e-6)
    assert int(kls[1]) == int(g['stop_iter'][-1])
    ts = eng.train_stats.cpu().numpy().reshape(3, 8)
    np.testing.assert_allclose(ts[0, 0] / ts[0, 3], g['loss_pi'].mean(), rtol=1e-3, atol=1e-5)
    np.testing.assert_allclose(ts[1, 0] / ts[1, 3], g['loss_r'].mean(), rtol=1e-3, atol=1e-5)
    np.testing.assert_allclose(ts[2, 0] / ts[2, 3], g['loss_c'].mean(), rtol=1e-3, atol=1e-5)


@pytest.mark.parametrize('precision', [0, 2])      # the 64-wide FVP / CG golden's precisions and bar
def test_fvp_cg_golden(cuda, golden_dir, precision):
    g, pmap, O, A = _golden(golden_dir, 'update_cpo')
    data, agent, buf, eng = _setup(cuda, g, pmap, O, A, lr_actor=None, lr_critic=1e-3)
    eng.precision = precision
    Pa, Pa_ref = eng.Pa, pmap.ref['actor']['size']
    total_ref = pmap.ref['total']

    def to_kernel(v):      # an actor vector in the reference's order -> the kernel layout's actor slice
        return pmap.to_kernel(np.concatenate([v, np.zeros(total_ref - Pa_ref, np.float32)]))[:Pa].to(cuda)

    def to_ref(v):
        full = torch.zeros(pmap.kernel['total'])
        full[:Pa] = v.cpu()
        _assert_pads_zero(pmap, actor_vector=full)
        return pmap.to_ref(full)[:Pa_ref].numpy()

    vec = to_kernel(g['vec'])
    out = torch.zeros_like(vec)
    eng.fvp(vec, out, float(g['cg_damping']))
    torch.cuda.synchronize()
    np.testing.assert_allclose(to_ref(out), g['fvp'], rtol=2e-4, atol=2e-6)
    x = eng.conjugate_gradients(to_kernel(g['bvec']), int(g['cg_iters']), float(g['cg_damping']))
    torch.cuda.synchronize()
    np.testing.assert_allclose(to_ref(x), g['xcg'], rtol=5e-3, atol=2e-5)
    eng.snapshot_old_policy()
    ev = eng.evaluate(agent.theta, None)
    assert abs(ev['kl']) < 1e-9 and abs(ev['ratio'] - 1.0) < 1e-5
    np.testing.assert_allclose(ev['loss_r'], -data['adv_r'].mean(), rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize('prec', ['fp32', 'bf16x3'])      # test_agent_gpu.py::test_cpo_update_golden's precisions
def test_cpo_update_golden(cuda, tmp_path, golden_dir, prec):
    """CPO._update of the unmodified reference with the narrow networks vs ours on identical data: same case analysis,
    same line-search step, same parameters afterwards (test_agent_gpu.py::test_cpo_update_golden's bars), pads +0."""
    import omnisafe_b200

    g, pmap, O, A = _golden(golden_dir, 'update_cpo')
    N, T = int(g['N']), int(g['T'])
    cfg = {
        'seed': int(g['seed']),
        'train_cfgs': {'device': 'cuda', 'vector_env_nums': N, 'total_steps': N * T * 2, 'matmul_precision': prec},
        'algo_cfgs': {'steps_per_epoch': N * T, 'batch_size': 32, 'update_iters': 2, 'cost_limit': float(g['cost_limit'])},
        'logger_cfgs': {'log_dir': str(tmp_path), 'window_lens': 10, 'use_tensorboard': False},
        'model_cfgs': {'actor': {'hidden_sizes': list(pmap.actor_hidden)},
                       'critic': {'hidden_sizes': list(pmap.critic_hidden)}},
        'env_cfgs': {'obs_dim': O, 'act_dim': A, 'max_episode_steps': 8, 'term_prob': 0.05},
    }
    algo = omnisafe_b200.Agent('CPO', 'SyntheticBox-v0', custom_cfgs=cfg).agent
    assert algo._engine.precision == PREC[prec]
    ac = algo._actor_critic
    assert ac.param_map.ref == pmap.ref
    ac.load_flat(pmap.to_kernel(g['theta0']))
    data = {k[5:]: g[k] for k in g.files if k.startswith('data_')}
    for k in ('obs', 'act', 'logp', 'adv_r', 'adv_c', 'target_value_r', 'target_value_c'):
        x = np.asarray(data[k], np.float32)
        algo._buf.data[k].copy_(torch.as_tensor(x.reshape(N, T, *x.shape[1:]).swapaxes(0, 1).copy()).to(cuda))
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
    got, want = pmap.to_ref(ac.theta.cpu()).numpy(), g['theta1']
    bad = ~np.isclose(got, want, rtol=2e-3, atol=2e-5)
    assert bad.mean() < 1e-3 and np.abs(got - want).max() < 5e-3, (bad.sum(), np.abs(got - want).max())
    _assert_pads_zero(pmap, theta=ac.theta, adam_m=ac.adam_m, adam_v=ac.adam_v)


# ---- whole runs ---------------------------------------------------------------------------------------------------------
SYNTHETIC = {'obs_dim': 60, 'act_dim': 8, 'max_episode_steps': 16, 'term_prob': 0.02}


def _custom(tmp, prec='bf16x3', epochs=2, env_cfgs=None, algo=None, actor=ACTOR, critic=CRITIC, save_model_freq=1):
    N, T = 64, 32
    extra = {'max_ep_len': 16} if algo and 'Saute' in algo else ({'cost_limit': 3.0} if algo and 'Early' in algo else {})
    return {'seed': 5,
            'train_cfgs': {'device': 'cuda', 'vector_env_nums': N, 'total_steps': N * T * epochs, 'parallel': 1,
                           'matmul_precision': prec},
            'algo_cfgs': {'steps_per_epoch': N * T, 'batch_size': 512, 'update_iters': 2, **extra},
            'logger_cfgs': {'log_dir': str(tmp), 'save_model_freq': save_model_freq, 'window_lens': 100,
                            'use_tensorboard': False},
            'model_cfgs': {'actor': {'hidden_sizes': list(actor)}, 'critic': {'hidden_sizes': list(critic)}},
            'env_cfgs': dict(SYNTHETIC if env_cfgs is None else env_cfgs)}


def _registered_env():
    import early_envs as ee
    import external_envs as xe

    from omnisafe_b200.envs import CMDP, ENV_REGISTRY, Box, env_register

    xe.register(CMDP, Box, env_register, ENV_REGISTRY.support_envs())
    ee.register(CMDP, Box, env_register, ENV_REGISTRY.support_envs())
    return ee.GRAPH_RESET_WIDE_ID, {'obs_dim': 45, 'act_dim': 3, 'max_episode_steps': 7}


RUNS = [('PPOLag', 'synthetic'), ('CPO', 'synthetic'), ('FOCOPS', 'synthetic'), ('P3O', 'synthetic'),
        ('PPOSaute', 'synthetic'), ('PPOEarlyTerminated', 'synthetic'), ('PPOLag', 'registered'), ('CPO', 'registered'),
        ('FOCOPS', 'registered'), ('P3O', 'registered'), ('PPOEarlyTerminated', 'registered')]


@pytest.mark.timeout(900)
@pytest.mark.parametrize('prec', list(PREC))
@pytest.mark.parametrize('algo,env', RUNS)
def test_pads_stay_zero_through_training(cuda, tmp_path, monkeypatch, algo, env, prec):
    import omnisafe_b200

    monkeypatch.delenv('OSB_NO_GRAPH', raising=False)
    env_id, env_cfgs = ('SyntheticBox-v0', None) if env == 'synthetic' else _registered_env()
    agent = omnisafe_b200.Agent(algo, env_id, custom_cfgs=_custom(tmp_path, prec, env_cfgs=env_cfgs, algo=algo))
    ac = agent.agent._actor_critic
    theta0 = ac.theta.clone()
    agent.learn()
    assert ac.param_map.actor_hidden == tuple(ACTOR) and ac.param_map.critic_hidden == tuple(CRITIC)
    assert torch.isfinite(ac.theta).all() and not torch.equal(ac.theta, theta0)
    _assert_pads_zero(ac.param_map, theta=ac.theta, adam_m=ac.adam_m, adam_v=ac.adam_v)
    pi = torch.load(os.path.join(agent.agent.logger.log_dir, 'torch_save', 'epoch-2.pt'), weights_only=False)['pi']
    assert {k: tuple(v.shape) for k, v in pi.items()} == {k: s for k, (_, s) in ac.param_map.ref['actor']['entries'].items()}


@pytest.mark.timeout(900)
@pytest.mark.parametrize('prec', list(PREC))
def test_pads_stay_zero_with_torch_hooks(cuda, tmp_path, monkeypatch, prec):
    """A subclass training the actor through `_loss_pi` (autograd on the supplied-dmu kernel) and the reward critic
    through a Huber hook on reference-shaped leaves."""
    from test_torch_critic_gpu import _agent, _hook

    from omnisafe_b200.algorithms import registry

    base = registry.get('PPOLag')
    cls = type('UserPPOLag', (base,), {
        '_loss_pi': lambda self, o, a, lp, adv: base._loss_pi(self, o, a, lp, adv),
        '_update_reward_critic': _hook('huber', 'reward_critic')})
    agent = _agent(monkeypatch, 'PPOLag', cls, _custom(tmp_path, prec))
    assert agent.agent._actor_hooks and agent.agent._critic_hooks
    ac = agent.agent._actor_critic
    theta0 = ac.theta.clone()
    agent.learn()
    assert torch.isfinite(ac.theta).all() and not torch.equal(ac.theta, theta0)
    _assert_pads_zero(ac.param_map, theta=ac.theta, adam_m=ac.adam_m, adam_v=ac.adam_v)


def _pad_twin(tmp, prec, algo, env_id, env_cfgs):
    """A narrow run and a 64-wide run that starts from the narrow run's parameters, zero-padded."""
    import omnisafe_b200

    narrow = omnisafe_b200.Agent(algo, env_id, custom_cfgs=_custom(tmp / 'narrow', prec, 1, env_cfgs, algo))
    wide = omnisafe_b200.Agent(algo, env_id, custom_cfgs=_custom(tmp / 'wide', prec, 1, env_cfgs, algo, [64, 64],
                                                                 [64, 64]))
    wide.agent._actor_critic.theta.copy_(narrow.agent._actor_critic.theta)
    return narrow, wide


def _bits(t):
    return t.detach().cpu().reshape(-1).view(torch.uint8) if t.dtype.is_floating_point else t.detach().cpu()


@pytest.mark.timeout(900)
@pytest.mark.parametrize('prec', list(PREC))
@pytest.mark.parametrize('algo,env', [('PPOLag', 'synthetic'), ('CPO', 'synthetic'), ('PPOLag', 'registered')])
def test_narrow_model_is_its_zero_padded_twin(cuda, tmp_path, monkeypatch, algo, env, prec, capsys):
    monkeypatch.delenv('OSB_NO_GRAPH', raising=False)
    env_id, env_cfgs = ('SyntheticBox-v0', None) if env == 'synthetic' else _registered_env()
    narrow, wide = _pad_twin(tmp_path, prec, algo, env_id, env_cfgs)
    for a in (narrow, wide):
        a.learn()
    n, w = narrow.agent, wide.agent
    for k in ('obs', 'act', 'reward', 'cost', 'value_r', 'value_c', 'logp', 'adv_r', 'adv_c', 'target_value_r'):
        assert torch.equal(_bits(n._buf.data[k]), _bits(w._buf.data[k])), f'slab {k}'
    nac, wac = n._actor_critic, w._actor_critic
    for k in ('theta', 'adam_m', 'adam_v', 'adam_step'):
        assert torch.equal(_bits(getattr(nac, k)), _bits(getattr(wac, k))), k
    # acting: step / predict / log_prob / critics on the same rows and the same noise
    O = nac.obs_dim
    obs = torch.randn(333, O, generator=torch.Generator().manual_seed(2)).cuda()
    for call in (lambda m: m.step(obs, deterministic=True), lambda m: m.step(obs),
                 lambda m: (m.actor.predict(obs, deterministic=True), m.actor.log_prob(m.actor.predict(obs))),
                 lambda m: (m.reward_critic(obs)[0], m.cost_critic(obs)[0])):
        torch.manual_seed(7)
        got = call(nac)
        torch.manual_seed(7)
        want = call(wac)
        for x, y in zip(got, want):
            assert torch.equal(_bits(x), _bits(y))
    # evaluation of the saved checkpoints: upstream's shapes for the narrow run, 64-wide for the twin
    for a in (narrow, wide):
        a.evaluate(num_episodes=3)
    capsys.readouterr()
    ne, we = narrow._evaluator, wide._evaluator
    assert ne.episode_lengths == we.episode_lengths
    assert torch.equal(_bits(ne.last_actions), _bits(we.last_actions))
    assert torch.equal(_bits(ne._theta), _bits(we._theta))
    if env == 'synthetic':      # many envs at once, the persistent evaluation launch
        r1 = ne.evaluate(num_episodes=40, num_envs=16)
        r2 = we.evaluate(num_episodes=40, num_envs=16)
        capsys.readouterr()
        assert r1 == r2


@pytest.mark.timeout(900)
def test_narrow_resume_bitwise(cuda, tmp_path):
    from test_resume_gpu import _custom as resume_custom
    from test_resume_gpu import _load, _train_and_resume

    cfg = resume_custom(tmp_path)
    cfg['model_cfgs'] = {'actor': {'hidden_sizes': ACTOR}, 'critic': {'hidden_sizes': CRITIC}}
    _train_and_resume(tmp_path, 'PPOLag', 'SyntheticBox-v0', cfg)
    pi = _load(os.path.join(str(tmp_path), 'resumed', 'torch_save', 'epoch-4.pt'))['pi']
    assert tuple(pi['mean.0.weight'].shape) == (ACTOR[0], 60) and tuple(pi['mean.2.weight'].shape) == tuple(ACTOR[::-1])
