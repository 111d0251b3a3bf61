"""GPU: identity, relu, sigmoid and softplus hidden layers (model_cfgs.actor / critic.activation) on every kernel path.

- goldens of the unmodified reference (make_golden_activation.py; actor [24, 40], critic [8, 64], the 'softplus' case
  with relu critics): a rollout epoch, PPOLag._update, CPO's Fisher-vector product and CG, and CPO._update, at the bars
  of the tanh tests of the same widths (test_hidden_sizes_gpu.py); the rollout also in tf32 at its 5e-3;
- the full-batch actor evaluation (mu) of every precision against the reference actor's mean;
- the policy step fed the rollout's rows gives the rollout's actions, values and log-probabilities bit for bit;
- Evaluator on the synthetic env and on a registered env against the evaluation oracles, with the actor activation
  read from config.json; the graph replay of a graph-safe registered env equals the eager loop;
- sigmoid and softplus pads stay bitwise +0 (theta, Adam moments) through training: PPOLag, CPO, FOCOPS and a subclass
  training through `_loss_pi` and a critic hook;
- a non-tanh run resumed from a checkpoint lands on the uninterrupted run's bits;
- a relu model and a tanh model whose calls alternate in one process each give their solo results.
"""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from test_hidden_sizes_gpu import _assert_pads_zero, _bits, _registered_env  # noqa: E402

pytestmark = pytest.mark.gpu
PREC = {'fp32': 0, 'tf32': 1, 'bf16x3': 2}
TAGS = ['identity', 'relu', 'sigmoid', 'softplus']
FN = {'identity': lambda x: x, 'relu': torch.relu, 'sigmoid': torch.sigmoid, 'softplus': F.softplus, 'tanh': torch.tanh}


@pytest.fixture(autouse=True)
def _default_spec_after():
    """Launches made directly through the C ABI read the process-wide spec: leave the default (tanh, 64 wide) behind."""
    yield
    from omnisafe_b200.models.actor_critic import set_net_spec

    set_net_spec(0, 0, (64, 64), (64, 64))


def _model_cfgs(actor_act, critic_act, actor=(24, 40), critic=(8, 64), lr_actor=3e-4, lr_critic=3e-4):
    from types import SimpleNamespace as NS

    return NS(actor=NS(hidden_sizes=list(actor), activation=actor_act, lr=lr_actor),
              critic=NS(hidden_sizes=list(critic), activation=critic_act, lr=lr_critic),
              actor_type='gaussian_learning', linear_lr_decay=False, weight_initialization_mode='kaiming_uniform')


def _golden(golden_dir, name, tag):
    from omnisafe_b200.models import ParamMap

    g = np.load(os.path.join(golden_dir, f'{name}_act_{tag}.npz'))
    O, A = (int(g['O']), int(g['A'])) if 'O' in g.files else (12, 3)     # update_ppolag: make_golden.py's 12 x 3
    pmap = ParamMap(O, A, [int(x) for x in g['actor_hidden']], [int(x) for x in g['critic_hidden']])
    return g, pmap, O, A, str(g['actor_activation']), str(g['critic_activation'])


def _mlp(p, x, act, dtype):
    """Linear-act-Linear-act-Linear of reference-named parameters."""
    names = list(p)[-6:]
    h = torch.as_tensor(x, dtype=dtype)
    for layer in range(2):
        h = FN[act](F.linear(h, torch.as_tensor(p[names[2 * layer]]).to(dtype),
                             torch.as_tensor(p[names[2 * layer + 1]]).to(dtype)))
    return F.linear(h, torch.as_tensor(p[names[4]]).to(dtype), torch.as_tensor(p[names[5]]).to(dtype))


# ---- goldens of the unmodified reference ------------------------------------------------------------------------------
def _rollout(cuda, g, pmap, O, A, aa, ca, precision):
    """One rollout epoch of the golden's model, env and noise; returns the model, the adapter and the buffer."""
    from test_rollout_gpu import _cfgs

    from omnisafe_b200.adapter.onpolicy_adapter import OnPolicyAdapter
    from omnisafe_b200.common.buffer import VectorOnPolicyBuffer
    from omnisafe_b200.models import ConstraintActorCritic

    N, T = int(g['N']), int(g['T'])
    cfgs = _cfgs(True, 10, False, obs_dim=O, act_dim=A, max_episode_steps=int(g['tmax']), term_prob=float(g['term_prob']))
    ad = OnPolicyAdapter('SyntheticBox-v0', N, int(g['seed']), cfgs, device=cuda)
    ad.precision = precision
    agent = ConstraintActorCritic(O, A, _model_cfgs(aa, ca), epochs=1, device=cuda)
    agent.load_flat(pmap.to_kernel(g['theta']))
    buf = VectorOnPolicyBuffer(O, A, T, 0.99, 0.95, 0.95, 'gae', 0.0, True, True, num_envs=N, device=cuda)
    ad.rollout(T, agent, buf, eps=torch.as_tensor(g['eps']).to(cuda))
    torch.cuda.synchronize()
    return agent, ad, buf


@pytest.mark.parametrize('precision', [0, 1, 2])
@pytest.mark.parametrize('tag', TAGS)
def test_rollout_golden_reference(cuda, golden_dir, tag, precision):
    g, pmap, O, A, aa, ca = _golden(golden_dir, 'rollout_ppolag', tag)
    agent, ad, buf = _rollout(cuda, g, pmap, O, A, aa, ca, precision)
    sl = {k: v.cpu().numpy() for k, v in buf.data.items() if v is not None}
    tf32 = precision == 1      # test_rollout_gpu.py's tf32 bar: 5e-3 on values / actions, logp 2e-2
    t = dict(rtol=5e-3, atol=5e-3) if tf32 else dict(rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(sl['obs'], g['slab_obs'], **t)
    np.testing.assert_allclose(sl['act'], g['slab_act'], **t)
    np.testing.assert_allclose(sl['reward'], g['slab_reward'], **t)
    if tf32:      # 5e-3 of the samples, and at least one, may cross the cost threshold
        assert (sl['cost'] != g['slab_cost']).sum() <= max(1.0, 5e-3 * sl['cost'].size)
    else:
        assert np.array_equal(sl['cost'], g['slab_cost'])
    np.testing.assert_allclose(sl['value_r'], g['slab_value_r'], **t)
    np.testing.assert_allclose(sl['value_c'], g['slab_value_c'], **t)
    np.testing.assert_allclose(sl['logp'], g['slab_logp'], **(dict(rtol=5e-3, atol=2e-2) if tf32 else dict(rtol=2e-5, atol=5e-5)))
    if not tf32:
        nz = ad._obs_normalizer
        np.testing.assert_allclose(nz.mean.cpu().numpy(), g['norm_mean'], **t)
        np.testing.assert_allclose(nz.std.cpu().numpy(), g['norm_std'], **t)
        buf.finish_paths()
        torch.cuda.synchronize()
        np.testing.assert_allclose(buf.data['adv_r'].cpu().numpy(), g['slab_adv_r'], rtol=1e-4, atol=5e-5)
        np.testing.assert_allclose(buf.data['adv_c'].cpu().numpy(), g['slab_adv_c'], rtol=1e-4, atol=5e-5)


def _setup(dev, g, pmap, O, A, aa, ca, lr_actor=3e-4, lr_critic=3e-4):
    """test_hidden_sizes_gpu._setup with the case's activations."""
    from omnisafe_b200.algorithms.engine import UpdateEngine
    from omnisafe_b200.common.buffer import VectorOnPolicyBuffer
    from omnisafe_b200.models import ConstraintActorCritic

    N, T = 8, 24
    data = {k[5:]: g[k] for k in g.files if k.startswith('data_')}
    agent = ConstraintActorCritic(O, A, _model_cfgs(aa, ca, lr_actor=lr_actor, lr_critic=lr_critic), epochs=1, device=dev)
    agent.load_flat(pmap.to_kernel(g['theta0']))
    buf = VectorOnPolicyBuffer(O, A, T, 0.99, 0.95, 0.95, 'gae', 0.0, True, True, num_envs=N, device=dev)
    for k in ('obs', 'act', 'logp', 'adv_r', 'adv_c', 'target_value_r', 'target_value_c'):
        x = np.asarray(data[k], np.float32)
        buf.data[k].copy_(torch.as_tensor(x.reshape(N, T, *x.shape[1:]).swapaxes(0, 1).copy()).to(dev))
    buf.adv_moments.copy_(torch.tensor([0.0, 1.0, 0.0, 1.0]))
    return data, agent, buf, UpdateEngine(agent, buf)


@pytest.mark.parametrize('precision', [0, 2])
@pytest.mark.parametrize('tag', TAGS)
def test_ppolag_update_epoch_golden(cuda, golden_dir, tag, precision):
    from test_update_gpu import _rows

    from omnisafe_b200.common.lagrange import Lagrange

    g, pmap, O, A, aa, ca = _golden(golden_dir, 'update_ppolag', tag)
    N, T = 8, 24
    data, agent, buf, eng = _setup(cuda, g, pmap, O, A, aa, ca)
    eng.precision = precision
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


@pytest.mark.parametrize('precision', [0, 2])
@pytest.mark.parametrize('tag', TAGS)
def test_fvp_cg_golden(cuda, golden_dir, tag, precision):
    g, pmap, O, A, aa, ca = _golden(golden_dir, 'update_cpo', tag)
    data, agent, buf, eng = _setup(cuda, g, pmap, O, A, aa, ca, lr_actor=None, lr_critic=1e-3)
    eng.precision = precision
    Pa, Pa_ref = eng.Pa, pmap.ref['actor']['size']
    total_ref = pmap.ref['total']

    def to_kernel(v):
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


@pytest.mark.parametrize('prec', ['fp32', 'bf16x3'])
@pytest.mark.parametrize('tag', TAGS)
def test_cpo_update_golden(cuda, tmp_path, golden_dir, tag, prec):
    import omnisafe_b200

    g, pmap, O, A, aa, ca = _golden(golden_dir, 'update_cpo', tag)
    N, T = int(g['N']), int(g['T'])
    cfg = {
        'seed': int(g['seed']),
        'train_cfgs': {'device': 'cuda', 'vector_env_nums': N, 'total_steps': N * T * 2, 'matmul_precision': prec},
        'algo_cfgs': {'steps_per_epoch': N * T, 'batch_size': 32, 'update_iters': 2, 'cost_limit': float(g['cost_limit'])},
        'logger_cfgs': {'log_dir': str(tmp_path), 'window_lens': 10, 'use_tensorboard': False},
        'model_cfgs': {'actor': {'hidden_sizes': list(pmap.actor_hidden), 'activation': aa},
                       'critic': {'hidden_sizes': list(pmap.critic_hidden), 'activation': ca}},
        'env_cfgs': {'obs_dim': O, 'act_dim': A, 'max_episode_steps': 8, 'term_prob': 0.05},
    }
    algo = omnisafe_b200.Agent('CPO', 'SyntheticBox-v0', custom_cfgs=cfg).agent
    ac = algo._actor_critic
    assert ac.activation == (aa, ca)
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
    got, want = pmap.to_ref(ac.theta.cpu()).numpy(), g['theta1']
    bad = ~np.isclose(got, want, rtol=2e-3, atol=2e-5)
    assert bad.mean() < 1e-3 and np.abs(got - want).max() < 5e-3, (bad.sum(), np.abs(got - want).max())
    _assert_pads_zero(pmap, theta=ac.theta, adam_m=ac.adam_m, adam_v=ac.adam_v)


# ---- acting and evaluation --------------------------------------------------------------------------------------------
@pytest.mark.parametrize('prec', ['fp32', 'tf32', 'bf16x3'])
@pytest.mark.parametrize('tag', TAGS)
def test_actor_eval_mean_is_the_reference_actor(cuda, golden_dir, tag, prec):
    """osb_actor_eval / _tc / _x3 (the full-batch mu of the natural-gradient family) on the reference actor's rows."""
    from omnisafe_b200.algorithms.engine import UpdateEngine
    from omnisafe_b200.common.buffer import VectorOnPolicyBuffer
    from omnisafe_b200.models import ConstraintActorCritic

    g, pmap, O, A, aa, ca = _golden(golden_dir, 'evaluate_actor', tag)
    agent = ConstraintActorCritic(O, A, _model_cfgs(aa, ca, pmap.actor_hidden, pmap.critic_hidden), epochs=1, device=cuda)
    agent.param_map.load_state_dict(agent.theta, 'actor', {k[3:]: g[k] for k in g.files if k.startswith('pi_')})
    N, T = 8, 8
    buf = VectorOnPolicyBuffer(O, A, T, 0.99, 0.95, 0.95, 'gae', 0.0, True, True, num_envs=N, device=cuda)
    buf.data['obs'].copy_(torch.as_tensor(g['obs']).view(T, N, O))
    eng = UpdateEngine(agent, buf)
    eng.precision = PREC[prec]
    eng.snapshot_old_policy()
    torch.cuda.synchronize()
    t = dict(rtol=5e-3, atol=5e-3) if prec == 'tf32' else dict(rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(eng.mu_old.cpu().numpy().reshape(-1, A), g['mean'], **t)


@pytest.mark.parametrize('precision', [0, 1, 2])
@pytest.mark.parametrize('tag', TAGS)
def test_policy_step_gives_the_rollout_bits(cuda, golden_dir, tag, precision):
    """The rollout's rows and noise fed to the policy step: the rollout's actions, log-probabilities and values, bit for
    bit on the tensor-core tiles (one forward, csrc/tc_forward.cuh), within 2e-5 on the fp32 tiles."""
    g, pmap, O, A, aa, ca = _golden(golden_dir, 'rollout_ppolag', tag)
    agent, _, buf = _rollout(cuda, g, pmap, O, A, aa, ca, precision)
    agent.precision = precision
    eps = torch.as_tensor(g['eps']).to(cuda)
    d = buf.data
    for t in range(int(g['T'])):
        out = agent._launch(d['obs'][t].contiguous(), 7, eps=eps[t].contiguous(), act=True, logp=True)
        for k in ('act', 'logp', 'value_r', 'value_c'):
            if precision == 0:
                np.testing.assert_allclose(out[k].cpu().numpy(), d[k][t].cpu().numpy(), rtol=2e-5, atol=2e-5)
            else:
                assert torch.equal(_bits(out[k]), _bits(d[k][t])), (t, k)


def _eval_case(tmp, act, O, A, seed, env_id, env_cfgs, precision):
    from test_evaluate_gpu import random_case, write_run

    cfg, pi, norm = random_case(O, A, seed=seed)
    cfg['env_id'], cfg['env_cfgs'] = env_id, env_cfgs
    cfg['model_cfgs'] = {'actor': {'hidden_sizes': [64, 64], 'activation': act}}
    return write_run(tmp, cfg, pi, norm, precision), pi, norm


@pytest.mark.parametrize('precision', ['fp32', 'bf16x3'])
@pytest.mark.parametrize('act', TAGS)
def test_evaluate_synthetic_matches_oracle(cuda, tmp_path, act, precision, capsys):
    from oracle import evaluator as eval_oracle
    from omnisafe_b200 import Evaluator

    O, A, E, n = 60, 8, 256, 300
    env_cfgs = {'obs_dim': O, 'act_dim': A, 'max_episode_steps': 12, 'term_prob': 0.08, 'cost_threshold': 0.0}
    run, pi, norm = _eval_case(tmp_path, act, O, A, 7, 'SyntheticBox-v0', env_cfgs, precision)
    ev = Evaluator()
    ev.load_saved(run, 'epoch-0.pt')
    rets, costs = ev.evaluate(num_episodes=n, cost_criteria=0.99, num_envs=E)
    capsys.readouterr()
    r, c, ln, nz = eval_oracle.evaluate(pi, norm, env_cfgs, n, 0.99, num_envs=E,
                                        actor=lambda p, x: _mlp(p, x, act, torch.float32).numpy())
    np.testing.assert_array_equal(ev.episode_lengths, ln)
    np.testing.assert_allclose(rets, r, rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(costs, c, rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(ev.normalizer.mean.cpu().numpy(), nz.mean, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize('act', ['relu', 'softplus'])
def test_evaluate_registered_matches_oracle_and_graph_equals_eager(cuda, tmp_path, monkeypatch, act, capsys):
    import early_envs as ee
    import registered_eval_oracle as reg_oracle
    from test_evaluate_registered_cpu import WIDE, WIDE_COST_LIMIT, wide_box, wide_case
    from test_evaluate_gpu import write_run

    from omnisafe_b200 import Evaluator
    from omnisafe_b200.envs import CMDP, ENV_REGISTRY, Box, env_register

    ee.register(CMDP, Box, env_register, ENV_REGISTRY.support_envs())
    O, A, E = 45, WIDE['act_dim'], 64
    pi, norm = wide_case(O, A, seed=21)
    results = {}
    for graph, env_id in ((False, ee.RESET_WIDE_ID), (False, ee.GRAPH_RESET_WIDE_ID), (True, ee.GRAPH_RESET_WIDE_ID)):
        if graph:
            monkeypatch.delenv('OSB_NO_GRAPH', raising=False)
        else:
            monkeypatch.setenv('OSB_NO_GRAPH', '1')
        cfg = {'algo': 'PPOEarlyTerminated', 'env_id': env_id, 'env_cfgs': {**WIDE, 'obs_dim': O},
               'algo_cfgs': {'obs_normalize': True, 'cost_limit': WIDE_COST_LIMIT},
               'model_cfgs': {'actor': {'hidden_sizes': [64, 64], 'activation': act}}}
        ev = Evaluator()
        ev.load_saved(write_run(tmp_path / f'{env_id}-{graph}', cfg, pi, norm, 'bf16x3'), 'epoch-0.pt')
        rets, costs = ev.evaluate(num_episodes=2000 if graph or env_id == ee.GRAPH_RESET_WIDE_ID else 2 * E + 3,
                                  cost_criteria=0.99, num_envs=E)
        results[(graph, env_id)] = (rets, costs, ev.episode_lengths, ev.last_actions.cpu().numpy())
    capsys.readouterr()
    r, c, ln, _, _ = reg_oracle.evaluate(wide_box(E, O, A, WIDE['max_episode_steps']), pi, norm, 2 * E + 3, 0.99,
                                         cost_limit=WIDE_COST_LIMIT, actor=lambda p, x: _mlp(p, x, act, torch.float32).numpy())
    rets, costs, lens, _ = results[(False, ee.RESET_WIDE_ID)]
    np.testing.assert_array_equal(lens, ln)
    np.testing.assert_allclose(rets, r, rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(costs, c, rtol=1e-4, atol=1e-4)
    eager, graph = results[(False, ee.GRAPH_RESET_WIDE_ID)], results[(True, ee.GRAPH_RESET_WIDE_ID)]
    for x, y in zip(eager, graph):
        assert np.array_equal(np.asarray(x), np.asarray(y))


# ---- whole runs ---------------------------------------------------------------------------------------------------------
def _custom(tmp, act, prec='bf16x3', epochs=2, env_cfgs=None, algo=None):
    from test_hidden_sizes_gpu import _custom as hidden_custom

    cfg = hidden_custom(tmp, prec, epochs, env_cfgs, algo)
    cfg['model_cfgs']['actor']['activation'] = act[0]
    cfg['model_cfgs']['critic']['activation'] = act[1]
    return cfg


PAD_ACTS = [('sigmoid', 'sigmoid'), ('softplus', 'sigmoid')]


@pytest.mark.timeout(900)
@pytest.mark.parametrize('prec', list(PREC))
@pytest.mark.parametrize('act', PAD_ACTS)
@pytest.mark.parametrize('algo,env', [('PPOLag', 'synthetic'), ('CPO', 'synthetic'), ('FOCOPS', 'synthetic'),
                                      ('PPOLag', 'registered')])
def test_pads_stay_zero_through_training(cuda, tmp_path, monkeypatch, algo, env, act, prec):
    import omnisafe_b200

    monkeypatch.delenv('OSB_NO_GRAPH', raising=False)
    env_id, env_cfgs = ('SyntheticBox-v0', None) if env == 'synthetic' else _registered_env()
    agent = omnisafe_b200.Agent(algo, env_id, custom_cfgs=_custom(tmp_path, act, prec, 3, env_cfgs, algo))
    ac = agent.agent._actor_critic
    assert ac.activation == act
    theta0 = ac.theta.clone()
    agent.learn()
    assert torch.isfinite(ac.theta).all() and not torch.equal(ac.theta, theta0)
    _assert_pads_zero(ac.param_map, theta=ac.theta, adam_m=ac.adam_m, adam_v=ac.adam_v)


@pytest.mark.timeout(900)
@pytest.mark.parametrize('prec', list(PREC))
@pytest.mark.parametrize('act', PAD_ACTS)
def test_pads_stay_zero_with_torch_hooks(cuda, tmp_path, monkeypatch, act, prec):
    from test_torch_critic_gpu import _agent, _hook

    from omnisafe_b200.algorithms import registry

    base = registry.get('PPOLag')
    cls = type('UserPPOLag', (base,), {
        '_loss_pi': lambda self, o, a, lp, adv: base._loss_pi(self, o, a, lp, adv),
        '_update_reward_critic': _hook('huber', 'reward_critic')})
    agent = _agent(monkeypatch, 'PPOLag', cls, _custom(tmp_path, act, prec, 3))
    assert agent.agent._actor_hooks and agent.agent._critic_hooks
    ac = agent.agent._actor_critic
    theta0 = ac.theta.clone()
    agent.learn()
    assert torch.isfinite(ac.theta).all() and not torch.equal(ac.theta, theta0)
    _assert_pads_zero(ac.param_map, theta=ac.theta, adam_m=ac.adam_m, adam_v=ac.adam_v)


@pytest.mark.timeout(900)
@pytest.mark.parametrize('act', [('softplus', 'relu'), ('sigmoid', 'identity')])
def test_resume_bitwise(cuda, tmp_path, act):
    from test_resume_gpu import _custom as resume_custom
    from test_resume_gpu import _train_and_resume

    cfg = resume_custom(tmp_path)
    cfg['model_cfgs'] = {'actor': {'hidden_sizes': [24, 40], 'activation': act[0]},
                         'critic': {'hidden_sizes': [8, 64], 'activation': act[1]}}
    _train_and_resume(tmp_path, 'PPOLag', 'SyntheticBox-v0', cfg)


@pytest.mark.timeout(900)
def test_external_graph_replay_equals_eager(cuda, tmp_path, monkeypatch):
    """PPOLag with a softplus actor and relu critics on a graph-safe registered env: the epochs replayed from the CUDA
    graph give the eager run's bits."""
    import omnisafe_b200

    env_id, env_cfgs = _registered_env()
    runs = {}
    for mode in ('eager', 'graph'):
        if mode == 'eager':
            monkeypatch.setenv('OSB_NO_GRAPH', '1')
        else:
            monkeypatch.delenv('OSB_NO_GRAPH', raising=False)
        agent = omnisafe_b200.Agent('PPOLag', env_id, custom_cfgs=_custom(tmp_path / mode, ('softplus', 'relu'),
                                                                           'bf16x3', 3, env_cfgs, 'PPOLag'))
        agent.learn()
        assert agent.agent._env.graph_mode == mode
        runs[mode] = agent.agent
    e, g = runs['eager'], runs['graph']
    for k in ('theta', 'adam_m', 'adam_v'):
        assert torch.equal(_bits(getattr(e._actor_critic, k)), _bits(getattr(g._actor_critic, k))), k
    for k in ('obs', 'act', 'value_r', 'value_c', 'logp'):
        assert torch.equal(_bits(e._buf.data[k]), _bits(g._buf.data[k])), k


@pytest.mark.parametrize('prec', list(PREC))
def test_models_with_different_activations_alternate(cuda, prec):
    from omnisafe_b200.models import ConstraintActorCritic

    models = [ConstraintActorCritic(60, 8, _model_cfgs(a, c), epochs=1, device=cuda,
                                    generator=torch.Generator().manual_seed(3))
              for a, c in (('relu', 'relu'), ('tanh', 'tanh'), ('softplus', 'sigmoid'))]
    obs = torch.randn(1000, 60, generator=torch.Generator().manual_seed(1)).cuda()

    def calls(m):
        m.precision = PREC[prec]
        torch.manual_seed(5)
        out = list(m.step(obs))
        out.append(m.actor.predict(obs, deterministic=True))
        out.append(m.reward_critic(obs)[0])
        return [_bits(x) for x in out]

    solo = [calls(m) for m in models]
    assert not all(torch.equal(x, y) for x, y in zip(solo[0], solo[1]))      # the activations reach the kernels
    for _ in range(2):
        for m, want in zip(models, solo):
            for x, y in zip(calls(m), want):
                assert torch.equal(x, y)
