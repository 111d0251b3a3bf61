"""GPU parity: fused minibatch forward/backward, optimiser, KL evaluation, Lagrange multiplier,
Fisher-vector product and CG vs the oracle and vs golden fixtures of the unmodified reference."""
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from oracle import actor_critic as oac
from oracle import learner as ol

pytestmark = pytest.mark.gpu


def _model_cfgs(lr_actor=3e-4, lr_critic=3e-4):
    return NS(actor=NS(hidden_sizes=[64, 64], activation='tanh', lr=lr_actor),
              critic=NS(hidden_sizes=[64, 64], activation='tanh', lr=lr_critic),
              actor_type='gaussian_learning', linear_lr_decay=False, weight_initialization_mode='kaiming_uniform')


def _setup(dev, data, N, T, O, A, theta, lr_actor=3e-4, lr_critic=3e-4):
    """Build agent + slab buffer from env-major `data` (as VectorOnPolicyBuffer.get() returns it)."""
    from omnisafe_b200.algorithms.engine import UpdateEngine
    from omnisafe_b200.common.buffer import VectorOnPolicyBuffer
    from omnisafe_b200.models import ConstraintActorCritic

    agent = ConstraintActorCritic(O, A, _model_cfgs(lr_actor, lr_critic), epochs=1, device=dev)
    agent.load_flat(theta)
    buf = VectorOnPolicyBuffer(O, A, T, 0.99, 0.95, 0.95, 'gae', 0.0, True, True, num_envs=N, device=dev)

    def tm(x):  # env-major [N*T, ...] -> time-major [T, N, ...]
        x = np.asarray(x, np.float32)
        return torch.as_tensor(x.reshape(N, T, *x.shape[1:]).swapaxes(0, 1).copy()).to(dev)

    for k_slab, k_data in (('obs', 'obs'), ('act', 'act'), ('logp', 'logp'), ('adv_r', 'adv_r'),
                           ('adv_c', 'adv_c'), ('target_value_r', 'target_value_r'),
                           ('target_value_c', 'target_value_c')):
        buf.data[k_slab].copy_(tm(data[k_data]))
    # `data` already holds standardised advantages: identity moments
    buf.adv_moments.copy_(torch.tensor([0.0, 1.0, 0.0, 1.0]))
    return agent, buf, UpdateEngine(agent, buf)


def _rows(perm_env_major, N, T):
    k = np.asarray(perm_env_major, np.int64)
    return ((k % T) * N + (k // T)).astype(np.int32)


def sigma_cases(unit, trained):
    """Parameter sets of a test at the reference's initial log_std = 0 (`unit`, under their usual ids) and at a trained
    log_std (`trained`, oracle.actor_critic.trained_log_std; ids end in '-trained'): the last argument is the flag."""
    return ([pytest.param(*c, False, id='-'.join(map(str, c))) for c in unit]
            + [pytest.param(*c, True, id='-'.join(map(str, c)) + '-trained') for c in trained])


def entropy_mean(log_std):
    """Mean entropy of the Gaussian policy over samples and action dims: 0.5 + 0.5 log 2 pi + mean_a log sigma_a."""
    return 0.5 + 0.5 * np.log(2 * np.pi) + float(np.mean(np.asarray(log_std, np.float64)))


def _theta(O, A, seed, trained):
    return oac.init_theta(O, A, seed=seed, log_std=oac.trained_log_std(A, seed) if trained else None)


def _rand_data(rng, N, T, O, A, theta):
    B = N * T
    obs = rng.standard_normal((B, O)).astype(np.float32)
    eps = rng.standard_normal((B, A)).astype(np.float32)
    act, v_r, v_c, logp = oac.step(theta, obs, eps, O, A)
    logp = (logp + 0.3 * rng.standard_normal(B)).astype(np.float32)   # push ratios across the clip range
    return {'obs': obs, 'act': act, 'logp': logp,
            'adv_r': rng.standard_normal(B).astype(np.float32), 'adv_c': rng.standard_normal(B).astype(np.float32),
            'target_value_r': rng.standard_normal(B).astype(np.float32),
            'target_value_c': rng.standard_normal(B).astype(np.float32)}


@pytest.mark.parametrize('O,A,N,T,loss_kind,trained', sigma_cases(
    [(60, 8, 20, 13, 0), (60, 8, 32, 8, 1), (17, 6, 9, 31, 3), (111, 8, 16, 10, 0), (376, 8, 7, 20, 0)],
    # ragged last tile, A = 1, A = 16 with more tiles than CTAs, obs dims > 64; every single-pass kind
    [(60, 8, 20, 13, 0), (17, 6, 9, 31, 3), (33, 1, 50, 11, 0), (64, 16, 300, 70, 1), (111, 8, 16, 10, 1)]))
def test_minibatch_grad_vs_autograd(cuda, O, A, N, T, loss_kind, trained):
    from omnisafe_b200._lib import current_stream, lib, ptr

    rng = np.random.default_rng(O + N)
    theta = _theta(O, A, 5, trained)
    data = _rand_data(rng, N, T, O, A, theta)
    agent, buf, eng = _setup(cuda, data, N, T, O, A, theta)
    B = N * T
    lam = 0.37
    lag = torch.tensor([lam], dtype=torch.float32, device=cuda)
    perm_em = rng.permutation(B)
    start, count = 3, B - 10
    perm = torch.as_tensor(_rows(perm_em, N, T)).to(cuda)
    coef = 1e-3
    d = buf.data
    lib().osb_minibatch_grad(ptr(agent.theta), O, A, ptr(d['obs']), ptr(d['act']), ptr(d['logp']),
                             ptr(d['adv_r']), ptr(d['adv_c']), ptr(d['target_value_r']), ptr(d['target_value_c']),
                             0, ptr(buf.adv_moments), ptr(perm), B, 0, start, count, loss_kind, 0.2, 0.01,
                             1.0, 0.0, ptr(lag), 0, 7, ptr(eng.gpart), ptr(eng.stats_part), 0, current_stream())
    nb = lib().osb_update_grid_blocks(count)
    lib().osb_grad_reduce(ptr(eng.gpart), ptr(eng.stats_part), nb, O, A, ptr(agent.theta), ptr(agent.grad),
                          coef, 7, ptr(eng.sumsq_part), ptr(agent.adam_step), ptr(eng.train_stats), 0,
                          current_stream())
    torch.cuda.synchronize()
    got = agent.grad.cpu().numpy()
    # oracle autograd
    L = ol.Learner(theta, O, A)
    idx = torch.as_tensor(perm_em[start:start + count])
    t = {k: torch.as_tensor(v)[idx] for k, v in data.items()}
    adv = (t['adv_r'] - lam * t['adv_c']) / (1 + lam)
    if loss_kind == 0:
        loss, _ = L.loss_pi_ppo(t['obs'], t['act'], t['logp'], adv, 0.2, 0.01)
    elif loss_kind == 1:
        loss = L.loss_pi_plain(t['obs'], t['act'], t['logp'], adv)
    else:
        loss = L.loss_pi_cost(t['obs'], t['act'], t['logp'], t['adv_c'])
    loss.backward()
    for net, tgt in (('reward_critic', 'target_value_r'), ('cost_critic', 'target_value_c')):
        lv = torch.nn.functional.mse_loss(oac.critic_value(L.params[net], t['obs']), t[tgt])
        for p_ in L.params[net].values():
            lv = lv + p_.pow(2).sum() * coef
        lv.backward()
    want = torch.cat([L.flat_grad(n) for n in ol.NETS]).numpy()
    lay = oac.layout(O, A)
    for net in ol.NETS:
        s, n = lay[net]['start'], lay[net]['size']
        scale = np.abs(want[s:s + n]).max()
        np.testing.assert_allclose(got[s:s + n], want[s:s + n], rtol=2e-4, atol=2e-5 * max(scale, 1e-3), err_msg=net)
    # the log_std block on its own (A entries next to ~10^4 weights in the actor's bar)
    rel = float(np.linalg.norm(got[:A] - want[:A]) / np.linalg.norm(want[:A]))
    print(f'actor.log_std: l2-rel {rel:.2e}')
    assert rel < 1e-4, rel
    np.testing.assert_allclose(got[:A], want[:A], rtol=2e-4, atol=2e-5 * np.abs(want[:A]).max(), err_msg='log_std')
    # slot 0: the loss without the entropy bonus; slot 4: the bonus; Loss/Loss_pi = slot 0 + slot 4 is the oracle loss,
    # bonus included (base/ppo.py:L76-84)
    ts = eng.train_stats.cpu().numpy().reshape(3, 8)
    bonus = -0.01 * entropy_mean(theta[:A]) if loss_kind == 0 else 0.0
    np.testing.assert_allclose(ts[0, 0], float(loss) - bonus, rtol=1e-3, atol=1e-4)
    np.testing.assert_allclose(ts[0, 4], bonus, rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(ts[0, 0] + ts[0, 4], float(loss), rtol=1e-3, atol=1e-4)


def test_ppolag_update_epoch_golden(cuda, golden_dir):
    """Same data / minibatch order / lambda as the unmodified PPOLag._update -> same parameters."""
    from omnisafe_b200.common.lagrange import Lagrange

    g = np.load(os.path.join(golden_dir, 'update_ppolag.npz'))
    data = {k[5:]: g[k] for k in g.files if k.startswith('data_')}
    N, T, O, A = 8, 24, 12, 3
    agent, buf, eng = _setup(cuda, data, N, T, O, A, g['theta0'])
    lag = Lagrange(float(g['cost_limit']), float(g['lam0']), float(g['lambda_lr']), device=cuda)
    ws = torch.tensor([0.0, float(g['Jc']) * 10, 0.0, 10.0], dtype=torch.float64, device=cuda)
    lag.update_lagrange_multiplier(ws)
    torch.cuda.synchronize()
    assert abs(float(lag.lagrangian_multiplier) - float(g['lam1'])) < 1e-6
    perms = torch.as_tensor(np.stack([_rows(p_, N, T) for p_ in g['perms'][::2]])).to(cuda)
    eng.ppo_epoch(loss_kind=0, lagrange=lag.state, net_mask=7, batch_size=int(g['batch_size']),
                  update_iters=int(g['update_iters']), clip=0.2, entropy_coef=0.0, critic_norm_coef=0.001,
                  max_grad_norm=40.0, lr_actor=3e-4, lr_critic=3e-4, target_kl=0.02, kl_early_stop=True,
                  perm=perms)
    torch.cuda.synchronize()
    got, want = agent.theta.cpu().numpy(), g['theta1']
    bad = ~np.isclose(got, want, rtol=2e-4, atol=2e-6)   # see test_cpo_update_golden on Adam + tiny grads
    assert bad.mean() < 1e-3 and np.abs(got - want).max() < 2e-3, (bad.sum(), np.abs(got - want).max())
    kls = eng.kl_state.cpu().numpy()
    np.testing.assert_allclose(kls[0], g['kl'][-1], rtol=2e-3, atol=1e-6)
    assert int(kls[1]) == int(g['stop_iter'][-1])
    ts = eng.train_stats.cpu().numpy().reshape(3, 8)
    np.testing.assert_allclose(ts[0, 0] / ts[0, 3], g['loss_pi'].mean(), rtol=1e-3, atol=1e-5)
    np.testing.assert_allclose(ts[1, 0] / ts[1, 3], g['loss_r'].mean(), rtol=1e-3, atol=1e-5)


def test_update_epoch_vs_oracle_early_stop_and_feistel(cuda):
    """(a) parity-mode epoch vs oracle incl. KL early stop; (b) the in-kernel Feistel order is a
    permutation: one full pass with batch == total equals the identity-order pass."""
    rng = np.random.default_rng(3)
    N, T, O, A = 16, 12, 60, 8
    theta = oac.init_theta(O, A, seed=2)
    data = _rand_data(rng, N, T, O, A, theta)
    B = N * T
    perms_em = np.stack([rng.permutation(B) for _ in range(4)])
    L = ol.Learner(theta, O, A, lr_actor=3e-3, lr_critic=1e-3)
    st = L.update_ppo(data, perms_em, 0.2, batch_size=64, target_kl=0.02, kl_early_stop=True)
    agent, buf, eng = _setup(cuda, data, N, T, O, A, theta)
    lag = torch.tensor([0.2, 0, 0, 0], dtype=torch.float32, device=cuda)
    perms = torch.as_tensor(np.stack([_rows(p_, N, T) for p_ in perms_em])).to(cuda)
    kw = dict(loss_kind=0, lagrange=lag, net_mask=7, clip=0.2, critic_norm_coef=0.001, max_grad_norm=40.0,
              lr_actor=3e-3, lr_critic=1e-3, target_kl=0.02, kl_early_stop=True)
    eng.ppo_epoch(batch_size=64, update_iters=4, perm=perms, **kw)
    torch.cuda.synchronize()
    assert st['iters'] < 4, 'test should exercise the early stop'
    assert int(eng.kl_state.cpu()[1]) == st['iters']
    got, want = agent.theta.cpu().numpy(), L.flat()
    bad = ~np.isclose(got, want, rtol=5e-4, atol=5e-6)
    assert bad.mean() < 1e-3 and np.abs(got - want).max() < 2e-2, (bad.sum(), np.abs(got - want).max())
    # (b) Feistel: full-batch pass is order independent
    a1, _, e1 = _setup(cuda, data, N, T, O, A, theta)
    a2, _, e2 = _setup(cuda, data, N, T, O, A, theta)
    ident = torch.arange(B, dtype=torch.int32, device=cuda)[None]
    e1.ppo_epoch(batch_size=B, update_iters=1, perm=ident, **kw)
    e2.ppo_epoch(batch_size=B, update_iters=1, perm=None, **kw)
    torch.cuda.synchronize()
    np.testing.assert_allclose(a1.theta.cpu().numpy(), a2.theta.cpu().numpy(), rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize('precision', [0, 2])      # exact fp32 FMA tiles / split-bf16 tensor-core tiles: same bar
def test_fvp_cg_eval_golden(cuda, golden_dir, precision):
    g = np.load(os.path.join(golden_dir, 'update_cpo.npz'))
    data = {k[5:]: g[k] for k in g.files if k.startswith('data_')}
    N, T, O, A = int(g['N']), int(g['T']), int(g['O']), int(g['A'])
    agent, buf, eng = _setup(cuda, data, N, T, O, A, g['theta0'], lr_actor=None, lr_critic=1e-3)
    eng.precision = precision
    vec = torch.as_tensor(g['vec']).to(cuda)
    out = torch.zeros_like(vec)
    eng.fvp(vec, out, float(g['cg_damping']))
    torch.cuda.synchronize()
    np.testing.assert_allclose(out.cpu().numpy(), g['fvp'], rtol=2e-4, atol=2e-6)
    x = eng.conjugate_gradients(torch.as_tensor(g['bvec']).to(cuda), int(g['cg_iters']), float(g['cg_damping']))
    torch.cuda.synchronize()
    np.testing.assert_allclose(x.cpu().numpy(), g['xcg'], rtol=5e-3, atol=2e-5)
    # evaluation of the unchanged policy: KL == 0, ratio == 1, surrogates == plain means
    eng.snapshot_old_policy()
    ev = eng.evaluate(agent.theta, None)
    assert abs(ev['kl']) < 1e-9 and abs(ev['ratio'] - 1.0) < 1e-5
    np.testing.assert_allclose(ev['loss_r'], -data['adv_r'].mean(), rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(ev['loss_c'], data['adv_c'].mean(), rtol=1e-4, atol=1e-6)
    # evaluation of a perturbed policy vs the oracle
    L = ol.Learner(g['theta0'], O, A, lr_actor=None)
    th2 = agent.theta.clone()
    th2[: eng.Pa] += 0.01 * torch.as_tensor(g['vec']).to(cuda)
    ev2 = eng.evaluate(th2, None)
    old = L.dist(torch.as_tensor(data['obs']))
    old = torch.distributions.Normal(old.loc.detach().clone(), old.scale.detach().clone())
    L.set_flat('actor', L.flat('actor') + 0.01 * g['vec'])
    with torch.no_grad():
        new = L.dist(torch.as_tensor(data['obs']))
        kl = torch.distributions.kl_divergence(old, new).mean().item()
        lr_ = L.loss_pi_plain(torch.as_tensor(data['obs']), torch.as_tensor(data['act']), torch.as_tensor(data['logp']),
                              torch.as_tensor(data['adv_r'])).item()
    np.testing.assert_allclose(ev2['kl'], kl, rtol=1e-3, atol=1e-8)
    np.testing.assert_allclose(ev2['loss_r'], lr_, rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize('precision', [0, 2])      # exact fp32 FMA tiles / split-bf16 tensor-core tiles (stepwise launches): same bar
def test_focops_update_epoch_golden(cuda, golden_dir, precision):
    """FOCOPS on the device (incl. the reference's broadcast quirk, via the forward-only mask pass)
    vs the unmodified FOCOPS._update: same parameters afterwards."""
    g = np.load(os.path.join(golden_dir, 'update_focops.npz'))
    data = {k[5:]: g[k] for k in g.files if k.startswith('data_')}
    N, T, O, A = int(g['N']), int(g['T']), int(g['O']), int(g['A'])
    agent, buf, eng = _setup(cuda, data, N, T, O, A, g['theta0'])
    eng.precision = precision
    lag = torch.tensor([float(g['lam1']), 0, 0, 0], dtype=torch.float32, device=cuda)
    perms = torch.as_tensor(np.stack([_rows(p_, N, T) for p_ in g['perms'][::2]])).to(cuda)
    eng.ppo_epoch(loss_kind=2, lagrange=lag, net_mask=7, batch_size=int(g['batch_size']),
                  update_iters=int(g['update_iters']), entropy_coef=0.0, focops_lam=float(g['focops_lam']),
                  focops_eta=float(g['focops_eta']), critic_norm_coef=0.001, max_grad_norm=40.0, lr_actor=3e-4,
                  lr_critic=3e-4, target_kl=0.02, kl_early_stop=True, perm=perms)
    torch.cuda.synchronize()
    got, want = agent.theta.cpu().numpy(), g['theta1']
    bad = ~np.isclose(got, want, rtol=2e-4, atol=2e-6)
    assert bad.mean() < 1e-3 and np.abs(got - want).max() < 2e-3, (bad.sum(), np.abs(got - want).max())
    np.testing.assert_allclose(float(eng.kl_state[0]), g['kl'][-1], rtol=2e-3, atol=1e-6)
    ts = eng.train_stats.cpu().numpy().reshape(3, 8)
    np.testing.assert_allclose(ts[0, 0] / ts[0, 3], g['loss_pi'].mean(), rtol=2e-3, atol=1e-5)


@pytest.mark.parametrize('precision', [0, 2])
def test_p3o_update_epoch_golden(cuda, golden_dir, precision):
    """P3O on the device (forward-only pass for the minibatch-mean relu gate) vs the unmodified
    P3O._update: same parameters afterwards."""
    g = np.load(os.path.join(golden_dir, 'update_p3o.npz'))
    data = {k[5:]: g[k] for k in g.files if k.startswith('data_')}
    N, T, O, A = int(g['N']), int(g['T']), int(g['O']), int(g['A'])
    agent, buf, eng = _setup(cuda, data, N, T, O, A, g['theta0'])
    eng.precision = precision
    perms = torch.as_tensor(np.stack([_rows(p_, N, T) for p_ in g['perms'][::2]])).to(cuda)
    eng.ppo_epoch(loss_kind=5, lagrange=None, net_mask=7, batch_size=int(g['batch_size']),
                  update_iters=int(g['update_iters']), clip=0.2, entropy_coef=0.0, focops_lam=float(g['kappa']),
                  focops_eta=float(g['Jc']) - float(g['cost_limit']), critic_norm_coef=0.001, max_grad_norm=40.0,
                  lr_actor=3e-4, lr_critic=3e-4, target_kl=0.02, kl_early_stop=True, perm=perms)
    torch.cuda.synchronize()
    got, want = agent.theta.cpu().numpy(), g['theta1']
    bad = ~np.isclose(got, want, rtol=2e-4, atol=2e-6)
    assert bad.mean() < 1e-3 and np.abs(got - want).max() < 2e-3, (bad.sum(), np.abs(got - want).max())
    np.testing.assert_allclose(float(eng.kl_state[0]), g['kl'][-1], rtol=2e-3, atol=1e-6)
    ts = eng.train_stats.cpu().numpy().reshape(3, 8)
    np.testing.assert_allclose(ts[0, 0] / ts[0, 3], g['loss_pi'].mean(), rtol=2e-3, atol=1e-5)
    np.testing.assert_allclose(ts[0, 2] / ts[0, 3], g['loss_pi_cost'].mean(), rtol=2e-3, atol=1e-5)


@pytest.mark.parametrize('jc_minus_limit', [-5.0, 0.3])
@pytest.mark.parametrize('tc', [0, 1])
def test_p3o_gate_vs_autograd(cuda, jc_minus_limit, tc):
    """Both states of the relu gate (inactive: plain PPO-clip gradient; active: + kappa d mean(ratio adv_c)),
    fp32 tiles and wgmma tiles, against autograd of the oracle loss."""
    from omnisafe_b200._lib import current_stream, lib, ptr

    N, T, O, A = 40, 25, 60, 8
    rng = np.random.default_rng(17)
    theta = oac.init_theta(O, A, seed=6)
    data = _rand_data(rng, N, T, O, A, theta)
    agent, buf, eng = _setup(cuda, data, N, T, O, A, theta)
    B = N * T
    perm_em = rng.permutation(B)
    perm = torch.as_tensor(_rows(perm_em, N, T)).to(cuda)
    kappa = 0.7
    d = buf.data
    fn = lib().osb_minibatch_grad_tc if tc else lib().osb_minibatch_grad
    nb = lib().osb_tc_grid_blocks(B, 1) if tc else lib().osb_update_grid_blocks(B)
    fn(ptr(agent.theta), O, A, ptr(d['obs']), ptr(d['act']), ptr(d['logp']), ptr(d['adv_r']), ptr(d['adv_c']),
       ptr(d['target_value_r']), ptr(d['target_value_c']), ptr(eng.mu_old), ptr(buf.adv_moments), ptr(perm), B, 0,
       0, B, 5, 0.2, 0.0, kappa, jc_minus_limit, 0, ptr(eng.logstd_old), 1, ptr(eng.gpart), ptr(eng.stats_part), 0,
       current_stream())
    lib().osb_grad_reduce(ptr(eng.gpart), ptr(eng.stats_part), nb, O, A, ptr(agent.theta), ptr(agent.grad), 0.0, 1,
                          ptr(eng.sumsq_part), ptr(agent.adam_step), ptr(eng.train_stats), 0, current_stream())
    torch.cuda.synchronize()
    got = agent.grad.cpu().numpy()[: eng.Pa]
    L = ol.Learner(theta, O, A)
    t = {k: torch.as_tensor(v) for k, v in data.items()}
    loss, _ = L.loss_pi_p3o(t['obs'], t['act'], t['logp'], t['adv_r'], t['adv_c'], 0.2, kappa, jc_minus_limit)
    loss.backward()
    want = L.flat_grad('actor').numpy()
    rel = np.linalg.norm(got - want) / np.linalg.norm(want)
    cos = float((got * want).sum() / (np.linalg.norm(got) * np.linalg.norm(want)))
    # TF32 tiles: samples within ~5e-4 of the clip boundary flip branch; on 1000 samples that bounds the
    # agreement at a few per cent (the direction stays the same)
    assert (rel < 1e-1 and cos > 0.995) if tc else rel < 1e-4, (rel, cos)
    np.testing.assert_allclose(float(eng.train_stats[0] + eng.train_stats[2]), float(loss), rtol=5e-3 if tc else 1e-4, atol=1e-5)
