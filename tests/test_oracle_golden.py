"""Pin the CPU oracle against (a) the reference's own known-answer tests and (b) golden fixtures
produced by the unmodified reference (tests/golden/make_golden.py)."""
import os

import numpy as np
import pytest

from oracle import actor_critic as oac
from oracle import gae as ogae
from oracle import rollout as orollout
from oracle.normalizer import Normalizer
from oracle.synthetic_env import SyntheticBoxEnv


def test_discount_cumsum_reference_known_answers():
    # reference tests/test_utils.py:L95-115
    x = np.array([1, 2, 3, 4, 5], np.float64)
    np.testing.assert_allclose(ogae.discount_cumsum(x, 0.9), [11.4265, 11.5850, 10.65, 8.5, 5.0], rtol=1e-5, atol=1e-8)
    np.testing.assert_allclose(ogae.discount_cumsum(x, 0.99), [14.6045, 13.7419, 11.8605, 8.95, 5.0], rtol=1e-5, atol=1e-8)
    np.testing.assert_allclose(ogae.discount_cumsum(x, 0.999), [14.9600, 13.9740, 11.9860, 8.9950, 5.0], rtol=1e-5, atol=1e-4)


def test_discount_cumsum_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, 'discount_cumsum.npz'))
    for i in range(int(g['n'])):
        y = ogae.discount_cumsum(g[f'x{i}'], float(g[f'd{i}']))
        assert np.array_equal(y, g[f'y{i}']), f'vector {i} not bit-identical to the reference'


def test_buffer_gae_golden_bit_exact(golden_dir):
    g = np.load(os.path.join(golden_dir, 'buffer_gae.npz'))
    out = ogae.dual_gae_slab(g['rew'], g['cost'], g['val_r'], g['val_c'], g['flags'], g['boot_r'],
                             g['boot_c'], float(g['gamma']), float(g['lam']), float(g['lam_c']),
                             float(g['pen']))
    for ours, ref in (('adv_r', 'raw_adv_r'), ('adv_c', 'raw_adv_c'), ('tv_r', 'raw_target_value_r'),
                      ('tv_c', 'raw_target_value_c'), ('disc_ret', 'raw_discounted_ret')):
        assert np.array_equal(out[ours], g[ref]), f'{ours} differs from the reference buffer'
    # get(): env-major order + standardisation
    T, N = g['rew'].shape
    sr, sc = ogae.standardize(out['adv_r'], out['adv_c'])
    em = lambda x: x.T.reshape(T * N, *x.shape[2:]) if x.ndim == 2 else x.transpose(1, 0, 2).reshape(T * N, -1)
    np.testing.assert_allclose(em(sr), g['get_adv_r'], rtol=2e-6, atol=2e-6)
    np.testing.assert_allclose(em(sc), g['get_adv_c'], rtol=2e-6, atol=2e-6)
    assert np.array_equal(em(out['tv_r']), g['get_target_value_r'])
    assert np.array_equal(em(g['obs']), g['get_obs'])


def test_buffer_other_estimators_golden_bit_exact(golden_dir):
    """'gae-rtg' / 'plain' / 'vtrace' (onpolicy_buffer.py:L305-331, L338-405) of the per-path oracle vs the
    reference buffer."""
    for fname in ('buffer_gae_rtg.npz', 'buffer_plain.npz', 'buffer_vtrace.npz'):
        g = np.load(os.path.join(golden_dir, fname))
        out = ogae.dual_gae_per_path(g['rew'], g['cost'], g['val_r'], g['val_c'], g['flags'], g['boot_r'],
                                     g['boot_c'], float(g['gamma']), float(g['lam']), float(g['lam_c']),
                                     float(g['pen']), estimator=str(g['estimator']))
        for ours, ref in (('adv_r', 'raw_adv_r'), ('adv_c', 'raw_adv_c'), ('tv_r', 'raw_target_value_r'),
                          ('tv_c', 'raw_target_value_c'), ('disc_ret', 'raw_discounted_ret')):
            assert np.array_equal(out[ours], g[ref]), f'{fname}: {ours} differs from the reference buffer'


def test_normalizer_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, 'normalizer.npz'))
    norm = Normalizer((5,))
    for i in range(int(g['nb'])):
        y = norm.normalize(g[f'x{i}'])
        np.testing.assert_allclose(norm.mean, g[f'mean{i}'], rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(norm.std, g[f'std{i}'], rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(y, g[f'y{i}'], rtol=1e-5, atol=1e-5)


def test_rollout_golden(golden_dir):
    """Oracle rollout == unmodified OnPolicyAdapter.rollout + buffer on the synthetic env."""
    g = np.load(os.path.join(golden_dir, 'rollout_ppolag.npz'))
    N, T, O, A = int(g['N']), int(g['T']), int(g['O']), int(g['A'])
    env = SyntheticBoxEnv(N, O, A, max_episode_steps=int(g['tmax']), seed=int(g['seed']),
                          term_prob=float(g['term_prob']))
    norm = Normalizer((O,))
    window = []
    sl = orollout.rollout_epoch(env, norm, g['theta'], T, g['eps'], window=window)
    tol = dict(rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(sl['obs'], g['slab_obs'], **tol)
    np.testing.assert_allclose(sl['act'], g['slab_act'], **tol)
    np.testing.assert_allclose(sl['rew'], g['slab_reward'], **tol)
    assert np.array_equal(sl['cost'], g['slab_cost'])
    np.testing.assert_allclose(sl['val_r'], g['slab_value_r'], **tol)
    np.testing.assert_allclose(sl['val_c'], g['slab_value_c'], **tol)
    np.testing.assert_allclose(sl['logp'], g['slab_logp'], rtol=1e-5, atol=2e-5)
    np.testing.assert_allclose(norm.mean, g['norm_mean'], **tol)
    np.testing.assert_allclose(norm.std, g['norm_std'], **tol)
    assert norm.count == int(g['norm_count'])
    out = ogae.dual_gae_slab(sl['rew'], sl['cost'], sl['val_r'], sl['val_c'], sl['flags'],
                             sl['boot_r'], sl['boot_c'], float(g['gamma']), float(g['lam']), float(g['lam_c']))
    np.testing.assert_allclose(out['adv_r'], g['slab_adv_r'], rtol=1e-4, atol=2e-5)
    np.testing.assert_allclose(out['adv_c'], g['slab_adv_c'], rtol=1e-4, atol=2e-5)
    np.testing.assert_allclose(out['tv_r'], g['slab_target_value_r'], rtol=1e-4, atol=2e-5)
    np.testing.assert_allclose(out['disc_ret'], g['slab_discounted_ret'], rtol=1e-4, atol=2e-5)
    # Logger window (maxlen 10): last finished episodes in (step, env) order
    w = np.array(window[-10:], np.float32)
    np.testing.assert_allclose(w[:, 0], g['win_ret'], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(w[:, 1], g['win_cost'])
    np.testing.assert_allclose(w[:, 2], g['win_len'])


def trained_golden(golden_dir, A):
    """One action dimension of rollout_ppolag_trained.npz (tests/golden/make_golden_trained_std.py) as a dict."""
    g = np.load(os.path.join(golden_dir, 'rollout_ppolag_trained.npz'))
    return {k[len(f'A{A}_'):]: g[k] for k in g.files if k.startswith(f'A{A}_')}


def _check_slabs(sl, g, tol):
    t = dict(rtol=tol, atol=tol)
    np.testing.assert_allclose(sl['obs'], g['slab_obs'], **t)
    np.testing.assert_allclose(sl['act'], g['slab_act'], **t)
    np.testing.assert_allclose(sl['rew'], g['slab_reward'], **t)
    assert np.array_equal(sl['cost'], g['slab_cost'])
    np.testing.assert_allclose(sl['val_r'], g['slab_value_r'], **t)
    np.testing.assert_allclose(sl['val_c'], g['slab_value_c'], **t)
    np.testing.assert_allclose(sl['logp'], g['slab_logp'], rtol=tol, atol=max(tol, 2e-5))


@pytest.mark.parametrize('A', [3, 9])
def test_rollout_golden_trained_std(golden_dir, A):
    """Oracle rollout == the unmodified reference with the actor's log_std at trained_log_std(A): sigma differs per
    action, so each action's sigma, 2 sigma^2 and log sigma reach the slabs."""
    g = trained_golden(golden_dir, A)
    N, T, O = int(g['N']), int(g['T']), int(g['O'])
    assert int(g['A']) == A
    theta = g['theta']
    np.testing.assert_array_equal(theta[:A], oac.trained_log_std(A))
    env = SyntheticBoxEnv(N, O, A, max_episode_steps=int(g['tmax']), seed=int(g['seed']), term_prob=float(g['term_prob']))
    norm, window = Normalizer((O,)), []
    sl = orollout.rollout_epoch(env, norm, theta, T, g['eps'], window=window)
    _check_slabs(sl, g, 1e-5)
    np.testing.assert_allclose(norm.mean, g['norm_mean'], rtol=1e-5, atol=1e-5)
    assert norm.count == int(g['norm_count'])
    w = np.array(window[-10:], np.float32)
    np.testing.assert_allclose(w[:, 0], g['win_ret'], rtol=1e-5, atol=1e-5)
    np.testing.assert_array_equal(w[:, 2], g['win_len'])
    # the fixture's log-probabilities are those of the trained sigma, not of sigma = 1
    eps = g['eps'].astype(np.float64)
    logp = (-0.5 * eps * eps - theta[:A].astype(np.float64) - 0.5 * np.log(2 * np.pi)).sum(-1)
    np.testing.assert_allclose(g['slab_logp'], logp, rtol=1e-5, atol=2e-5)


def test_external_golden_trained_std(golden_dir, monkeypatch):
    """Two epochs of the unmodified reference on the WideBox CMDP (asymmetric action box) at a trained log_std."""
    import external_envs as xe

    g = np.load(os.path.join(golden_dir, 'rollout_external_trained.npz'))
    N, T, O, A, E = int(g['N']), int(g['T']), int(g['O']), int(g['A']), int(g['epochs_rolled'])
    np.testing.assert_array_equal(g['theta'][:A], oac.trained_log_std(A))
    scale = orollout.action_scale
    monkeypatch.setattr(orollout, 'action_scale', lambda act: scale(act, g['act_lo'], g['act_hi']))
    env, norm, window = xe.WideBoxOracle(N, O, A, int(g['tmax']), seed=int(g['seed'])), Normalizer((O,)), []
    eps = g['eps'].reshape(E, T, N, A)
    for e in range(E):
        sl = orollout.rollout_epoch(env, norm, g['theta'], T, eps[e], window=window)
    _check_slabs(sl, g, 2e-5)
    np.testing.assert_allclose(norm.mean, g['norm_mean'], rtol=2e-5, atol=2e-5)
    assert norm.count == int(g['norm_count'])
    w = np.array(window[-10:], np.float32)
    np.testing.assert_allclose(w[:, 0], g['win_ret'], rtol=2e-5, atol=2e-5)
    np.testing.assert_array_equal(w[:, 2], g['win_len'])


def test_rollout_reward_cost_normalize_golden(golden_dir):
    """Two epochs of the unmodified reference with RewardNormalize / CostNormalize on (PDO defaults) vs the
    oracle rollout + the oracle scalar normalisers applied to the finished slabs (the wrappers commute
    with the rollout: the policy never sees rewards)."""
    g = np.load(os.path.join(golden_dir, 'rollout_pdo.npz'))
    N, T, O, A = int(g['N']), int(g['T']), int(g['O']), int(g['A'])
    env = SyntheticBoxEnv(N, O, A, max_episode_steps=int(g['tmax']), seed=int(g['seed']),
                          term_prob=float(g['term_prob']))
    norm, rnorm, cnorm = Normalizer((O,)), Normalizer(()), Normalizer(())
    for e in range(int(g['epochs_rolled'])):
        sl = orollout.rollout_epoch(env, norm, g['theta'], T, g['eps'][e * T:(e + 1) * T])
        rew = orollout.normalize_rows(rnorm, sl['rew'])
        cost = orollout.normalize_rows(cnorm, sl['cost'])
    tol = dict(rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(sl['obs'], g['slab_obs'], **tol)
    np.testing.assert_allclose(rew, g['slab_reward'], rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(cost, g['slab_cost'], rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose([rnorm.mean, rnorm.std, cnorm.mean, cnorm.std],
                               [g['rnorm_mean'], g['rnorm_std'], g['cnorm_mean'], g['cnorm_std']], rtol=1e-5)
    assert rnorm.count == int(g['rnorm_count']) and cnorm.count == int(g['cnorm_count'])
    out = ogae.dual_gae_slab(rew, cost, sl['val_r'], sl['val_c'], sl['flags'], sl['boot_r'], sl['boot_c'],
                             float(g['gamma']), float(g['lam']), float(g['lam_c']))
    np.testing.assert_allclose(out['adv_r'], g['slab_adv_r'], rtol=1e-4, atol=5e-5)
    np.testing.assert_allclose(out['adv_c'], g['slab_adv_c'], rtol=1e-4, atol=5e-5)


def _load_update(golden_dir, name):
    g = np.load(os.path.join(golden_dir, name))
    data = {k[5:]: g[k] for k in g.files if k.startswith('data_')}
    return g, data


def test_lagrange_and_ppolag_update_golden(golden_dir):
    """Oracle PPO-Lag update == unmodified PPOLag._update (same minibatch order)."""
    from oracle import learner as ol

    g, data = _load_update(golden_dir, 'update_ppolag.npz')
    lag = ol.Lagrange(float(g['cost_limit']), float(g['lam0']), float(g['lambda_lr']))
    lam1 = lag.update(float(g['Jc']))
    assert abs(lam1 - float(g['lam1'])) < 1e-7
    L = ol.Learner(g['theta0'], 12, 3)
    perms = g['perms'][::2]   # RandomSampler draws a second, unused randperm per pass
    st = L.update_ppo(data, perms, lam1, batch_size=int(g['batch_size']))
    np.testing.assert_allclose(L.flat(), g['theta1'], rtol=1e-5, atol=1e-6)
    assert st['iters'] == int(g['stop_iter'][-1])
    np.testing.assert_allclose(st['kl'][-1], g['kl'][-1], rtol=1e-4, atol=1e-7)
    np.testing.assert_allclose(st['loss_pi'], g['loss_pi'], rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(st['loss_r'], g['loss_r'], rtol=1e-4, atol=1e-6)


def test_fvp_and_cg_golden(golden_dir):
    import torch

    from oracle import actor_critic as oac
    from oracle import learner as ol

    g, data = _load_update(golden_dir, 'update_cpo.npz')
    O, A = int(g['O']), int(g['A'])
    L = ol.Learner(g['theta0'], O, A, lr_actor=None, lr_critic=1e-3)
    obs = torch.as_tensor(data['obs'])
    fv = L.fvp(g['vec'], obs, float(g['cg_damping'])).numpy()
    np.testing.assert_allclose(fv, g['fvp'], rtol=1e-4, atol=1e-6)
    x = ol.conjugate_gradients(lambda v: L.fvp(v, obs, float(g['cg_damping'])), g['bvec'], int(g['cg_iters'])).numpy()
    np.testing.assert_allclose(x, g['xcg'], rtol=2e-3, atol=1e-5)
    # analytic Gauss-Newton form used by the CUDA kernel (SURVEY §8a row 13)
    nets = oac.unflatten(torch.as_tensor(g['theta0']), O, A)
    pa = {k: v.clone().requires_grad_(True) for k, v in nets['actor'].items()}
    params = [pa[k] for k in ('log_std', 'w1', 'b1', 'w2', 'b2', 'w3', 'b3')]
    mu = oac.mlp(pa, obs)
    vec = torch.as_tensor(g['vec'])
    vs, i = [], 0
    for p_ in params:
        vs.append(vec[i:i + p_.numel()].view_as(p_)); i += p_.numel()
    # J v via double-backward trick on a dummy cotangent
    u = torch.zeros_like(mu, requires_grad=True)
    gr = torch.autograd.grad(mu, params[1:], u, create_graph=True)
    jv = torch.autograd.grad(gr, u, vs[1:])[0]
    sig2 = torch.exp(pa['log_std']) ** 2
    cot = jv / sig2 / (obs.shape[0] * A)
    gn = torch.autograd.grad(mu, params[1:], cot)
    flat = torch.cat([(2.0 / A) * vs[0]] + [t.reshape(-1) for t in gn]) + float(g['cg_damping']) * vec
    np.testing.assert_allclose(flat.detach().numpy(), g['fvp'], rtol=1e-4, atol=1e-6)


def test_cpo_case_known_answers():
    """reference tests/test_policy.py:L57-74: b_grads=[1], q=r=0 and (ep_costs, s) =
    (-1, 1), (-1, -1), (1, -1), (1, 1) give optim_case 3, 2, 1, 0 (CPO.yaml target_kl = 0.01)."""
    from oracle.learner import cpo_determine_case

    b_dot_b, q, r, kl = 1.0, 0.0, 0.0, 0.01
    assert cpo_determine_case(b_dot_b, -1.0, q, r, 1.0, kl)[0] == 3
    assert cpo_determine_case(b_dot_b, -1.0, q, r, -1.0, kl)[0] == 2
    assert cpo_determine_case(b_dot_b, 1.0, q, r, -1.0, kl)[0] == 1
    assert cpo_determine_case(b_dot_b, 1.0, q, r, 1.0, kl)[0] == 0
    assert cpo_determine_case(1e-8, -1.0, q, r, 1.0, kl)[0] == 4


def test_focops_update_golden(golden_dir):
    """Oracle FOCOPS update (with the reference's [b,1] x [b] broadcast) == unmodified FOCOPS._update."""
    from oracle import learner as ol

    g, data = _load_update(golden_dir, 'update_focops.npz')
    O, A = int(g['O']), int(g['A'])
    L = ol.Learner(g['theta0'], O, A)
    st = L.update_ppo(data, g['perms'][::2], float(g['lam1']), batch_size=int(g['batch_size']),
                      focops={'lam': float(g['focops_lam']), 'eta': float(g['focops_eta'])})
    np.testing.assert_allclose(L.flat(), g['theta1'], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(st['loss_pi'], g['loss_pi'], rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(st['kl'][-1], g['kl'][-1], rtol=1e-4, atol=1e-7)


def test_p3o_update_golden(golden_dir):
    """Oracle P3O update (PPO clip + kappa * relu(mean(ratio adv_c) + Jc - limit)) == unmodified P3O._update."""
    from oracle import learner as ol

    g, data = _load_update(golden_dir, 'update_p3o.npz')
    O, A = int(g['O']), int(g['A'])
    L = ol.Learner(g['theta0'], O, A)
    st = L.update_ppo(data, g['perms'][::2], 0.0, batch_size=int(g['batch_size']),
                      p3o={'kappa': float(g['kappa']), 'jc_minus_limit': float(g['Jc']) - float(g['cost_limit'])})
    np.testing.assert_allclose(L.flat(), g['theta1'], rtol=1e-5, atol=1e-6)
    # the reference logs the PPO part and the penalty separately (Loss/Loss_pi, Loss/Loss_pi_cost)
    np.testing.assert_allclose(st['loss_pi'], g['loss_pi'] + g['loss_pi_cost'], rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(st['kl'][-1], g['kl'][-1], rtol=1e-4, atol=1e-7)


def test_pid_lagrange_golden(golden_dir):
    """oracle PIDLagrangian vs the reference class over the recorded cost sequences (bit-exact: both are
    Python-float recurrences)."""
    from oracle.learner import PIDLagrangian

    g = np.load(os.path.join(golden_dir, 'pid_lagrange.npz'))
    keys = ('pid_kp', 'pid_ki', 'pid_kd', 'pid_d_delay', 'pid_delta_p_ema_alpha', 'pid_delta_d_ema_alpha',
            'sum_norm', 'diff_norm', 'penalty_max', 'lagrangian_multiplier_init', 'cost_limit')
    for i in range(int(g['n_cfgs'])):
        cfg = {k: g[f'cfg_{i}_{k}'].item() for k in keys}
        pid = PIDLagrangian(**cfg)
        lam = [pid.pid_update(float(c)) for c in g['costs']]
        np.testing.assert_array_equal(np.asarray(lam), g[f'lam_{i}'])


def test_pcpo_step_golden(golden_dir):
    """oracle PCPO projection step on the golden data reproduces the reference's logged q, r, s and,
    through the accepted line-search fraction, its final step norm."""
    import torch

    from oracle import learner as ol

    g, data = _load_update(golden_dir, 'update_pcpo.npz')
    O, A = int(g['O']), int(g['A'])
    L = ol.Learner(g['theta0'], O, A, lr_actor=None, lr_critic=1e-3)
    obs, act, logp = (torch.as_tensor(data[k]) for k in ('obs', 'act', 'logp'))
    damping, iters, kl = float(g['cg_damping']), int(g['cg_iters']), float(g['target_kl'])
    fvp = lambda v: L.fvp(v, obs, damping)   # noqa: E731
    L.zero_grad('actor')
    L.loss_pi_plain(obs, act, logp, torch.as_tensor(data['adv_r'])).backward()
    grads = -L.flat_grad('actor')
    x = ol.conjugate_gradients(fvp, grads.numpy(), iters)
    hx = fvp(x)
    xhx = float(x.dot(hx))
    L.zero_grad('actor')
    L.loss_pi_cost(obs, act, logp, torch.as_tensor(data['adv_c'])).backward()
    b = L.flat_grad('actor')
    p = ol.conjugate_gradients(fvp, b.numpy(), iters)
    r, s = float(grads.dot(p)), float(b.dot(p))
    np.testing.assert_allclose([xhx, r, s], [g['misc_q'][-1], g['misc_r'][-1], g['misc_s'][-1]], rtol=2e-3)
    step = ol.pcpo_step_direction(xhx, hx, p, r, s, float(g['ep_cost']) - float(g['cost_limit']), kl)
    frac = 0.8 ** (int(g['misc_AcceptanceStep'][-1]) - 1)
    np.testing.assert_allclose(float((frac * step).norm()), g['misc_FinalStepNorm'][-1], rtol=5e-3)


def test_trpo_family_actor_step_golden(golden_dir):
    """oracle natural direction + TRPO line search vs the unmodified TRPOLag._update / OnCRPO._update
    (cost-surrogate branch): same xHx, alpha, accepted step, step norm, KL and actor parameters."""
    import torch

    from oracle import actor_critic as oac
    from oracle import learner as ol

    for fname in ('update_trpolag.npz', 'update_oncrpo.npz', 'update_rcpo.npz'):
        g, data = _load_update(golden_dir, fname)
        O, A = int(g['O']), int(g['A'])
        L = ol.Learner(g['theta0'], O, A, lr_actor=None, lr_critic=1e-3)
        obs, act, logp = (torch.as_tensor(data[k]) for k in ('obs', 'act', 'logp'))
        adv_r, adv_c = torch.as_tensor(data['adv_r']), torch.as_tensor(data['adv_c'])
        if str(g['name']) == 'OnCRPO':
            jc, limit, dist_ = float(g['ep_cost']), float(g['extra_cost_limit']), float(g['extra_distance'])
            assert jc > limit + dist_            # the fixture exercises the cost branch
            adv, cost_mode = adv_c, True
        else:
            lam = float(g['lam1'])               # the multiplier is updated before the actor (trpo_lag.py:L67-73)
            adv, cost_mode = (adv_r - lam * adv_c) / (1 + lam), False
        rcpo = str(g['name']) == 'RCPO'          # NaturalPG family: no line search, no KL logged
        accept, kl, step, x, x_hx, alpha = ol.trpo_actor_step(L, obs, act, logp, adv, cost_surrogate=cost_mode,
                                                              search=not rcpo)
        if not rcpo:
            assert accept == int(g['misc_AcceptanceStep'][-1])
        np.testing.assert_allclose([x_hx, alpha, float(step.norm()), float(x.norm())],
                                   [g['misc_xHx'][-1], g['misc_Alpha'][-1], g['misc_FinalStepNorm'][-1], g['misc_H_inv_g'][-1]],
                                   rtol=2e-3)
        if not rcpo:
            np.testing.assert_allclose(kl, g['kl'][-1], rtol=2e-3, atol=1e-7)
        na = oac.layout(O, A)['actor']['size']
        np.testing.assert_allclose(L.flat('actor'), g['theta1'][:na], rtol=2e-3, atol=2e-5)


def test_first_order_family_update_golden(golden_dir):
    """Oracle update with the penalty / multiplier each class derives from Jc == unmodified IPO / CPPOPID /
    PDO ._update: IPO's interior-point penalty (ipo.py:L68-74), CPPOPID's PID controller
    (pid_lagrange.py:L95-125), PDO's Adam multiplier on the unclipped policy-gradient loss."""
    from oracle import learner as ol

    for fname in ('update_ipo.npz', 'update_cppopid.npz', 'update_pdo.npz'):
        g, data = _load_update(golden_dir, fname)
        name, O, A, jc = str(g['name']), int(g['O']), int(g['A']), float(g['ep_cost'])
        if name == 'IPO':
            lam = float(g['extra_kappa']) / (float(g['extra_cost_limit']) - jc + 1e-8)
            lam = lam if 0 <= lam <= 1.0 else 1.0                      # penalty_max = 1.0 (IPO.yaml)
        elif name == 'CPPOPID':
            pid = ol.PIDLagrangian(0.1, 0.01, 0.01, 10, 0.95, 0.95, True, False, 100.0, 0.001, float(g['lagrange_cost_limit']))
            lam = pid.pid_update(jc)
        else:
            lag = ol.Lagrange(float(g['lagrange_cost_limit']), 0.001, 0.035)
            lam = lag.update(jc)
        np.testing.assert_allclose(lam, float(g['lam1']), rtol=1e-5, atol=1e-7, err_msg=name)
        L = ol.Learner(g['theta0'], O, A)
        st = L.update_ppo(data, g['perms'][::2], float(lam), batch_size=int(g['batch_size']), plain=(name == 'PDO'))
        np.testing.assert_allclose(L.flat(), g['theta1'], rtol=1e-5, atol=1e-6, err_msg=name)
        np.testing.assert_allclose(st['kl'][-1], g['kl'][-1], rtol=1e-4, atol=1e-7, err_msg=name)


def test_rollout_saute_golden(golden_dir):
    """Oracle rollout with the SauteAdapter semantics (safety-state augmentation, unsafe reward, z = 1 on the
    final observations) == unmodified PPOSaute rollout on the synthetic env (adapter/saute_adapter.py:L135-217).
    Pins the specification of the §8f rank-4 row before its CUDA implementation exists."""
    g = np.load(os.path.join(golden_dir, 'rollout_pposaute.npz'))
    N, T, O, A = int(g['N']), int(g['T']), int(g['O']), int(g['A'])
    gam, L = float(g['algo_saute_gamma']), float(g['algo_max_ep_len'])
    budget = float(g['algo_safety_budget']) * (1 - gam ** L) / (1 - gam) / L       # saute_adapter.py:L62-68
    env = SyntheticBoxEnv(N, O, A, max_episode_steps=int(g['tmax']), seed=int(g['seed']),
                          term_prob=float(g['term_prob']))
    norm = Normalizer((O,))
    window = []
    sl = orollout.rollout_epoch(env, norm, g['theta'], T, g['eps'], window=window,
                                saute={'budget': budget, 'gamma': gam, 'unsafe_reward': float(g['algo_unsafe_reward'])})
    tol = dict(rtol=1e-5, atol=1e-5)
    assert sl['obs'].shape == g['slab_obs'].shape == (T, N, O + 1)
    np.testing.assert_allclose(sl['obs'], g['slab_obs'], **tol)
    np.testing.assert_allclose(sl['act'], g['slab_act'], **tol)
    np.testing.assert_allclose(sl['rew'], g['slab_reward'], **tol)
    assert (sl['rew'] == np.float32(-0.5)).mean() > 0.2          # the unsafe branch is exercised
    assert np.array_equal(sl['cost'], g['slab_cost'])
    np.testing.assert_allclose(sl['val_r'], g['slab_value_r'], **tol)
    out = ogae.dual_gae_slab(sl['rew'], sl['cost'], sl['val_r'], sl['val_c'], sl['flags'], sl['boot_r'], sl['boot_c'],
                             float(g['gamma']), float(g['lam']), float(g['lam_c']))
    np.testing.assert_allclose(out['adv_r'], g['slab_adv_r'], rtol=1e-4, atol=2e-5)      # bootstrap on z = 1 finals
    w = np.array(window[-10:], np.float32)
    np.testing.assert_allclose(w[:, 0], g['win_ret'], rtol=1e-5, atol=1e-5)              # returns keep the raw reward


def test_simmer_controller_and_rollout_golden(golden_dir):
    """Oracle SimmerPIDAgent == the reference controller over a cost sequence (two gain settings, the clamp to
    the budget bound included), and the oracle rollout started at the relative budget == an unmodified
    PPOSimmerPID rollout (adapter/simmer_adapter.py:L97-131)."""
    import torch

    from oracle import learner as ol

    c = np.load(os.path.join(golden_dir, 'simmer_controller.npz'))
    scale = float(c['scale'])
    for i in range(2):
        kp, ki, kd, polyak = (float(v) for v in c[f'cfg_{i}'])
        agent = ol.SimmerPIDAgent(kp, ki, kd, polyak, torch.ones(3, 1) * 25.0 * scale)
        budget = torch.ones(3, 1) * 15.0 * scale
        hist = []
        for cost in c['costs']:
            budget = agent.act(budget, torch.as_tensor(cost) * scale)
            hist.append(budget.numpy().copy())
        np.testing.assert_allclose(np.stack(hist), c[f'budget_{i}'], rtol=1e-6, atol=1e-7)

    g = np.load(os.path.join(golden_dir, 'rollout_pposimmer.npz'))
    N, T, O, A = int(g['N']), int(g['T']), int(g['O']), int(g['A'])
    gam, L = float(g['algo_saute_gamma']), float(g['algo_max_ep_len'])
    per_step = (1 - gam ** L) / (1 - gam) / L
    budget, upper = float(g['algo_safety_budget']) * per_step, float(g['algo_upper_budget']) * per_step
    env = SyntheticBoxEnv(N, O, A, max_episode_steps=int(g['tmax']), seed=int(g['seed']), term_prob=float(g['term_prob']))
    sl = orollout.rollout_epoch(env, Normalizer((O,)), g['theta'], T, g['eps'],
                                saute={'budget': budget, 'gamma': gam, 'unsafe_reward': float(g['algo_unsafe_reward']),
                                       'z0': budget / upper})
    np.testing.assert_allclose(sl['obs'], g['slab_obs'], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(sl['rew'], g['slab_reward'], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(sl['val_r'], g['slab_value_r'], rtol=1e-5, atol=1e-5)


def test_rollout_early_terminated_golden(golden_dir):
    """Oracle rollout with the EarlyTerminatedAdapter semantics (accumulated cost over the limit: reward 0, terminated,
    env reset; the accumulator survives ordinary episode ends) == unmodified PPOEarlyTerminated rollout on the synthetic
    env with one env, as upstream requires (adapter/early_terminated_adapter.py:L42, L56-98)."""
    g = np.load(os.path.join(golden_dir, 'rollout_ppoearly.npz'))
    N, T, O, A = int(g['N']), int(g['T']), int(g['O']), int(g['A'])
    assert N == 1
    env = SyntheticBoxEnv(N, O, A, max_episode_steps=int(g['tmax']), seed=int(g['seed']), term_prob=float(g['term_prob']))
    window = []
    sl = orollout.rollout_epoch(env, Normalizer((O,)), g['theta'], T, g['eps'], window=window,
                                early={'cost_limit': float(g['algo_cost_limit']), 'acc': np.zeros(N, np.float32)})
    tol = dict(rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(sl['obs'], g['slab_obs'], **tol)
    np.testing.assert_allclose(sl['act'], g['slab_act'], **tol)
    assert np.array_equal(sl['rew'] == 0, g['slab_reward'] == 0) and (sl['rew'] == 0).sum() >= 10     # early terminations happen
    np.testing.assert_allclose(sl['rew'], g['slab_reward'], **tol)
    assert np.array_equal(sl['cost'], g['slab_cost'])
    np.testing.assert_allclose(sl['val_r'], g['slab_value_r'], **tol)
    w = np.array(window[-10:], np.float32)
    np.testing.assert_allclose(w[:, 0], g['win_ret'], rtol=1e-5, atol=1e-5)
    assert np.array_equal(w[:, 1], g['win_cost']) and np.array_equal(w[:, 2], g['win_len'])


def test_cup_update_golden(golden_dir):
    """Oracle CUP (PPO stage on adv_r, then the KL-regularised cost projection stage, first_order/cup.py:L93-215)
    == unmodified CUP._update.  Pins the specification before the CUDA loss kind exists."""
    from oracle import learner as ol

    g, data = _load_update(golden_dir, 'update_cup.npz')
    O, A = int(g['O']), int(g['A'])
    lam = ol.Lagrange(float(g['cost_limit']), 0.001, 0.035).update(float(g['Jc']))
    np.testing.assert_allclose(lam, float(g['lam1']), rtol=1e-5)
    L = ol.Learner(g['theta0'], O, A)
    st = L.update_ppo(data, g['perms'][0:4:2], 0.0, batch_size=int(g['batch_size']))
    assert st['iters'] == int(g['stop_iter'][-1])
    done = L.update_cup_stage2(data, g['perms'][4:8:2], float(lam), batch_size=int(g['batch_size']))
    assert done == int(g['second_stop_iter'][-1])
    np.testing.assert_allclose(L.flat(), g['theta1'], rtol=1e-5, atol=1e-6)


def test_multirank_update_golden(golden_dir):
    """The reference under parallel = 2 (two gloo ranks of the unmodified reference, tests/golden/
    make_golden_parallel2.py): clip locally -> average -> Adam per minibatch, rank-averaged KL, all-reduced Jc."""
    from oracle import learner as ol

    g = np.load(os.path.join(golden_dir, 'update_ppolag_parallel2.npz'))
    O, A = int(g['O']), int(g['A'])
    datas = [{k[len(f'r{r}_data_'):]: g[k] for k in g.files if k.startswith(f'r{r}_data_')} for r in (0, 1)]
    lag = ol.Lagrange(float(g['cost_limit']), float(g['lam0']), float(g['lambda_lr']))
    lam = lag.update(float(g['Jc']))
    assert abs(lam - float(g['lam1'])) < 1e-6
    L = ol.Learner(g['theta0'], O, A)
    st = ol.update_ppo_multirank(L, datas, [g['perms_r0'][::2], g['perms_r1'][::2]], lam, batch_size=int(g['batch_size']))   # every DataLoader pass draws two permutations, the second one is used
    got, want = L.flat(), g['theta1']
    np.testing.assert_allclose(got, want, rtol=2e-4, atol=2e-6)
    assert st['iters'] == int(g['stop_iter'][-1])
    np.testing.assert_allclose(st['kl'][-1], g['kl'][-1], rtol=1e-3, atol=1e-7)
