"""Pin the float64 reference of the two-pass losses (FOCOPS and P3O in oracle/optim64.py) on the CPU: the decomposed
FOCOPS loss against the reference's [b, b] broadcast (Learner.loss_pi_focops run in float64) and the P3O loss against
Learner.loss_pi_p3o, value and gradient, in every mask / gate state; ppo_epoch64 against the float32
Learner.update_ppo with clipping active; ppo_epoch64 against the FOCOPS._update and P3O._update goldens of the
unmodified reference."""
import os

import numpy as np
import pytest
import torch
from torch.distributions import Normal, kl_divergence

from oracle import actor_critic as oac
from oracle import learner as ol
from oracle import optim64 as o64
from test_optimizer_ref_cpu import LAM, MOMENTS, _raw, _standardised
from test_update_gpu import _rand_data


def _perturbed(theta, O, A, seed, scale=0.05, log_std=0.15):
    """theta with the actor moved away from itself: weights by `scale` relative noise, log_std by +-log_std, so
    every sample has a KL of at least ~A log_std^2 / 2 against the unperturbed actor."""
    rng = np.random.default_rng(seed)
    lay = oac.layout(O, A)['actor']
    th = np.array(theta, np.float32, copy=True)
    n = lay['size']
    th[:n] += (scale * np.abs(th[:n]).mean() * rng.standard_normal(n)).astype(np.float32)
    th[:A] = (rng.choice([-1.0, 1.0], A) * log_std).astype(np.float32)
    return th


def _learner64(theta, O, A):
    """Learner with float64 actor leaves, so its verbatim losses run in float64."""
    L = ol.Learner(theta, O, A)
    L.params['actor'] = {k: v.detach().double().requires_grad_(True) for k, v in L.params['actor'].items()}
    return L


def _grad(params):
    return torch.cat([p.grad.reshape(-1) for p in params.values()]).numpy()


def _batch(b, O, A, seed):
    rng = np.random.default_rng(seed)
    theta_old = oac.init_theta(O, A, seed=seed % 5)
    theta = _perturbed(theta_old, O, A, seed)
    data = _rand_data(rng, 1, b, O, A, theta_old)
    t = {k: torch.as_tensor(v).double() for k, v in data.items()}
    with torch.no_grad():
        old = oac.actor_dist(_learner64(theta_old, O, A).params['actor'], t['obs'])
    return theta, t, Normal(old.loc.detach().clone(), old.scale.detach().clone())


@pytest.mark.parametrize('mask', ['mixed', 'in', 'out'])
@pytest.mark.parametrize('b', [1, 7, 64, 512])
def test_focops_decomposed_vs_broadcast(b, mask):
    """mean_i(m_i kl_i) - mean_i(m_i) mean_j(ratio_j adv_j) / lam == the mean of the reference's [b, b] matrix
    (kl[b, 1] - ratio[b] adv[b] / lam) * m[b, 1], entropy bonus included: value and gradient in float64."""
    O, A = 12, 3
    if b == 1 and mask == 'mixed':
        pytest.skip('one sample has no mixed mask')
    theta, t, old = _batch(b, O, A, seed=b + 3)
    L = _learner64(theta, O, A)
    with torch.no_grad():
        kl = kl_divergence(L.dist(t['obs']), old).sum(-1).numpy()
    s = np.sort(kl)
    eta = {'mixed': 0.5 * (s[b // 2 - 1] + s[b // 2]) if b > 1 else 0.0, 'in': 2 * s[-1] + 1.0, 'out': 0.5 * s[0]}[mask]
    m = kl <= eta
    assert {'mixed': 0 < m.mean() < 1, 'in': m.all(), 'out': not m.any()}[mask], (mask, m.mean())
    adv = (t['adv_r'] - LAM * t['adv_c']) / (1 + LAM)
    lam_f, ent = 1.5, 0.01
    want, _ = L.loss_pi_focops(t['obs'], t['act'], t['logp'], adv, old.loc, old.scale, lam_f, eta, ent)
    want.backward()
    L2 = _learner64(theta, O, A)
    got, info = o64.actor_loss64(L2.dist(t['obs']), old, t['act'], t['logp'], adv, None, None, loss_kind=2,
                                 entropy_coef=ent, focops_lam=lam_f, focops_eta=eta)
    got.backward()
    np.testing.assert_allclose(float(got.detach()), float(want.detach()), rtol=1e-12, atol=1e-15)
    gw, gg = _grad(L.params['actor']), _grad(L2.params['actor'])
    np.testing.assert_allclose(gg, gw, rtol=1e-10, atol=1e-13 * np.abs(gw).max())
    assert info['pass1'] == m.mean() and info['stats'][3] == m.mean()
    np.testing.assert_allclose(info['stats'][2], kl.mean(), rtol=1e-14)
    np.testing.assert_allclose(info['margin'], np.abs(kl - eta).min(), rtol=1e-14)
    # slot 0: the loss without the entropy bonus
    np.testing.assert_allclose(info['stats'][0], float(want) + ent * float(L.dist(t['obs']).entropy().mean()),
                               rtol=1e-12, atol=1e-15)
    if mask == 'out':     # only the entropy bonus is left: -ent / A on every log_std, zero elsewhere
        np.testing.assert_allclose(gg[:A], -ent / A, rtol=1e-14)
        assert not gg[A:].any()


@pytest.mark.parametrize('gate', ['on', 'off'])
@pytest.mark.parametrize('b', [1, 64, 512])
def test_p3o_vs_learner(b, gate):
    """actor_loss64 kind 5 == Learner.loss_pi_p3o in float64 (PPO clip on adv_r with the entropy bonus + kappa
    relu(mean(ratio adv_c) + Jc - limit)), relu gate active and inactive."""
    O, A = 12, 3
    theta, t, _ = _batch(b, O, A, seed=b + 11)
    L = _learner64(theta, O, A)
    with torch.no_grad():
        d = L.dist(t['obs'])
        surr = float((torch.exp(d.log_prob(t['act']).sum(-1) - t['logp']) * t['adv_c']).mean())
    jc = -surr + (0.3 if gate == 'on' else -0.3)
    kappa, ent = 0.7, 0.01
    want, _ = L.loss_pi_p3o(t['obs'], t['act'], t['logp'], t['adv_r'], t['adv_c'], 0.2, kappa, jc, ent)
    want.backward()
    L2 = _learner64(theta, O, A)
    got, info = o64.actor_loss64(L2.dist(t['obs']), None, t['act'], t['logp'], None, t['adv_r'], t['adv_c'],
                                 loss_kind=5, clip=0.2, entropy_coef=ent, focops_lam=kappa, focops_eta=jc)
    got.backward()
    np.testing.assert_allclose(float(got.detach()), float(want.detach()), rtol=1e-12, atol=1e-15)
    gw, gg = _grad(L.params['actor']), _grad(L2.params['actor'])
    np.testing.assert_allclose(gg, gw, rtol=1e-10, atol=1e-13 * np.abs(gw).max())
    np.testing.assert_allclose(info['pass1'], surr, rtol=1e-12)
    np.testing.assert_allclose(info['margin'], 0.3, rtol=1e-9)
    assert info['gate'] == (kappa if gate == 'on' else 0.0)
    np.testing.assert_allclose(info['stats'][2], kappa * 0.3 if gate == 'on' else 0.0, rtol=1e-9)


def _epoch_data(seed):
    rng = np.random.default_rng(seed)
    N, T, O, A = 16, 24, 12, 3
    theta = oac.init_theta(O, A, seed=3)
    data = _raw(_rand_data(rng, N, T, O, A, theta))
    perms = np.stack([rng.permutation(N * T) for _ in range(2)])
    return theta, data, perms, O, A


@pytest.mark.parametrize('kind', [2, 5])
def test_ppo_epoch64_two_pass_vs_learner(monkeypatch, kind):
    """Learner.update_ppo(focops= / p3o=) (float32, verbatim broadcast) on standardised advantages vs ppo_epoch64
    kinds 2 / 5 on the raw ones, every network clipping on every step: the same norms and clip decisions, the same
    pass-1 decisions with margin, parameters within fp32 rounding of the update."""
    theta, data, perms, O, A = _epoch_data({2: 42, 5: 47}[kind])
    max_norm = 0.02
    if kind == 2:
        lam_f, eta = 1.5, 0.02
        extra = dict(focops={'lam': lam_f, 'eta': eta})
    else:
        lam_f, eta = 0.7, 0.08        # mean(ratio adv_c) of a 100-row minibatch spreads by ~0.1: both gate states
        extra = dict(p3o={'kappa': lam_f, 'jc_minus_limit': eta})
    kw = dict(batch_size=100, clip=0.2, entropy_coef=0.01, critic_norm_coef=0.05, max_grad_norm=max_norm,
              target_kl=10.0, kl_early_stop=False)
    norms = []
    clip = ol.clip_grad_norm_

    def recording_clip(params, max_grad_norm):
        norms.append(float(clip(params, max_grad_norm)))
        return norms[-1]

    monkeypatch.setattr(ol, 'clip_grad_norm_', recording_clip)
    L = ol.Learner(theta, O, A, lr_actor=3e-3, lr_critic=1e-3)
    st = L.update_ppo(_standardised(data), perms, LAM, **kw, **extra)
    state, rec, passes = o64.ppo_epoch64(theta, data, MOMENTS, perms, LAM, net_mask=7, loss_kind=kind,
                                         update_iters=2, lrs=(3e-3, 1e-3, 1e-3), focops_lam=lam_f, focops_eta=eta,
                                         **kw)
    assert passes == 2 and len(rec['steps']) == 2 * 4
    got = np.array(norms).reshape(-1, 3)[:, [2, 0, 1]]
    want = np.array([r['norm'] for r in rec['steps']])
    np.testing.assert_allclose(got, want, rtol=1e-4)
    assert (want > 1.5 * max_norm).all(), want
    pass1 = np.array([r['pass1'] for r in rec['steps']])
    margin = np.array([r['margin'] for r in rec['steps']])
    print(f'kind {kind}: pass-1 values {np.round(pass1, 4)}, margins min {margin.min():.2e}')
    if kind == 2:
        # the first step's KLs are 0 (all in); the policy then drifts past eta and the masks become mixed, no KL
        # within 1e-6 of eta (the float32 Learner's KLs are good to ~1e-8 here)
        assert pass1[0] == 1.0 and (pass1 < 0.5).any() and (margin > 1e-6).all(), (pass1, margin)
    else:
        gates = np.array([r['gate'] for r in rec['steps']])
        assert set(gates) == {0.0, lam_f} and (margin > 0.01).all(), (gates, margin)
    # logged actor loss: the Learner's value is slot 0 + the P3O penalty - entropy_coef x the mean entropy
    slot0 = np.array([r['stats'][0] for r in rec['steps']])
    pen = np.array([r['stats'][2] for r in rec['steps']]) if kind == 5 else 0.0
    ent = np.array([r['entropy'] for r in rec['steps']])
    np.testing.assert_allclose(st['loss_pi'], slot0 + pen - kw['entropy_coef'] * ent, rtol=1e-5, atol=1e-6)
    diff = np.abs(state['theta'] - L.flat())
    upd = np.abs(state['theta'] - theta)
    print(f'kind {kind}: |64 - 32| max {diff.max():.2e}, relative to the update '
          f'{np.linalg.norm(diff) / np.linalg.norm(upd):.2e}')
    assert np.linalg.norm(diff) < 1e-4 * np.linalg.norm(upd)
    np.testing.assert_allclose(state['theta'], L.flat(), rtol=1e-4, atol=1e-6)
    np.testing.assert_array_equal(state['step'], [8, 8, 8])


def _golden_epoch(g, kind, lam, lam_f, eta):
    data = {k[5:]: g[k] for k in g.files if k.startswith('data_')}
    return o64.ppo_epoch64(g['theta0'], data, [0.0, 1.0, 0.0, 1.0], g['perms'][::2], lam, net_mask=7, loss_kind=kind,
                           batch_size=int(g['batch_size']), update_iters=int(g['update_iters']), clip=0.2,
                           focops_lam=lam_f, focops_eta=eta, critic_norm_coef=0.001, max_grad_norm=40.0,
                           target_kl=0.02, kl_early_stop=True)


def _check_golden(g, state, rec, passes):
    got, want = state['theta'], g['theta1']
    bad = ~np.isclose(got, want, rtol=2e-4, atol=2e-6)
    print(f'golden: max |diff| {np.abs(got - want).max():.2e}, {bad.sum()} off')
    assert bad.mean() < 1e-3 and np.abs(got - want).max() < 2e-3, (bad.sum(), np.abs(got - want).max())
    assert passes == int(g['stop_iter'][-1])
    np.testing.assert_allclose(rec['kl'][-1], g['kl'][-1], rtol=2e-3, atol=1e-6)
    np.testing.assert_array_equal(state['step'], [len(rec['steps'])] * 3)
    np.testing.assert_allclose(np.mean([r['loss'][0] for r in rec['steps']]), g['loss_pi'].mean(), rtol=2e-3,
                               atol=1e-5)


def test_ppo_epoch64_focops_golden(golden_dir):
    """FOCOPS._update of the unmodified reference, at the bar of test_update_gpu::test_focops_update_epoch_golden."""
    g = np.load(os.path.join(golden_dir, 'update_focops.npz'))
    state, rec, passes = _golden_epoch(g, 2, float(g['lam1']), float(g['focops_lam']), float(g['focops_eta']))
    _check_golden(g, state, rec, passes)
    np.testing.assert_allclose([r['loss'][0] for r in rec['steps']], g['loss_pi'][:len(rec['steps'])], rtol=1e-4,
                               atol=1e-6)


def test_ppo_epoch64_p3o_golden(golden_dir):
    """P3O._update of the unmodified reference, at the bar of test_update_gpu::test_p3o_update_epoch_golden."""
    g = np.load(os.path.join(golden_dir, 'update_p3o.npz'))
    state, rec, passes = _golden_epoch(g, 5, 0.0, float(g['kappa']), float(g['Jc']) - float(g['cost_limit']))
    _check_golden(g, state, rec, passes)
    n = len(rec['steps'])
    np.testing.assert_allclose([r['stats'][2] for r in rec['steps']], g['loss_pi_cost'][:n], rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose([r['loss'][0] for r in rec['steps']], g['loss_pi'][:n], rtol=1e-4, atol=1e-6)
