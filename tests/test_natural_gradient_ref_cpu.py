"""Pin the float64 natural-gradient reference (oracle/fisher64.py) on the CPU: the Fisher-vector product and the
conjugate-gradient solve against the golden fixture of the unmodified reference (update_cpo.npz), the surrogate
gradients against the float32 oracle autograd, and the advantage standardisation against pre-standardised data."""
import os

import numpy as np
import pytest
import torch

from oracle import actor_critic as oac
from oracle import fisher64 as f64
from oracle import learner as ol
from test_update_gpu import sigma_cases


@pytest.fixture(scope='module')
def cpo(golden_dir):
    g = np.load(os.path.join(golden_dir, 'update_cpo.npz'))
    data = {k[5:]: g[k] for k in g.files if k.startswith('data_')}
    O, A = int(g['O']), int(g['A'])
    return g, data, O, A, g['theta0'][:oac.layout(O, A)['actor']['size']]


def _trained(theta, A):
    """theta with the actor's log_std set to oracle.actor_critic.trained_log_std (sigma 0.2 to 1.5)."""
    theta = np.array(theta, np.float32)
    theta[:A] = oac.trained_log_std(A)
    return theta


def test_fvp64_golden(cpo):
    g, data, O, A, th = cpo
    fv = f64.fvp64(th, g['vec'], data['obs'], float(g['cg_damping']))
    np.testing.assert_allclose(fv, g['fvp'], rtol=1e-4, atol=1e-6)
    # the chunked sum is the same mean KL
    np.testing.assert_allclose(f64.fvp64(th, g['vec'], data['obs'], float(g['cg_damping']), chunk=50), fv,
                               rtol=1e-12, atol=1e-14)


def test_cg64_golden(cpo):
    g, data, O, A, th = cpo
    d = float(g['cg_damping'])
    x, steps, norms = f64.cg64(lambda v: f64.fvp64(th, v, data['obs'], d), g['bvec'], int(g['cg_iters']))
    np.testing.assert_allclose(x, g['xcg'], rtol=2e-3, atol=1e-5)
    assert steps == int(g['cg_iters']) and len(norms) == steps


@pytest.mark.parametrize('kind,trained', sigma_cases([('ratio',), ('cost',)], [('ratio',), ('cost',)]))
def test_surrogate_grad64_vs_oracle_autograd(cpo, kind, trained):
    g, data, O, A, th = cpo
    theta0 = _trained(g['theta0'], A) if trained else g['theta0']
    th = theta0[:th.size]
    lam = 0.37
    grad, loss = f64.surrogate_grad64(th, data, [0.0, 1.0, 0.0, 1.0], lam, kind)
    L = ol.Learner(theta0, O, A, lr_actor=None)
    t = {k: torch.as_tensor(v) for k, v in data.items()}
    if kind == 'ratio':
        want_loss = L.loss_pi_plain(t['obs'], t['act'], t['logp'], (t['adv_r'] - lam * t['adv_c']) / (1 + lam))
    else:
        want_loss = L.loss_pi_cost(t['obs'], t['act'], t['logp'], t['adv_c'])
    want_loss.backward()
    want = L.flat_grad('actor').numpy()
    assert np.linalg.norm(grad - want) / np.linalg.norm(want) < 1e-5
    np.testing.assert_allclose(grad, want, rtol=1e-4, atol=1e-6 * np.abs(want).max())
    np.testing.assert_allclose(loss, float(want_loss), rtol=1e-5, atol=1e-7)


def test_moments_and_eval64(cpo):
    """Raw advantages with moments == standardised advantages with identity moments; eval64 at theta_old == theta
    gives KL 0 and the plain surrogates, and at a perturbed actor the oracle KL / surrogates.  Both at the golden's
    log_std = 0 and at a trained log_std, where the perturbed actor's log_std also moves by 0.05 to 0.3 per action, so
    the KL sees sigma_old != sigma."""
    g, data, O, A, th = cpo
    m = [0.37, 2.3, -0.41, 1.0]
    raw = dict(data, adv_r=data['adv_r'] * np.float32(2.3) + np.float32(0.37), adv_c=data['adv_c'] - np.float32(0.41))
    for trained in (False, True):
        theta0 = _trained(g['theta0'], A) if trained else g['theta0']
        th = theta0[:th.size]
        for kind in ('ratio', 'cost'):
            a, la = f64.surrogate_grad64(th, raw, m, 0.37, kind)
            b, lb = f64.surrogate_grad64(th, data, [0.0, 1.0, 0.0, 1.0], 0.37, kind)
            np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-7 * np.abs(b).max())
            np.testing.assert_allclose(la, lb, rtol=1e-5, atol=1e-7)
        ev = f64.eval64(th, th, data, [0.0, 1.0, 0.0, 1.0], 0.0)
        assert ev['kl'] == 0.0
        if not trained:     # the golden's log-probs are those of the log_std = 0 policy
            np.testing.assert_allclose(ev['loss_r'], -data['adv_r'].astype(np.float64).mean(), rtol=1e-4, atol=1e-6)
            np.testing.assert_allclose(ev['ratio'], 1.0, atol=1e-5)
        th2 = (th + 0.01 * g['vec']).astype(np.float32)
        if trained:
            th2[:A] = th[:A] + oac.log_std_shift(A)
        ev2 = f64.eval64(th2, th, raw, m, 0.37)
        L = ol.Learner(theta0, O, A, lr_actor=None)
        obs = torch.as_tensor(data['obs'])
        with torch.no_grad():
            old = L.dist(obs)
            old = torch.distributions.Normal(old.loc.clone(), old.scale.clone())
            L.set_flat('actor', th2)
            new = L.dist(obs)
            kl = torch.distributions.kl_divergence(old, new).mean().item()
            t = {k: torch.as_tensor(v) for k, v in data.items()}
            loss = L.loss_pi_plain(t['obs'], t['act'], t['logp'], (t['adv_r'] - 0.37 * t['adv_c']) / 1.37).item()
            loss_c = L.loss_pi_cost(t['obs'], t['act'], t['logp'], t['adv_c']).item()
            ratio = torch.exp(new.log_prob(t['act']).sum(-1) - t['logp']).mean().item()
        np.testing.assert_allclose(ev2['kl'], kl, rtol=1e-3, atol=1e-9)
        np.testing.assert_allclose([ev2['loss'], ev2['loss_c'], ev2['ratio']], [loss, loss_c, ratio], rtol=1e-4, atol=1e-6)
        np.testing.assert_allclose(f64.mean64(th, data['obs']), old.loc.numpy(), rtol=1e-5, atol=1e-6)
