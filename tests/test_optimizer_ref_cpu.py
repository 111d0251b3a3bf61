"""Pin the float64 optimiser reference (oracle/optim64.py) on the CPU: against the float32 oracle
Learner.update_ppo with clipping active (critics only, and every network), against the update_ppolag.npz golden of
the unmodified reference, against a hand-written clip + Adam on supplied gradients, and for an Adam state carried
across ppo_epoch64 calls."""
import os

import numpy as np
import pytest

from oracle import actor_critic as oac
from oracle import learner as ol
from oracle import optim64 as o64
from test_update_gpu import _rand_data

MOMENTS = [0.37, 2.3, -0.41, 1.0]
LAM = 0.37


def _raw(data):
    out = dict(data)
    out['adv_r'] = (data['adv_r'] * np.float32(MOMENTS[1]) + np.float32(MOMENTS[0])).astype(np.float32)
    out['adv_c'] = (data['adv_c'] + np.float32(MOMENTS[2])).astype(np.float32)
    return out


def _standardised(data):
    out = dict(data)
    out['adv_r'] = ((data['adv_r'].astype(np.float64) - MOMENTS[0]) / MOMENTS[1]).astype(np.float32)
    out['adv_c'] = (data['adv_c'].astype(np.float64) - MOMENTS[2]).astype(np.float32)
    return out


@pytest.mark.parametrize('regime', ['critics', 'all'])
def test_ppo_epoch64_vs_learner(monkeypatch, regime):
    """Learner.update_ppo (float32) on standardised advantages vs ppo_epoch64 on the raw ones: the same clip
    decision for every network on every step, and parameters within fp32 rounding of the update."""
    rng = np.random.default_rng(5)
    N, T, O, A = 16, 24, 12, 3
    theta = oac.init_theta(O, A, seed=3)
    data = _raw(_rand_data(rng, N, T, O, A, theta))
    if regime == 'critics':
        data['target_value_r'] = data['target_value_r'] * np.float32(50)
        data['target_value_c'] = data['target_value_c'] * np.float32(50)
    max_norm = 5.0 if regime == 'critics' else 0.02
    perms = np.stack([rng.permutation(N * T) for _ in range(2)])
    kw = dict(batch_size=100, clip=0.2, entropy_coef=0.01, critic_norm_coef=0.05, max_grad_norm=max_norm,
              target_kl=10.0, kl_early_stop=False)
    norms = []
    clip = ol.clip_grad_norm_

    def recording_clip(params, max_grad_norm):
        norms.append(float(clip(params, max_grad_norm)))
        return norms[-1]

    monkeypatch.setattr(ol, 'clip_grad_norm_', recording_clip)
    L = ol.Learner(theta, O, A, lr_actor=3e-3, lr_critic=1e-3)
    L.update_ppo(_standardised(data), perms, LAM, **kw)
    state, rec, passes = o64.ppo_epoch64(theta, data, MOMENTS, perms, LAM, net_mask=7, loss_kind=0,
                                         update_iters=2, lrs=(3e-3, 1e-3, 1e-3), **kw)
    assert passes == 2 and len(rec['steps']) == 2 * 4
    # Learner order per minibatch: reward critic, cost critic, actor
    got = np.array(norms).reshape(-1, 3)[:, [2, 0, 1]]
    want = np.array([r['norm'] for r in rec['steps']])
    np.testing.assert_allclose(got, want, rtol=1e-4)
    clipped = want > max_norm
    assert ((got > max_norm) == clipped).all()
    if regime == 'critics':
        assert clipped[:, 1:].all() and not clipped[:, 0].any(), want
    else:
        assert clipped.all(), want
    diff = np.abs(state['theta'] - L.flat())
    upd = np.abs(state['theta'] - theta)
    print(f'{regime}: norms min/max {want.min():.3g} / {want.max():.3g}; |64 - 32| max {diff.max():.2e}, '
          f'relative to the update {np.linalg.norm(diff) / np.linalg.norm(upd):.2e}')
    assert np.linalg.norm(diff) < 1e-4 * np.linalg.norm(upd)
    np.testing.assert_allclose(state['theta'], L.flat(), rtol=1e-4, atol=1e-6)
    np.testing.assert_array_equal(state['step'], [8, 8, 8])


def test_ppo_epoch64_golden(golden_dir):
    """The PPOLag._update golden of the unmodified reference (max_grad_norm 40, KL early stop), at the bar of
    test_update_gpu::test_ppolag_update_epoch_golden."""
    g = np.load(os.path.join(golden_dir, 'update_ppolag.npz'))
    data = {k[5:]: g[k] for k in g.files if k.startswith('data_')}
    lam = ol.Lagrange(float(g['cost_limit']), float(g['lam0']), float(g['lambda_lr'])).update(float(g['Jc']))
    state, rec, passes = o64.ppo_epoch64(g['theta0'], data, [0.0, 1.0, 0.0, 1.0], g['perms'][::2], lam, net_mask=7,
                                         loss_kind=0, batch_size=int(g['batch_size']),
                                         update_iters=int(g['update_iters']), critic_norm_coef=0.001,
                                         max_grad_norm=40.0, target_kl=0.02, kl_early_stop=True)
    got, want = state['theta'], g['theta1']
    bad = ~np.isclose(got, want, rtol=2e-4, atol=2e-6)
    print(f'golden: max |diff| {np.abs(got - want).max():.2e}')
    assert bad.mean() < 1e-3 and np.abs(got - want).max() < 2e-3, (bad.sum(), np.abs(got - want).max())
    assert passes == int(g['stop_iter'][-1])
    np.testing.assert_allclose(rec['kl'][-1], g['kl'][-1], rtol=1e-3, atol=1e-7)
    np.testing.assert_allclose([r['loss'][1] for r in rec['steps']], g['loss_r'], rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose([r['loss'][2] for r in rec['steps']], g['loss_c'], rtol=1e-4, atol=1e-6)
    assert (np.array([r['coef'] for r in rec['steps']]) == 1.0).all()
    np.testing.assert_array_equal(state['step'], [len(rec['steps'])] * 3)


def _adam_by_hand(theta, m, v, t, g, lr):
    m = 0.9 * m + 0.1 * g
    v = 0.999 * v + 0.001 * g * g
    return theta - lr / (1 - 0.9 ** t) * m / (np.sqrt(v) / np.sqrt(1 - 0.999 ** t) + 1e-8), m, v


@pytest.mark.parametrize('max_norm', [0.0, 1e-4, 0.3, 1e6])
def test_step64_vs_hand_written(max_norm):
    """step64 == clip (coefficient max / (norm + 1e-6), the critic L2 gradient inside the norm) + Adam with bias
    correction, written out in numpy, over 30 steps with three learning rates and a partial net_mask."""
    O, A = 7, 2
    theta = oac.init_theta(O, A, seed=1)
    lay = oac.layout(O, A)
    rng = np.random.default_rng(2)
    lrs, coef = (1e-3, 3e-3, 7e-4), 0.05
    state = o64.init_state(theta)
    th, m, v = (state[k].copy() for k in ('theta', 'm', 'v'))
    for t in range(1, 31):
        mask = 7 if t % 3 else 6
        g = rng.standard_normal(theta.size) * rng.choice([1e-4, 1.0, 30.0])
        state, rec = o64.step64(state, g, max_grad_norm=max_norm, lrs=lrs, critic_norm_coef=coef, O=O,
                                net_mask=mask)
        for k, net in enumerate(o64.NETS):
            sl = slice(lay[net]['start'], lay[net]['start'] + lay[net]['size'])
            if not (mask >> k) & 1:
                assert rec['norm'][k] == 0 and not rec['grad'][sl].any()
                continue
            gk = g[sl] + (2 * coef * th[sl] if k else 0.0)
            n = np.linalg.norm(gk)
            c = min(max_norm / (n + 1e-6), 1.0) if max_norm > 0 else 1.0
            np.testing.assert_allclose([rec['norm'][k], rec['coef'][k]], [n, c], rtol=1e-12)
            np.testing.assert_allclose(rec['grad'][sl], c * gk, rtol=1e-10, atol=1e-13 * np.abs(gk).max())
            if k:
                np.testing.assert_allclose(rec['l2'][k], coef * (th[sl] ** 2).sum(), rtol=1e-12)
            th[sl], m[sl], v[sl] = _adam_by_hand(th[sl], m[sl], v[sl], state['step'][k], c * gk, lrs[k])
        np.testing.assert_allclose(state['theta'], th, rtol=1e-12, atol=1e-15)
        # torch's lerp / addcmul round differently from the written-out moments: 1e-12 of the largest entry
        np.testing.assert_allclose(state['m'], m, rtol=1e-10, atol=1e-12 * np.abs(m).max())
        np.testing.assert_allclose(state['v'], v, rtol=1e-10, atol=1e-12 * np.abs(v).max())
    assert list(state['step']) == [20, 30, 30]


def test_ppo_epoch64_state_continues():
    """Two ppo_epoch64 calls of one pass each, the second continuing the first's state, == one call of two passes
    (critics only: no KL reference policy in between)."""
    rng = np.random.default_rng(9)
    N, T, O, A = 8, 20, 10, 2
    theta = oac.init_theta(O, A, seed=4)
    data = _raw(_rand_data(rng, N, T, O, A, theta))
    perms = np.stack([rng.permutation(N * T) for _ in range(2)])
    kw = dict(net_mask=6, loss_kind=1, batch_size=48, critic_norm_coef=0.05, max_grad_norm=0.5, lrs=(0, 2e-3, 5e-4))
    both, rb, _ = o64.ppo_epoch64(theta, data, MOMENTS, perms, LAM, update_iters=2, **kw)
    one, r1, _ = o64.ppo_epoch64(theta, data, MOMENTS, perms[:1], LAM, update_iters=1, **kw)
    two, r2, _ = o64.ppo_epoch64(None, data, MOMENTS, perms[1:], LAM, update_iters=1, state=one, **kw)
    for k in ('theta', 'm', 'v', 'step'):
        np.testing.assert_array_equal(two[k], both[k])
    np.testing.assert_array_equal(both['step'], [0, 8, 8])
    assert np.array_equal(np.array([r['coef'] for r in r1['steps'] + r2['steps']]),
                          np.array([r['coef'] for r in rb['steps']]))
    Pa = oac.layout(O, A)['actor']['size']
    assert (both['theta'][:Pa] == theta[:Pa]).all() and not both['m'][:Pa].any()
