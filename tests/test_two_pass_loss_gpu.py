"""GPU: the two-pass loss kinds FOCOPS (2) and P3O (5) against the float64 reference (oracle/optim64.py actor_loss64,
minibatch64, ppo_epoch64; pinned to the verbatim reference losses and to the FOCOPS / P3O goldens in
test_two_pass_ref_cpu).

Pass 1 of a two-pass minibatch runs the actor forward only; pass1_gate reduces its statistics rows into the FOCOPS
mask mean or the P3O relu gate, which pass 2 reads for every sample's gradient.  On the tf32 and bf16x3 paths pass 1
runs on osb_tc_grid_blocks(count, 1) CTAs (up to every SM), pass 2 on a third of them: from ~5.6 k rows on an H100
SXM the two grids differ, and the 16 384-row (bench) and ~21 000-row (more tiles than SMs) minibatches cover that.

  a. One minibatch of osb_minibatch_grad / _tc / _x3 + osb_grad_reduce: every network's gradient (critic L2 term
     included) and the logged actor slots 0, 2 and 4, on raw advantages with non-trivial moments, an entropy bonus,
     an actor perturbed away from the old policy (mu_old / logstd_old from a float64 old policy, the same for every
     precision), a non-zero mb_start and a ragged count.  Regimes: FOCOPS mask mixed / all in / all out, P3O gate on /
     off, each chosen from the float64 values with its margin asserted.
  b. Whole UpdateEngine.ppo_epoch runs (fp32, tf32, bf16x3 stepwise, and O = 111 at precision 2, which takes the fp32
     tiles) with clipping active on every network: one step, then two passes over 3.5 minibatches of 8 192 rows; the
     P3O data make the gate change between minibatches.  A KL early stop after the first of three passes.

Each case prints its worst error and its decision margins."""
import functools
import time

import numpy as np
import pytest
import torch
from torch.distributions import Normal, kl_divergence

from oracle import actor_critic as oac
from oracle import fisher64 as f64
from oracle import optim64 as o64
from test_optimizer_gpu import (LRS, REGIMES, _check_regime, _compare_epoch, _compare_stats, _compare_step,
                                _host, _regime_data)
from test_update_gpu import _rand_data, _rows, _setup

pytestmark = pytest.mark.gpu

MOMENTS = [0.37, 2.3, -0.41, 1.0]
LAM = 0.37            # Lagrange multiplier of the FOCOPS advantage mix; P3O trains on adv_r (no multiplier)
ENT = 0.01
COEF = 0.01           # critic L2 coefficient
FOCOPS_LAM = 1.5
KAPPA = 0.7
FOCOPS, P3O = 2, 5
FNS = {'fp32': 'osb_minibatch_grad', 'tf32': 'osb_minibatch_grad_tc', 'bf16x3': 'osb_minibatch_grad_x3'}
REGIME_KIND = {'focops_mixed': FOCOPS, 'focops_in': FOCOPS, 'focops_out': FOCOPS, 'p3o_on': P3O, 'p3o_off': P3O}


def _lib():
    from omnisafe_b200._lib import current_stream, lib, ptr
    return lib(), ptr, current_stream()


def _slab(x, N, T):
    """env-major [N * T, ...] -> the buffer's time-major [T, N, ...]"""
    x = np.asarray(x, np.float32)
    return torch.as_tensor(x.reshape(N, T, *x.shape[1:]).swapaxes(0, 1).copy())


# ---- a: one minibatch ---------------------------------------------------------------------------------------------

# (O, A, count): the headline shape at one tile, the bench minibatch (pass 1 on more CTAs than pass 2) and ~21 000
# rows (more tiles than SMs in pass 1); O % 4 != 0; A = 1; the A > 8 template; obs dims > 64 (fp32 and tf32 only)
SIZES = [(60, 8, 100), (60, 8, 16384), (60, 8, 21003), (17, 6, 100), (17, 6, 3001), (33, 1, 100), (33, 1, 3001),
         (64, 16, 100), (64, 16, 21003), (45, 9, 100), (45, 9, 3001), (111, 8, 100), (111, 8, 3001), (376, 8, 3001)]
START = 37


@functools.lru_cache(maxsize=None)
def _mb_data(O, A, count):
    """Env-major batch (raw advantages), the perturbed actor theta, the old policy's float64 means rounded to float32
    (what every kernel reads), and a sample order whose minibatch window [START, START + count) leaves out the `hole`
    rows whose float64 KL is nearest to the median: a mixed FOCOPS mask can then be cut with a margin that no
    precision's rounding crosses (neighbouring KLs of 21 000 samples lie ~1e-6 apart)."""
    T = 8
    hole = max(8, count // 20)
    N = -(-(count + START + 27 + hole) // T)
    rng = np.random.default_rng(100 * O + A + count)
    theta_old = oac.init_theta(O, A, seed=O + A)
    data = _rand_data(rng, N, T, O, A, theta_old)
    data['adv_r'] = (data['adv_r'] * np.float32(MOMENTS[1]) + np.float32(MOMENTS[0])).astype(np.float32)
    data['adv_c'] = (data['adv_c'] + np.float32(MOMENTS[2])).astype(np.float32)
    # critic targets off-centre, so that the output-bias gradients 2 mean(v - target) are ~1 and do not cancel (a
    # near-zero reference would turn an absolute error at the precision's level into a large relative one)
    data['target_value_r'] = (data['target_value_r'] + np.float32(0.5)).astype(np.float32)
    data['target_value_c'] = (data['target_value_c'] - np.float32(0.5)).astype(np.float32)
    Pa = oac.layout(O, A)['actor']['size']
    theta = theta_old.copy()
    theta[:Pa] += (0.5 * np.abs(theta_old[:Pa]).mean() * rng.standard_normal(Pa)).astype(np.float32)
    theta[:A] = (rng.choice([-1.0, 1.0], A) * 0.15).astype(np.float32)    # every sample's KL >= ~A * 0.01
    mu_old = f64.mean64(theta_old[:Pa], data['obs']).astype(np.float32)
    new = Normal(torch.as_tensor(f64.mean64(theta[:Pa], data['obs'])), torch.exp(f64._t64(theta[:A])))
    kl = kl_divergence(new, Normal(f64._t64(mu_old), torch.exp(f64._t64(theta_old[:A])))).sum(-1).numpy()
    near = np.argsort(np.abs(kl - np.median(kl)))[:hole]
    perm = np.concatenate([rng.permutation(np.setdiff1d(np.arange(N * T), near)), rng.permutation(near)])
    return N, T, theta, data, mu_old, theta_old[:A].copy(), perm


@functools.lru_cache(maxsize=None)
def _mb_ref(O, A, count, regime):
    """The regime's parameters chosen from the float64 per-sample values, and the float64 gradient / statistics."""
    t0 = time.perf_counter()
    N, T, theta, data, mu_old, logstd_old, perm = _mb_data(O, A, count)
    idx = perm[START:START + count]
    Pa = oac.layout(O, A)['actor']['size']
    obs = data['obs'][idx]
    new = Normal(torch.as_tensor(f64.mean64(theta[:Pa], obs)), torch.exp(f64._t64(theta[:A])))
    kind = REGIME_KIND[regime]
    if kind == FOCOPS:
        old = Normal(f64._t64(mu_old[idx]), torch.exp(f64._t64(logstd_old)))
        kl = np.sort(kl_divergence(new, old).sum(-1).numpy())
        if regime == 'focops_mixed':    # midpoint of the widest gap between neighbouring KLs in the middle half
            lo, hi = count // 4, 3 * count // 4
            i = lo + int(np.argmax(np.diff(kl[lo:hi + 1])))
            eta = 0.5 * (kl[i] + kl[i + 1])
        else:
            eta = 2.0 * kl[-1] + 1.0 if regime == 'focops_in' else 0.5 * kl[0]
        lam, lam_f = LAM, FOCOPS_LAM
    else:
        ratio = torch.exp(new.log_prob(f64._t64(data['act'][idx])).sum(-1) - f64._t64(data['logp'][idx]))
        surr = float((ratio * (f64._t64(data['adv_c'][idx]) - MOMENTS[2])).mean())
        eta = -surr + (0.2 if regime == 'p3o_on' else -0.2)
        lam, lam_f = 0.0, KAPPA
    grad, info = o64.minibatch64(theta, data, MOMENTS, idx, lam, loss_kind=kind, old_mu=mu_old, old_logstd=logstd_old,
                                 critic_norm_coef=COEF, clip=0.2, entropy_coef=ENT, focops_lam=lam_f, focops_eta=eta)
    if kind == FOCOPS:
        m = info['pass1']
        assert {'focops_mixed': 0.25 <= m <= 0.75, 'focops_in': m == 1.0, 'focops_out': m == 0.0}[regime], m
        assert info['margin'] >= 1e-4, info['margin']
    else:
        assert info['gate'] == (KAPPA if regime == 'p3o_on' else 0.0) and info['margin'] >= 0.05, info
    lay = oac.layout(O, A)
    for net in ('reward_critic', 'cost_critic'):
        o = lay[net]['entries']['b3'][0]
        assert abs(grad[o]) > 0.2, (net, grad[o])
    print(f'float64 reference ({count} rows): {time.perf_counter() - t0:.2f} s')
    return dict(kind=kind, lam=lam, lam_f=lam_f, eta=eta, grad=grad, info=info)


def _rna(x):
    """cvt.rna.tf32.f32: float32 rounded to 10 mantissa bits, ties away from zero."""
    u = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    return torch.as_tensor(((u + 0x1000) & 0xFFFFE000).astype(np.uint32).view(np.float32).astype(np.float64))


@functools.lru_cache(maxsize=None)
def _tf32_clip_reference(O, A, count, regime):
    """The float64 actor gradient of a P3O case with each sample's PPO-clip decision taken from a forward on
    tf32-rounded operands (obs, weights and hidden activations, as the tf32 tiles see them), and the number of
    decisions that differ from float64.  A sample whose ratio lies within tf32 rounding of 1 +- clip carries its whole
    surrogate gradient or none of it, a jump no precision bar for the other samples covers."""
    N, T, theta, data, mu_old, logstd_old, perm = _mb_data(O, A, count)
    ref = _mb_ref(O, A, count, regime)
    idx = perm[START:START + count]
    Pa = oac.layout(O, A)['actor']['size']
    obs, act, logp = data['obs'][idx], f64._t64(data['act'][idx]), f64._t64(data['logp'][idx])
    adv_r = (f64._t64(data['adv_r'][idx]) - MOMENTS[0]) / MOMENTS[1]
    adv_c = f64._t64(data['adv_c'][idx]) - MOMENTS[2]
    q = f64._leaves(theta[:Pa], O)
    h1 = torch.tanh(_rna(obs) @ _rna(q['w1']).T + q['b1'])
    h2 = torch.tanh(_rna(h1) @ _rna(q['w2']).T + q['b2'])
    mu_t = _rna(h2) @ _rna(q['w3']).T + q['b3']

    def ratio_of(mu, log_std):
        return torch.exp(Normal(mu, torch.exp(log_std)).log_prob(act).sum(-1) - logp)

    def active(r):      # the unclipped branch carries the gradient: s1 <= s2
        return torch.where(adv_r >= 0, r <= 1.2, r >= 0.8)
    a64 = active(ratio_of(torch.as_tensor(f64.mean64(theta[:Pa], obs)), q['log_std']))
    a_t = active(ratio_of(mu_t, q['log_std']))
    p = f64._leaves(theta[:Pa], O, grad=True)
    d = oac.actor_dist(p, f64._t64(obs))
    ratio = torch.exp(d.log_prob(act).sum(-1) - logp)
    loss = -(a_t.double() * ratio * adv_r).mean() - ENT * d.entropy().mean()
    if ref['info']['gate']:
        loss = loss + ref['lam_f'] * ((ratio * adv_c).mean() + ref['eta'])
    loss.backward()
    return torch.cat([v.grad.reshape(-1) for v in p.values()]).numpy(), int((a64 != a_t).sum())


def _check_grad(path, got, want, O, A, kind, clip_ref=None):
    """Per parameter block: fp32 / bf16x3 l2 1e-4 + rtol 2e-4 / atol 2e-5 x block max; tf32 5e-3 (2e-2 on the actor
    of P3O, whose PPO clip flips near the boundary) and cos > 0.9999.  A block whose reference is zero (the actor
    weights of an all-out FOCOPS mask) must be zero."""
    lay = oac.layout(O, A)
    worst = 0.0
    for net in o64.NETS:
        for name, (off, shape) in lay[net]['entries'].items():
            n = int(np.prod(shape))
            g, w = got[off:off + n], want[off:off + n]
            if not w.any():
                assert not g.any(), (net, name, np.abs(g).max())
                continue
            rel = float(np.linalg.norm(g - w) / np.linalg.norm(w))
            worst = max(worst, rel)
            if path == 'tf32' and net == 'actor' and kind == P3O:
                # 2e-2 against float64 and against float64 with the tf32 clip decisions; cos > 0.9999 against the
                # latter (a flipped decision is a jump of one sample's whole gradient, not a rounding error)
                wc = clip_ref[off:off + n]
                rel_c = float(np.linalg.norm(g - wc) / np.linalg.norm(wc))
                cos = float((g * wc).sum() / (np.linalg.norm(g) * np.linalg.norm(wc)))
                assert rel < 2e-2 and rel_c < 2e-2 and cos > 0.9999, (net, name, rel, rel_c, cos)
            elif path == 'tf32':
                cos = float((g * w).sum() / (np.linalg.norm(g) * np.linalg.norm(w)))
                assert rel < 5e-3 and cos > 0.9999, (net, name, rel, cos)
            else:
                assert rel < 1e-4, (net, name, rel)
                np.testing.assert_allclose(g, w, rtol=2e-4, atol=2e-5 * np.abs(w).max(), err_msg=f'{net}.{name}')
    return worst


MB_CASES = [(path, O, A, count, regime) for O, A, count in SIZES for path in FNS for regime in REGIME_KIND
            if not (path == 'bf16x3' and O > 64)]


@pytest.mark.timeout(300)
@pytest.mark.parametrize('path,O,A,count,regime', MB_CASES)
def test_two_pass_minibatch_grad_vs_fp64(cuda, path, O, A, count, regime):
    lib, ptr, stream = _lib()
    N, T, theta, data, mu_old, logstd_old, perm = _mb_data(O, A, count)
    ref = _mb_ref(O, A, count, regime)
    agent, buf, eng = _setup(cuda, data, N, T, O, A, theta)
    buf.adv_moments.copy_(torch.tensor(MOMENTS))
    eng.mu_old.copy_(_slab(mu_old, N, T))
    eng.logstd_old.copy_(torch.as_tensor(logstd_old))
    eng.train_stats.zero_()
    # rows a kernel does not write must not be read: poison the partials
    eng.gpart.fill_(float('nan'))
    eng.stats_part.fill_(float('nan'))
    lag = torch.tensor([LAM], dtype=torch.float32, device=cuda) if ref['kind'] == FOCOPS else None
    rows = torch.as_tensor(_rows(perm, N, T)).to(cuda)
    d = buf.data
    rc = getattr(lib, FNS[path])(
        ptr(agent.theta), O, A, ptr(d['obs']), ptr(d['act']), ptr(d['logp']), ptr(d['adv_r']), ptr(d['adv_c']),
        ptr(d['target_value_r']), ptr(d['target_value_c']), ptr(eng.mu_old), ptr(buf.adv_moments), ptr(rows), N * T, 0,
        START, count, ref['kind'], 0.2, ENT, ref['lam_f'], ref['eta'], ptr(lag), ptr(eng.logstd_old), 7, ptr(eng.gpart),
        ptr(eng.stats_part), 0, stream)
    assert rc == 0, rc
    if path == 'fp32':
        nb = nb1 = lib.osb_update_grid_blocks(count)
    else:
        nb, nb1 = lib.osb_tc_grid_blocks(count, 7), lib.osb_tc_grid_blocks(count, 1)
    lib.osb_grad_reduce(ptr(eng.gpart), ptr(eng.stats_part), nb, O, A, ptr(agent.theta), ptr(agent.grad), COEF, 7,
                        ptr(eng.sumsq_part), ptr(agent.adam_step), ptr(eng.train_stats), 0, stream)
    torch.cuda.synchronize()
    if path != 'fp32' and count >= 16384:
        assert nb1 > nb, (nb1, nb)
    got = agent.grad.cpu().numpy().astype(np.float64)
    assert np.isfinite(got).all()
    clip_ref, flips = (None, 0)
    if path == 'tf32' and ref['kind'] == P3O:
        clip_ref, flips = _tf32_clip_reference(O, A, count, regime)
    worst = _check_grad(path, got, ref['grad'], O, A, ref['kind'], clip_ref)
    info = ref['info']
    ts = eng.train_stats.cpu().numpy().reshape(3, 8).astype(np.float64)
    st = eng.stats_part.cpu().numpy()[:nb * 24].reshape(nb, 3, 8).astype(np.float64)
    assert st[:, 0, 3].sum() == count
    slot4 = st[:, 0, 4].sum() / count
    want = info['stats']
    margin = 'gap/2 around eta' if ref['kind'] == FOCOPS else '|mean + Jc - limit|'
    print(f'[{path} O={O} A={A} count={count} {regime}] nb1 {nb1} nb {nb}; worst block l2 {worst:.2e}'
          + (f' ({flips} PPO-clip decisions of a tf32 forward differ from float64)' if clip_ref is not None else '') + '; '
          f'{margin} {info["margin"]:.3e}; pass 1 {info["pass1"]:.6g}; slots 0/2/4 '
          f'{ts[0, 0]:.6g}/{ts[0, 2]:.6g}/{slot4:.6g} vs {want[0]:.6g}/{want[2]:.6g}/{want[3]:.6g}')
    rtol = 5e-3 if path == 'tf32' else 1e-3
    np.testing.assert_allclose(ts[0, 0], want[0], rtol=rtol, atol=1e-4, err_msg='slot 0')
    np.testing.assert_allclose(ts[0, 1], want[1], rtol=rtol, atol=1e-4, err_msg='slot 1 (ratio)')
    np.testing.assert_allclose(ts[0, 2], want[2], rtol=rtol, atol=1e-4, err_msg='slot 2')
    if ref['kind'] == FOCOPS:      # the mask decisions themselves (tf32: a KL error of ~1e-4 may flip a sample)
        assert abs(slot4 - want[3]) <= (2.0 / count if path == 'tf32' else 0.0), (slot4, want[3])
    else:
        assert not st[:, 0, 4].any()


# ---- b: whole epochs --------------------------------------------------------------------------------------------------

def _gate_flip(data, perms, batch, seed, shift=0.5):
    """P3O data whose gate changes between minibatches: adv_c + shift on the rows of pass 0's even minibatches, - shift
    on the others; every later pass takes its minibatches from one of the two groups at a time (the shuffled first
    group, then the shuffled second), so every minibatch mean of ratio * adv_c is ~+-shift."""
    rng = np.random.default_rng(seed)
    data = dict(data)
    B = perms.shape[1]
    first = np.concatenate([perms[0][s:s + batch] for s in range(0, B, 2 * batch)])
    second = np.setdiff1d(perms[0], first)
    adv_c = data['adv_c'].copy()
    adv_c[first] += np.float32(shift)
    adv_c[second] -= np.float32(shift)
    data['adv_c'] = adv_c
    out = [perms[0]] + [np.concatenate([rng.permutation(first), rng.permutation(second)]) for _ in perms[1:]]
    return data, np.stack(out)


def _kind_args(kind):
    """(Lagrange multiplier, focops_lam, focops_eta): P3O with Jc - limit = 0 on gate-flip data; FOCOPS's eta comes
    from _focops_eta."""
    return (LAM, FOCOPS_LAM, None) if kind == FOCOPS else (0.0, KAPPA, 0.0)


def _focops_eta(theta, data, perms, lam, factor, **kw):
    """`factor` x the full-batch mean KL after one all-in pass: the first step's KLs are 0 (all in), later steps cut
    the growing KLs, so the mask mean changes from minibatch to minibatch and every pass-1 reduction matters."""
    kw = dict(kw, focops_eta=1e9)
    _, rec, _ = o64.ppo_epoch64(theta, data, MOMENTS, perms[:1], lam, update_iters=1, **kw)
    return factor * rec['kl'][0]


def _check_decisions(kind, rec, lam_f):
    """FOCOPS: the mask means start at 1 and take at least three values below it.  Mixed masks of 8 192 KLs have
    samples within fp32 rounding of eta (margins printed); a flipped sample moves the gradient by ~1 / batch, inside
    the epoch bars.  P3O: both gate states, each at least 0.05 from the relu boundary."""
    margins = np.array([r['margin'] for r in rec['steps']])
    if kind == FOCOPS:
        means = np.array([r['pass1'] for r in rec['steps']])
        assert means[0] == 1.0 and len(set(means[means < 1.0])) >= 3, means
    else:
        gates = {r['gate'] for r in rec['steps']}
        assert gates == {0.0, lam_f} and (margins >= 0.05).all(), (gates, margins)
    return margins.min()


def _device_epoch(cuda, O, A, N, T, theta, data, precision):
    agent, buf, eng = _setup(cuda, data, N, T, O, A, theta)
    buf.adv_moments.copy_(torch.tensor(MOMENTS))
    eng.precision = precision
    eng.train_stats.zero_()
    return agent, buf, eng


def _one_step(eng, agent, buf, rows, *, kind, lam, lam_f, eta, batch, max_norm, coef):
    """The first minibatch through the path's gradient kernel + osb_optim_fused, after the old-policy snapshot."""
    lib, ptr, stream = _lib()
    O, A = eng.O, eng.A
    path = 'bf16x3' if eng._x3() else 'tf32' if eng._tc() else 'fp32'
    eng.snapshot_old_policy()
    lag = torch.tensor([lam], dtype=torch.float32, device=agent.theta.device) if kind == FOCOPS else None
    d = buf.data
    rc = getattr(lib, FNS[path])(
        ptr(agent.theta), O, A, ptr(d['obs']), ptr(d['act']), ptr(d['logp']), ptr(d['adv_r']), ptr(d['adv_c']),
        ptr(d['target_value_r']), ptr(d['target_value_c']), ptr(eng.mu_old), ptr(buf.adv_moments), ptr(rows),
        rows.numel(), 0, 0, batch, kind, 0.2, ENT, lam_f, eta, ptr(lag), ptr(eng.logstd_old), 7, ptr(eng.gpart),
        ptr(eng.stats_part), ptr(eng.stop_flag), stream)
    assert rc == 0, rc
    nb = lib.osb_update_grid_blocks(batch) if path == 'fp32' else lib.osb_tc_grid_blocks(batch, 7)
    lib.osb_optim_fused(ptr(eng.gpart), ptr(eng.stats_part), nb, O, A, ptr(agent.theta), ptr(agent.grad),
                        ptr(agent.adam_m), ptr(agent.adam_v), ptr(agent.adam_step), coef, max_norm, LRS[0], LRS[1],
                        LRS[1], 7, ptr(eng.sumsq_part), ptr(eng.train_stats), ptr(eng.stop_flag), stream)
    torch.cuda.synchronize()
    return path


def _compare_actor_slot2(path, eng, rec):
    ts = eng.train_stats.cpu().numpy().reshape(3, 8)
    n = len(rec['steps'])
    want = np.mean([r['stats'][2] for r in rec['steps']])
    np.testing.assert_allclose(ts[0, 2] / n, want, rtol=5e-3 if path == 'tf32' else 1e-3, atol=1e-5,
                               err_msg='logged slot 2 of the actor')


EPOCH_CASES = [(kind, precision, 60) for kind in (FOCOPS, P3O) for precision in (0, 1, 2)]
EPOCH_CASES += [(FOCOPS, 2, 111), (P3O, 2, 111)]      # obs dims > 64 at precision 2: the fp32 tiles, the fp32 bars


@pytest.mark.timeout(600)
@pytest.mark.parametrize('kind,precision,O', EPOCH_CASES)
def test_two_pass_epoch_vs_fp64(cuda, kind, precision, O):
    """UpdateEngine.ppo_epoch (launch per minibatch on every path: the two-pass kinds never take the persistent
    bf16x3 kernel) vs ppo_epoch64, every network clipping: one step, then two passes over 3.5 minibatches of 8 192
    rows (short last one) -- theta, m, v, adam_step, the logged losses and the actor's slot 2, the final KL."""
    A, batch = 8, 8192
    rows_n = batch * 7 // 2
    T = 64
    N = rows_n // T
    theta, data, perms = _regime_data(O, A, N, T, 'all', seed=O + kind)
    if kind == P3O:
        data, perms = _gate_flip(data, perms, batch, seed=O)
    _, max_norm, coef = REGIMES['all']
    lam, lam_f, eta = _kind_args(kind)
    lrs = (LRS[0], LRS[1], LRS[1])          # ppo_epoch takes one critic learning rate
    kw = dict(net_mask=7, loss_kind=kind, batch_size=batch, critic_norm_coef=coef, max_grad_norm=max_norm, lrs=lrs,
              clip=0.2, entropy_coef=ENT, focops_lam=lam_f, focops_eta=eta)
    t0 = time.perf_counter()
    if kind == FOCOPS:
        # twice the KL: the masks turn mixed in the second pass while the actor gradient stays above max_grad_norm
        eta = kw['focops_eta'] = _focops_eta(theta, data, perms, lam, 2.0, **kw)
    one, rec1, _ = o64.ppo_epoch64(theta, data, MOMENTS, perms[:1, :batch], lam, update_iters=1, **kw)
    want, rec, passes = o64.ppo_epoch64(theta, data, MOMENTS, perms, lam, update_iters=2, **kw)
    t_ref = time.perf_counter() - t0
    assert passes == 2 and len(rec['steps']) == 8
    _check_regime(rec, 'all', 7)
    margin = _check_decisions(kind, rec, lam_f)
    rows = torch.as_tensor(np.stack([_rows(p, N, T) for p in perms])).to(cuda)
    run = dict(kind=kind, lam=lam, lam_f=lam_f, eta=eta, batch=batch, max_norm=max_norm, coef=coef)
    agent, buf, eng = _device_epoch(cuda, O, A, N, T, theta, data, precision)
    path = _one_step(eng, agent, buf, rows[0].contiguous(), **run)
    got1 = _host(agent)
    assert (got1['step'] == 1).all(), got1['step']
    w1 = _compare_step(path, got1, one, rec1['steps'][0], O, A, 7, max_norm)
    agent, buf, eng = _device_epoch(cuda, O, A, N, T, theta, data, precision)
    lag = torch.tensor([lam, 0, 0, 0], dtype=torch.float32, device=cuda) if kind == FOCOPS else None
    eng.ppo_epoch(loss_kind=kind, lagrange=lag, net_mask=7, batch_size=batch, update_iters=2, clip=0.2,
                  entropy_coef=ENT, focops_lam=lam_f, focops_eta=eta, critic_norm_coef=coef, max_grad_norm=max_norm,
                  lr_actor=lrs[0], lr_critic=lrs[1], target_kl=10.0, kl_early_stop=False, perm=rows)
    torch.cuda.synchronize()
    got = _host(agent)
    np.testing.assert_array_equal(got['step'], want['step'])
    assert (got['step'] == 8).all()
    we = _compare_epoch(path, got, want, theta, O, A, 7)
    _compare_stats(path, eng, rec, 7)
    _compare_actor_slot2(path, eng, rec)
    kl = float(eng.kl_state[0])
    np.testing.assert_allclose(kl, rec['kl'][-1], rtol=0.3 if path == 'tf32' else 2e-2)
    if kind == P3O:
        decisions = 'P3O gates ' + ''.join('1' if r['gate'] else '0' for r in rec['steps'])
    else:
        decisions = f'FOCOPS eta {eta:.3g}, mask means ' + ' '.join(f'{r["pass1"]:.3g}' for r in rec['steps'])
    print(f'[{path} kind {kind} O={O}] float64 reference {t_ref:.1f} s; decision margin {margin:.3g}, {decisions}; '
          f'one step worst block l2 {w1:.2e}; epoch ' + ', '.join(f'{k} {v:.2e}' for k, v in we.items()) +
          f'; KL {kl:.4g} vs {rec["kl"][-1]:.4g}')


@pytest.mark.timeout(600)
@pytest.mark.parametrize('precision', [0, 1, 2])
@pytest.mark.parametrize('kind', [FOCOPS, P3O])
def test_two_pass_kl_stop(cuda, kind, precision):
    """A KL early stop after the first of three passes: adam_step = the minibatches of one pass and theta / m / v of
    that pass -- the pass-1 launches, pass1_gate and the pass-2 launches of the stopped passes change nothing."""
    O, A, N, T, batch = 60, 8, 32, 112, 1024
    theta, data, _ = _regime_data(O, A, N, T, 'critics', 21 + kind)
    # reward advantages half a standard deviation above their mean: the logged FOCOPS loss (mean(m kl) - mean(m)
    # mean(ratio adv) / lam) then does not cancel to ~1e-3, where mask flips at tf32 rounding would dominate it
    data['adv_r'] = (data['adv_r'] + np.float32(0.5 * MOMENTS[1])).astype(np.float32)
    rng = np.random.default_rng(22 + kind)
    perms = np.stack([rng.permutation(N * T) for _ in range(3)])
    if kind == P3O:
        data, perms = _gate_flip(data, perms, batch, seed=23)
    _, max_norm, coef = REGIMES['critics']
    lam, lam_f, eta = _kind_args(kind)
    lrs = (LRS[0], LRS[1], LRS[1])
    kw = dict(net_mask=7, loss_kind=kind, batch_size=batch, critic_norm_coef=coef, max_grad_norm=max_norm, lrs=lrs,
              clip=0.2, entropy_coef=ENT, focops_lam=lam_f, focops_eta=eta)
    if kind == FOCOPS:
        eta = kw['focops_eta'] = _focops_eta(theta, data, perms, lam, 0.5, **kw)
    s1, r1, p1 = o64.ppo_epoch64(theta, data, MOMENTS, perms, lam, update_iters=3, target_kl=1e-12, kl_early_stop=True,
                                 **kw)
    n_mb = -(-N * T // batch)
    assert p1 == 1 and len(r1['steps']) == n_mb
    if kind == P3O:
        assert {r['gate'] for r in r1['steps']} == {0.0, lam_f} and min(r['margin'] for r in r1['steps']) >= 0.05
    else:       # the mask mean changes within the pass that runs
        means = [r['pass1'] for r in r1['steps']]
        assert means[0] == 1.0 and min(means) < 1.0, means
    agent, buf, eng = _device_epoch(cuda, O, A, N, T, theta, data, precision)
    path = 'bf16x3' if eng._x3() else 'tf32' if eng._tc() else 'fp32'
    lag = torch.tensor([lam, 0, 0, 0], dtype=torch.float32, device=cuda) if kind == FOCOPS else None
    rows = torch.as_tensor(np.stack([_rows(p, N, T) for p in perms])).to(cuda)
    eng.ppo_epoch(loss_kind=kind, lagrange=lag, net_mask=7, batch_size=batch, update_iters=3, clip=0.2,
                  entropy_coef=ENT, focops_lam=lam_f, focops_eta=eta, critic_norm_coef=coef, max_grad_norm=max_norm,
                  lr_actor=lrs[0], lr_critic=lrs[1], target_kl=1e-12, kl_early_stop=True, perm=rows)
    torch.cuda.synchronize()
    got = _host(agent)
    kls = eng.kl_state.cpu().numpy()
    assert int(kls[1]) == 1 and kls[2] == 1.0, kls
    assert (got['step'] == n_mb).all(), got['step']
    _compare_stats(path, eng, r1, 7)
    _compare_actor_slot2(path, eng, r1)
    w = _compare_epoch(path, got, s1, theta, O, A, 7)
    means = ' '.join(f'{r["pass1"]:.3g}' for r in r1['steps']) if kind == FOCOPS else '-'
    print(f'[{path} kind {kind}] KL stop after pass 1 of 3: adam_step {got["step"].tolist()}; FOCOPS mask means '
          f'{means}; ' +
          ', '.join(f'{k} {v:.2e}' for k, v in w.items()))
