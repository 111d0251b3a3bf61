"""GPU: the optimiser step that ends every minibatch -- partial-gradient reduction, critic L2 term, per-network
clip_grad_norm_, (several ranks: average) and torch Adam -- on every device path, with clipping active, against the
float64 reference oracle/optim64.py (pinned to the float32 oracle and the PPOLag golden in test_optimizer_ref_cpu).

  a. osb_optim_fused, osb_grad_reduce + osb_clip_adam, and the split NCCL-order sequence of two ranks emulated on
     one GPU, on synthetic partial gradients: 288 consecutive steps with the Adam state carried over, three learning
     rates, and per step a different nblocks x critic_norm_coef x max_grad_norm x net_mask combination.
  b. The clipping invariant: a clipped network's stored gradient has norm max_grad_norm * n / (n + 1e-6), an
     unclipped one keeps its norm -- on every path and precision.
  c. Whole update passes from the minibatch gradient kernels (fp32, tf32, bf16x3 stepwise) and from the persistent
     bf16x3 kernel (speculative Adam, its redo when a network clips, and the non-speculative slices), in three
     clipping regimes, against ppo_epoch64; a KL early stop and a second ppo_epoch continuing the Adam state.

Device calls go through the C ABI or UpdateEngine with explicit sample orders.  Each case prints its worst error."""
import os

import numpy as np
import pytest
import torch

from oracle import actor_critic as oac
from oracle import optim64 as o64
from test_update_gpu import _default_spec_after, _rand_data, _rows, _setup, _theta, net_cases, oracle_nets, sigma_cases  # noqa: F401

pytestmark = pytest.mark.gpu

MOMENTS = [0.37, 2.3, -0.41, 1.0]
LAM = 0.37
LRS = (3e-4, 1e-3, 2.5e-3)          # actor, reward critic, cost critic: all different
# at a trained log_std: the actor at lr 1e-2, so log_std moves ~1e-2 per minibatch step, with the entropy bonus on
LRS_TRAINED, ENT_TRAINED = (1e-2, 1e-3, 2.5e-3), 0.01
NEPI = 512                          # parameters one CTA of the persistent bf16x3 kernel updates in one pass

# ---- helpers -------------------------------------------------------------------------------------------------------


def _lib():
    from omnisafe_b200._lib import current_stream, lib, ptr
    return lib(), ptr, current_stream()


def _host(agent):
    return {'theta': agent.theta.cpu().numpy().astype(np.float64), 'm': agent.adam_m.cpu().numpy().astype(np.float64),
            'v': agent.adam_v.cpu().numpy().astype(np.float64), 'step': agent.adam_step[:3].cpu().numpy().astype(np.int64),
            'grad': agent.grad.cpu().numpy().astype(np.float64)}


def _slices(O, A):
    lay = oac.layout(O, A)
    return [slice(lay[n]['start'], lay[n]['start'] + lay[n]['size']) for n in o64.NETS]


def _l2(got, want):
    return float(np.linalg.norm(got - want) / max(np.linalg.norm(want), 1e-300))


def _check_invariant(grad, rec, k, sl, max_norm, rtol_unclipped):
    """Part b for network k: a clipped network's gradient norm is max_norm * n / (n + 1e-6) (to fp32 rounding
    whatever the precision of n); an unclipped one keeps the norm n."""
    got = float(np.linalg.norm(grad[sl]))
    n = rec['norm'][k]
    if rec['coef'][k] < 1.0:
        want = max_norm * n / (n + 1e-6)
        assert abs(got - want) <= 1e-5 * want, ('clipped norm', k, got, want)
    else:
        assert abs(got - n) <= rtol_unclipped * n, ('unclipped norm', k, got, n)
    return got


# ---- a + b: optimiser kernels on synthetic partial gradients ----------------------------------------------------------

SHAPES_A = [(1, 1), (17, 6), (60, 8), (64, 16), (376, 8)]
NBLOCKS = [1, 15, 16, 17, 33, 148]
COEFS = [0.0, 0.05]
MAX_NORMS = [0.0, 1e-4, 0.3, 1e6]   # 0: clipping off; 1e-4: clipped norms small enough that the + 1e-6 shows
MASKS = [1, 2, 3, 4, 6, 7]
STEPS = len(NBLOCKS) * len(COEFS) * len(MAX_NORMS) * len(MASKS)      # 288: every combination once


def _combo(k):
    nb = NBLOCKS[k % 6]
    coef = COEFS[(k // 6) % 2]
    max_norm = MAX_NORMS[(k // 12) % 4]
    return nb, coef, max_norm, MASKS[k // 48]


def _synthetic_grads(gen, P, sls, nb, max_norm, clip_mask, cuda):
    """[nb][P] float32 partials whose sum has, per network, norm 10 * max_norm (clip_mask bit set) or 0.1 * max_norm;
    with clipping off, norm 1e3 (large gradients that must pass unchanged)."""
    gpart = torch.randn(nb, P, generator=gen, device=cuda)
    for k, sl in enumerate(sls):
        target = 1e3 if max_norm <= 0 else (10.0 if (clip_mask >> k) & 1 else 0.1) * min(max_norm, 1e3)
        n = sl.stop - sl.start
        gpart[:, sl] *= target / np.sqrt(n * nb)
    return gpart


# the two-rank sequence runs the clip_adam kernel of reduce_clip_adam; its grid-wide norm fold over > 32 CTAs
# (O = 376) is covered there, so the two-rank case skips that shape and its three float64 steps per step
SYNTH_CASES = [(path, O, A) for path in ('optim_fused', 'reduce_clip_adam', 'nccl_order_2ranks') for O, A in SHAPES_A
               if not (path == 'nccl_order_2ranks' and O > 64)]


@pytest.mark.timeout(600)
@pytest.mark.parametrize('path,O,A', SYNTH_CASES)
def test_optimizer_steps_vs_fp64(cuda, path, O, A):
    """288 steps; every step checks theta, m, v, the stored (clipped) gradient, adam_step and train_stats rows 0-3
    against step64 and the float64 sums of the partials / loss statistics."""
    lib, ptr, stream = _lib()
    theta0 = oac.init_theta(O, A, seed=O + A)
    rng = np.random.default_rng(O * 7 + A)
    data = _rand_data(rng, 4, 4, O, A, theta0)
    agent, buf, eng = _setup(cuda, data, 4, 4, O, A, theta0)
    P, sls = eng.P, _slices(O, A)
    gen = torch.Generator(device=cuda).manual_seed(O + 100 * A)
    ref = o64.init_state(theta0)
    ts_ref = np.zeros((3, 8))
    worst = dict.fromkeys(('theta', 'm', 'v', 'grad', 'stats', 'invariant'), 0.0)
    seen = set()
    for k in range(STEPS):
        nb, coef, max_norm, mask = _combo(k)
        clip_mask = int(rng.integers(0, 8))
        gpart = _synthetic_grads(gen, P, sls, nb, max_norm, clip_mask, cuda)
        stats = torch.rand(nb, 3, 8, generator=gen, device=cuda)
        stats[:, :, 3] = torch.randint(1, 129, (nb, 3), generator=gen, device=cuda).float()   # rows per CTA
        eng.gpart[:nb * P].copy_(gpart.reshape(-1))
        eng.stats_part[:nb * 24].copy_(stats.reshape(-1))
        gsum = gpart.double().sum(0).cpu().numpy()
        ssum = stats.double().sum(0).cpu().numpy()
        before = ref
        ref, rec = o64.step64(ref, gsum, max_grad_norm=max_norm, lrs=LRS, critic_norm_coef=coef, O=O, net_mask=mask)
        if path == 'optim_fused':
            lib.osb_optim_fused(ptr(eng.gpart), ptr(eng.stats_part), nb, O, A, ptr(agent.theta), ptr(agent.grad),
                                ptr(agent.adam_m), ptr(agent.adam_v), ptr(agent.adam_step), coef, max_norm, *LRS, mask,
                                ptr(eng.sumsq_part), ptr(eng.train_stats), ptr(eng.stop_flag), stream)
        else:
            lib.osb_grad_reduce(ptr(eng.gpart), ptr(eng.stats_part), nb, O, A, ptr(agent.theta), ptr(agent.grad), coef,
                                mask, ptr(eng.sumsq_part), ptr(agent.adam_step), ptr(eng.train_stats),
                                ptr(eng.stop_flag), stream)
            if path == 'reduce_clip_adam':
                lib.osb_clip_adam(ptr(agent.grad), ptr(agent.theta), ptr(agent.adam_m), ptr(agent.adam_v),
                                  ptr(agent.adam_step), ptr(eng.sumsq_part), O, A, max_norm, *LRS, 1.0, coef,
                                  ptr(eng.train_stats), 1, 1, mask, ptr(eng.stop_flag), stream)
            else:
                # rank 0 clips its own gradient, a second rank's clipped gradient is summed in (the all-reduce), then
                # Adam on the sum / 2: policy_gradient.py:L437-443 + distributed.py avg_grads
                lib.osb_clip_adam(ptr(agent.grad), ptr(agent.theta), ptr(agent.adam_m), ptr(agent.adam_v),
                                  ptr(agent.adam_step), ptr(eng.sumsq_part), O, A, max_norm, *LRS, 1.0, coef,
                                  ptr(eng.train_stats), 1, 0, mask, ptr(eng.stop_flag), stream)
                clipped0 = agent.grad.cpu().numpy().astype(np.float64)
                g1 = gpart[0].double().cpu().numpy()[::-1].copy() * 3.0        # the second rank's gradient
                _, rec1 = o64.step64(before, g1, max_grad_norm=max_norm, lrs=LRS, critic_norm_coef=coef, O=O,
                                     net_mask=mask)
                g1c = rec1['grad'].astype(np.float32)
                agent.grad.add_(torch.as_tensor(g1c).to(cuda))
                lib.osb_clip_adam(ptr(agent.grad), ptr(agent.theta), ptr(agent.adam_m), ptr(agent.adam_v),
                                  ptr(agent.adam_step), ptr(eng.sumsq_part), O, A, max_norm, *LRS, 0.5, coef,
                                  ptr(eng.train_stats), 0, 1, mask, ptr(eng.stop_flag), stream)
                avg = 0.5 * (rec['grad'] + g1c.astype(np.float64))
                ref, _ = o64.step64(before, avg, max_grad_norm=0.0, lrs=LRS, critic_norm_coef=0.0, O=O, net_mask=mask)
        torch.cuda.synchronize()
        got = _host(agent)
        ts = eng.train_stats.cpu().numpy().reshape(3, 8).astype(np.float64)
        for j, sl in enumerate(sls):
            if not (mask >> j) & 1:
                continue
            seen.add((j, max_norm, rec['coef'][j] < 1.0))
            ts_ref[j, :3] += ssum[j, :3] / ssum[j, 3]
            ts_ref[j, 0] += rec['l2'][j]
            ts_ref[j, 3] += 1
            want_grad = rec['grad'][sl]
            if path == 'nccl_order_2ranks':
                worst['invariant'] = max(worst['invariant'], abs(_check_invariant(clipped0, rec, j, sl, max_norm, 1e-5)
                                                                 / np.linalg.norm(want_grad) - 1.0))
                want_grad = want_grad + g1c[sl]
            else:
                worst['invariant'] = max(worst['invariant'], abs(_check_invariant(got['grad'], rec, j, sl, max_norm, 1e-5)
                                                                 / np.linalg.norm(want_grad) - 1.0))
            errs = {'grad': _l2(got['grad'][sl], want_grad), 'm': _l2(got['m'][sl], ref['m'][sl]),
                    'v': _l2(got['v'][sl], ref['v'][sl]),
                    'theta': _l2(got['theta'][sl] - theta0[sl], ref['theta'][sl] - theta0[sl])}
            for key, e in errs.items():
                worst[key] = max(worst[key], e)
                # the suite's 1e-4 l2 bar; at max_grad_norm 1e-4 a dropped + 1e-6 moves grad and m by 1e-3
                assert e < 1e-4, (k, j, key, e, nb, coef, max_norm, mask)
        np.testing.assert_array_equal(got['step'], ref['step'])
        np.testing.assert_allclose(ts[:, :4], ts_ref[:, :4], rtol=2e-5, atol=1e-6, err_msg=f'train_stats, step {k}')
        worst['stats'] = max(worst['stats'], float(np.abs(ts[:, :4] - ts_ref[:, :4]).max() / np.abs(ts_ref).max()))
    print(f'[{path} O={O} A={A}] worst l2-rel over {STEPS} steps: ' +
          ', '.join(f'{key} {e:.2e}' for key, e in worst.items()))
    # every network in a mask took part clipped and not clipped under max_grad_norm 0.3 and 1e-4
    for j in range(3):
        for mx in (1e-4, 0.3):
            assert (j, mx, True) in seen and (j, mx, False) in seen, (j, mx)
        assert not any(c for (jj, mx, c) in seen if jj == j and mx in (0.0, 1e6))


def test_stop_flag_is_a_noop(cuda):
    """With the device stop flag set (KL early stop), every optimiser entry point and the persistent bf16x3 pass
    leave theta, grad, m, v, adam_step and train_stats bit-identical."""
    lib, ptr, stream = _lib()
    O, A, N, T = 60, 8, 32, 48
    theta0 = oac.init_theta(O, A, seed=3)
    data = _rand_data(np.random.default_rng(4), N, T, O, A, theta0)
    agent, buf, eng = _setup(cuda, data, N, T, O, A, theta0)
    P, B = eng.P, N * T
    g = torch.Generator(device=cuda).manual_seed(0)
    agent.adam_m.copy_(torch.randn(P, generator=g, device=cuda))
    agent.adam_v.copy_(torch.rand(P, generator=g, device=cuda))
    agent.adam_step.fill_(5)
    agent.grad.copy_(torch.randn(P, generator=g, device=cuda))
    eng.train_stats.copy_(torch.randn(24, generator=g, device=cuda))
    eng.gpart.normal_(generator=g)
    eng.stats_part.uniform_(1.0, 2.0, generator=g)
    eng.stop_flag.fill_(1)
    lag = torch.tensor([LAM, 0, 0, 0], dtype=torch.float32, device=cuda)
    d = buf.data
    bufs = (agent.theta, agent.grad, agent.adam_m, agent.adam_v, agent.adam_step, eng.train_stats)
    snap = [b.clone() for b in bufs]
    calls = {
        'osb_optim_fused': lambda: lib.osb_optim_fused(
            ptr(eng.gpart), ptr(eng.stats_part), 17, O, A, ptr(agent.theta), ptr(agent.grad), ptr(agent.adam_m),
            ptr(agent.adam_v), ptr(agent.adam_step), 0.05, 0.3, *LRS, 7, ptr(eng.sumsq_part), ptr(eng.train_stats),
            ptr(eng.stop_flag), stream),
        'osb_grad_reduce': lambda: lib.osb_grad_reduce(
            ptr(eng.gpart), ptr(eng.stats_part), 17, O, A, ptr(agent.theta), ptr(agent.grad), 0.05, 7,
            ptr(eng.sumsq_part), ptr(agent.adam_step), ptr(eng.train_stats), ptr(eng.stop_flag), stream),
        'osb_clip_adam': lambda: lib.osb_clip_adam(
            ptr(agent.grad), ptr(agent.theta), ptr(agent.adam_m), ptr(agent.adam_v), ptr(agent.adam_step),
            ptr(eng.sumsq_part), O, A, 0.3, *LRS, 1.0, 0.05, ptr(eng.train_stats), 1, 1, 7, ptr(eng.stop_flag), stream),
        'osb_ppo_update_iter_x3': lambda: lib.osb_ppo_update_iter_x3(
            ptr(agent.theta), ptr(agent.grad), ptr(agent.adam_m), ptr(agent.adam_v), ptr(agent.adam_step), O, A,
            ptr(d['obs']), ptr(d['act']), ptr(d['logp']), ptr(d['adv_r']), ptr(d['adv_c']), ptr(d['target_value_r']),
            ptr(d['target_value_c']), ptr(buf.adv_moments), 0, B, 7, 512, 0, 0.2, 0.0, ptr(lag), 7, 0.05, 0.3, *LRS,
            ptr(eng.gpart), ptr(eng.stats_part), ptr(eng.train_stats), ptr(eng.stop_flag), 0, 0, 1, 0, 0, stream),
    }
    for name, call in calls.items():
        call()
        torch.cuda.synchronize()
        for b, s in zip(bufs, snap):
            assert torch.equal(b, s), name
        print(f'{name}: no-op with the stop flag set')


# ---- c: whole update passes vs ppo_epoch64 ---------------------------------------------------------------------------

REGIMES = {   # critic-target scale, max_grad_norm, critic_norm_coef; the norms are far from the threshold (asserted)
    'critics': (50.0, 1.5, 0.05),   # critic gradients ~3-17, actor ~0.05-0.6: only the critics clip
    'all': (1.0, 0.02, 0.05),       # every network clips
    'none': (1.0, 40.0, 0.05),      # none does
    'small': (None, 1e-4, 0.0),     # every network clips at norms < 0.03 on the first step, so the + 1e-6 shows
}
# critic_norm_coef 0.05: the L2 term is about half of the critic norm, so leaving it out of the norm is visible. The
# 'small' regime has no L2 term, advantages of 1e-2 standard deviations and critic targets within ~0.1 of the values.


def _regime_data(O, A, N, T, regime, seed, trained=False, nets=None):
    rng = np.random.default_rng(seed)
    theta = _theta(O, A, seed % 7, trained, nets)
    data = _rand_data(rng, N, T, O, A, theta, nets)
    data['adv_r'] = (data['adv_r'] * np.float32(MOMENTS[1]) + np.float32(MOMENTS[0])).astype(np.float32)
    data['adv_c'] = (data['adv_c'] + np.float32(MOMENTS[2])).astype(np.float32)
    scale = REGIMES[regime][0]
    if scale is None:
        adv_r = (data['adv_r'] - np.float32(MOMENTS[0])) / np.float32(MOMENTS[1])
        data['adv_r'] = (np.float32(MOMENTS[0]) + np.float32(MOMENTS[1] * 1e-2) * adv_r).astype(np.float32)
        data['adv_c'] = (np.float32(MOMENTS[2]) + np.float32(1e-2) * (data['adv_c'] - np.float32(MOMENTS[2]))).astype(np.float32)
        with oracle_nets(nets):
            v_r, v_c = oac.values(theta, data['obs'], O, A)
        data['target_value_r'] = (v_r + np.float32(0.1) * data['target_value_r']).astype(np.float32)
        data['target_value_c'] = (v_c + np.float32(0.1) * data['target_value_c']).astype(np.float32)
    else:
        data['target_value_r'] = data['target_value_r'] * np.float32(scale)
        data['target_value_c'] = data['target_value_c'] * np.float32(scale)
    perms = np.stack([rng.permutation(N * T) for _ in range(2)])
    return theta, data, perms


def _check_regime(rec, regime, mask):
    coefs = np.array([r['coef'] for r in rec['steps']])
    norms = np.array([r['norm'] for r in rec['steps']])
    max_norm = REGIMES[regime][1]
    on = [j for j in range(3) if (mask >> j) & 1]
    want = {'critics': [False, True, True], 'none': [False] * 3}.get(regime, [True] * 3)
    for j in on:
        assert ((coefs[:, j] < 1.0) == want[j]).all(), (regime, j, norms[:, j])
        assert (np.abs(np.log(norms[:, j] / max_norm)) > np.log(1.5)).all(), (regime, j, norms[:, j])
        if regime == 'small':    # 1e-6 / n is at least 3x the 1e-5 bar of the clipped-norm check on the first step
            assert norms[0, j] < 0.03, (j, norms[0, j])


def _engine_case(cuda, O, A, N, T, theta, data, nets=None):
    agent, buf, eng = _setup(cuda, data, N, T, O, A, theta, nets=nets)
    buf.adv_moments.copy_(torch.tensor(MOMENTS))
    eng.train_stats.zero_()
    return agent, buf, eng


def _run_passes(path, agent, buf, eng, perms_rows, *, mask, loss_kind, batch, max_norm, coef, lrs=LRS, ent=0.0):
    """update passes over perms_rows [iters][rows] (slab rows): 'x3_fused' = one osb_ppo_update_iter_x3 per pass,
    otherwise the minibatch gradient kernel of the precision + osb_optim_fused per minibatch."""
    lib, ptr, stream = _lib()
    O, A = eng.O, eng.A
    d = buf.data
    lag = torch.tensor([LAM, 0, 0, 0], dtype=torch.float32, device=agent.theta.device)
    a = agent
    for it in range(perms_rows.shape[0]):
        perm = perms_rows[it]
        total = perm.numel()
        if path == 'x3_fused':
            lib.osb_ppo_update_iter_x3(
                ptr(a.theta), ptr(a.grad), ptr(a.adam_m), ptr(a.adam_v), ptr(a.adam_step), O, A, ptr(d['obs']),
                ptr(d['act']), ptr(d['logp']), ptr(d['adv_r']), ptr(d['adv_c']), ptr(d['target_value_r']),
                ptr(d['target_value_c']), ptr(buf.adv_moments), ptr(perm), total, 0, batch, loss_kind, 0.2, ent,
                ptr(lag), mask, coef, max_norm, *lrs, ptr(eng.gpart), ptr(eng.stats_part), ptr(eng.train_stats),
                ptr(eng.stop_flag), 0, 0, 1, 0, 0, stream)
            continue
        fn = {'fp32': lib.osb_minibatch_grad, 'tf32': lib.osb_minibatch_grad_tc, 'bf16x3': lib.osb_minibatch_grad_x3}[path]
        for start in range(0, total, batch):
            count = min(batch, total - start)
            fn(ptr(a.theta), O, A, ptr(d['obs']), ptr(d['act']), ptr(d['logp']), ptr(d['adv_r']), ptr(d['adv_c']),
               ptr(d['target_value_r']), ptr(d['target_value_c']), ptr(eng.mu_old), ptr(buf.adv_moments), ptr(perm),
               total, 0, start, count, loss_kind, 0.2, ent, 1.0, 0.0, ptr(lag), ptr(eng.logstd_old), mask,
               ptr(eng.gpart), ptr(eng.stats_part), ptr(eng.stop_flag), stream)
            nb = lib.osb_update_grid_blocks(count) if path == 'fp32' else lib.osb_tc_grid_blocks(count, mask)
            lib.osb_optim_fused(ptr(eng.gpart), ptr(eng.stats_part), nb, O, A, ptr(a.theta), ptr(a.grad),
                                ptr(a.adam_m), ptr(a.adam_v), ptr(a.adam_step), coef, max_norm, *lrs, mask,
                                ptr(eng.sumsq_part), ptr(eng.train_stats), ptr(eng.stop_flag), stream)
    torch.cuda.synchronize()


# bars the suite already applies to the same arithmetic: per-step gradients 1e-4 l2 per block (fp32, bf16x3) / 5e-3
# (tf32, whole network); whole epochs |diff| < 5e-3 |update| (bf16x3, test_update_x3_gpu), bad.mean() < 1e-3 at rtol
# 2e-4 / atol 2e-6 (fp32, test_update_gpu), |diff| < 0.15 |update| (tf32, test_update_tc_gpu)
STEP_BAR = {'fp32': 1e-4, 'bf16x3': 1e-4, 'x3_fused': 1e-4, 'tf32': 5e-3}
EPOCH_BAR = {'fp32': 5e-3, 'bf16x3': 5e-3, 'x3_fused': 5e-3, 'tf32': 0.15}


def _compare_step(path, got, want_state, want_rec, O, A, mask, max_norm):
    """After one minibatch step: the clipped gradient, m and v per parameter block; the invariant (b)."""
    lay = oac.layout(O, A)
    bar = STEP_BAR[path]
    worst = 0.0
    for j, net in enumerate(o64.NETS):
        if not (mask >> j) & 1:
            continue
        sl = slice(lay[net]['start'], lay[net]['start'] + lay[net]['size'])
        _check_invariant(got['grad'], want_rec, j, sl, max_norm, bar)
        blocks = [(net, sl)] if path == 'tf32' else \
            [(f'{net}.{name}', slice(o, o + int(np.prod(shape)))) for name, (o, shape) in lay[net]['entries'].items()]
        for name, b in blocks:
            for key, g, w in (('grad', got['grad'][b], want_rec['grad'][b]), ('m', got['m'][b], want_state['m'][b]),
                              ('v', got['v'][b], want_state['v'][b])):
                e = _l2(g, w)
                worst = max(worst, e)
                assert e < bar, (path, 'one step', name, key, e)
    return worst


def _compare_epoch(path, got, want, theta0, O, A, mask):
    worst = {}
    for j, sl in enumerate(_slices(O, A)):
        if not (mask >> j) & 1:
            assert (got['theta'][sl] == theta0[sl]).all() and not got['m'][sl].any()
            continue
        upd = want['theta'][sl] - theta0[sl]
        for key, g, w in (('theta', got['theta'][sl] - theta0[sl], upd), ('m', got['m'][sl], want['m'][sl]),
                          ('v', got['v'][sl], want['v'][sl])):
            e = _l2(g, w)
            worst[key] = max(worst.get(key, 0.0), e)
            assert e < EPOCH_BAR[path], (path, 'epoch', o64.NETS[j], key, e)
        if path == 'fp32':
            bad = ~np.isclose(got['theta'][sl], want['theta'][sl], rtol=2e-4, atol=2e-6)
            assert bad.mean() < 1e-3, (o64.NETS[j], bad.sum())
    return worst


def _compare_stats(path, eng, rec, mask, ent=None):
    ts = eng.train_stats.cpu().numpy().reshape(3, 8)
    n = len(rec['steps'])
    rtol = 5e-3 if path == 'tf32' else 1e-3
    for j in range(3):
        if not (mask >> j) & 1:
            continue
        assert ts[j, 3] == n, (j, ts[j, 3], n)
        want = np.mean([r['loss'][j] for r in rec['steps']])
        np.testing.assert_allclose(ts[j, 0] / n, want, rtol=rtol, atol=1e-5, err_msg=f'logged loss of {o64.NETS[j]}')
    if ent is not None and mask & 1:    # the actor's entropy bonus at the sigma of every minibatch (ent: its coefficient)
        want = np.mean([-ent * r['entropy'] for r in rec['steps']])
        np.testing.assert_allclose(ts[0, 4] / n, want, rtol=rtol, atol=1e-7, err_msg='entropy bonus')


def _epoch_case(cuda, path, O, A, mask, loss_kind, regime, batch, seed, trained=False, nets=None):
    """One minibatch step, then two passes over 3.5 minibatches (short last one), each from the same initial state,
    on the device and in float64.  trained: a trained log_std, the actor at LRS_TRAINED and the entropy bonus on.
    nets: a network spec of test_update_gpu.NETS (tanh 64 wide if None)."""
    rows = batch * 7 // 2
    T = 64 if rows % 64 == 0 else 32
    N = rows // T
    theta, data, perms = _regime_data(O, A, N, T, regime, seed, trained, nets)
    _, max_norm, coef = REGIMES[regime]
    lrs, ent = (LRS_TRAINED, ENT_TRAINED) if trained else (LRS, 0.0)
    kw = dict(net_mask=mask, loss_kind=loss_kind, batch_size=batch, critic_norm_coef=coef, max_grad_norm=max_norm,
              lrs=lrs, clip=0.2, entropy_coef=ent)
    with oracle_nets(nets):
        one, rec1, _ = o64.ppo_epoch64(theta, data, MOMENTS, perms[:1, :batch], LAM, update_iters=1, **kw)
        want, rec, passes = o64.ppo_epoch64(theta, data, MOMENTS, perms, LAM, update_iters=2, **kw)
    assert passes == 2 and len(rec['steps']) == 8
    _check_regime(rec, regime, mask)
    rows_dev = torch.as_tensor(np.stack([_rows(p, N, T) for p in perms])).to(cuda)
    run = dict(mask=mask, loss_kind=loss_kind, batch=batch, max_norm=max_norm, coef=coef, lrs=lrs, ent=ent)
    agent, buf, eng = _engine_case(cuda, O, A, N, T, theta, data, nets)
    _run_passes(path, agent, buf, eng, rows_dev[:1, :batch].contiguous(), **run)
    got1 = _host(agent)
    assert (got1['step'] == [(mask >> j) & 1 for j in range(3)]).all(), got1['step']
    w1 = _compare_step(path, got1, one, rec1['steps'][0], O, A, mask, max_norm)
    agent, buf, eng = _engine_case(cuda, O, A, N, T, theta, data, nets)
    _run_passes(path, agent, buf, eng, rows_dev, **run)
    got = _host(agent)
    np.testing.assert_array_equal(got['step'], want['step'])
    assert (got['step'] == [8 * ((mask >> j) & 1) for j in range(3)]).all()
    for j, sl in enumerate(_slices(O, A)):      # invariant (b) on the last (short) minibatch step
        if (mask >> j) & 1:
            _check_invariant(got['grad'], rec['steps'][-1], j, sl, max_norm, STEP_BAR[path] * 10)
    we = _compare_epoch(path, got, want, theta, O, A, mask)
    _compare_stats(path, eng, rec, mask, ent if loss_kind == 0 else 0.0)
    return w1, we


def _spec_slices(mask, batch, O, A):
    """Parameters per CTA slice of every trained network in the persistent kernel: S = ceil(size / G) with G the
    kernel's grid width for this minibatch size."""
    lib, _, _ = _lib()
    G = lib.osb_tc_grid_blocks(batch, mask)
    lay = oac.layout(O, A)
    return G, [-(-lay[n]['size'] // G) for j, n in enumerate(o64.NETS) if (mask >> j) & 1]


X3_SHAPES = [(60, 8), (64, 8), (63, 16), (17, 6), (33, 1), (64, 16)]
X3_MASKS = [7, 3, 6, 2]
# Every net_mask runs speculatively on three shapes (regimes critics / all: the redo; none: no redo) and
# non-speculatively on the other three (all three regimes); the loss kind rotates independently.
X3_CASES = [(O, A, mask, ['spec', 'nonspec'][(si + mi) % 2], ['critics', 'all', 'none'][si // 2], [0, 1, 3][(si + mi // 2) % 3])
            for si, (O, A) in enumerate(X3_SHAPES) for mi, mask in enumerate(X3_MASKS)]
X3_CASES += [
    (60, 8, 2, 'full', 'all', 0),        # one network, gridDim.y == 1: as many CTAs as SMs (slice ~62 parameters)
    (64, 16, 3, 'full', 'all', 1),       # actor + reward critic at the grid cap of a multi-network launch
    (33, 1, 7, 'spec', 'small', 0),      # clipped norms < 0.03: a dropped + 1e-6 moves the clipped norm > 3e-5
    (64, 16, 6, 'nonspec', 'small', 1),
]
# at a trained log_std, the actor at lr 1e-2: sigma changes ~1 % per minibatch, so a sigma the kernel does not stage
# again after each Adam step drifts from ppo_epoch64's (every single-pass kind; A = 1 and A = 16; spec / nonspec / full)
X3_TRAINED = [(60, 8, 7, 'spec', 'none', 0), (17, 6, 3, 'nonspec', 'all', 1), (33, 1, 7, 'spec', 'all', 3),
              (64, 16, 3, 'full', 'none', 0)]
# test_update_gpu.NETS with every network clipping: A = 1 and A = 16 (the A > 8 kernel, whose template argument packs
# the activation), all three networks (ACT_MIXED unless the activations agree), the actor alone and the critics alone,
# speculative and non-speculative Adam
X3_NETS = [(33, 1, 7, 'spec', 'all', 0, False, 'tanh-relu'), (64, 16, 7, 'nonspec', 'all', 1, False, 'sp-id'),
           (60, 8, 7, 'spec', 'all', 1, False, 'sig-sp'),
           (64, 16, 1, 'spec', 'all', 3, False, 'sig-sp'), (60, 8, 6, 'nonspec', 'all', 0, False, 'sig-1'),
           (17, 6, 6, 'spec', 'all', 1, False, 'sp-id'), (64, 16, 7, 'spec', 'all', 0, True, 'tanh-relu'),
           (33, 1, 1, 'nonspec', 'all', 3, False, 'sig-1'), (64, 16, 6, 'nonspec', 'all', 0, False, 'tanh-relu')]


@pytest.mark.timeout(600)
@pytest.mark.parametrize('O,A,mask,mode,regime,loss_kind,trained,nets', net_cases(sigma_cases(X3_CASES, X3_TRAINED),
                                                                                  X3_NETS))
def test_persistent_x3_passes_vs_fp64(cuda, O, A, mask, mode, regime, loss_kind, trained, nets):
    """The persistent bf16x3 kernel (optimiser inside): speculative Adam (slice <= 512 parameters), its redo when a
    network clips, and the non-speculative slices; W1 / b1 (ones column when O < 64) / W3 (A up to 16) written into
    the weight-tile image and read back by the next three minibatches; log_std and its sigma staged again after every
    minibatch (trained)."""
    lib, _, _ = _lib()
    cap = lib.osb_tc_grid_blocks(1 << 40, mask)      # SMs (one network) or a third of them
    batch = {'spec': 4096, 'nonspec': 1024, 'full': 128 * (cap + 4)}[mode]
    G, S = _spec_slices(mask, batch, O, A)
    assert all((s <= NEPI) == (mode != 'nonspec') for s in S), (mode, G, S)
    assert mode != 'full' or G == cap, (G, cap)
    w1, we = _epoch_case(cuda, 'x3_fused', O, A, mask, loss_kind, regime, batch, seed=O + 10 * A + mask, trained=trained,
                         nets=nets)
    kind = f'{mode} redo' if mode != 'nonspec' and regime != 'none' else mode
    print(f'[x3_fused {kind} O={O} A={A} mask={mask} {regime} kind {loss_kind} G={G} S={S}{" " + nets if nets else ""}] '
          f'one step worst block '
          f'l2 {w1:.2e}; epoch ' + ', '.join(f'{k} {v:.2e}' for k, v in we.items()))


@pytest.mark.timeout(600)
@pytest.mark.parametrize('path,O,A,regime,trained,nets', net_cases(sigma_cases(
    [(path, O, A, regime) for path in ('fp32', 'tf32', 'bf16x3') for O, A in ((60, 8), (17, 6))
     for regime in ('critics', 'all', 'none')],
    # tf32 only with every network clipped: unclipped at lr 1e-2 its trajectory leaves float64's within the two passes
    # (last-step actor gradient norm 1.82 vs 1.53 on an H100)
    [('fp32', 60, 8, 'none'), ('bf16x3', 60, 8, 'none')] + [(path, 17, 6, 'all') for path in ('fp32', 'tf32', 'bf16x3')]),
    # test_update_gpu.NETS, every network clipping, A = 1 and A = 16.  tf32 at 17 x 6: at 60 x 8 the first minibatch
    # of sp-id and sig-sp has PPO-clip decisions that tf32 rounding flips (the one-step actor gradient measured 6e-2
    # l2-rel on an H100, 5e-4 with the ratio loss on the same data), a jump of whole samples no rounding bar covers
    [('fp32', 33, 1, 'all', False, 'sig-sp'), ('tf32', 17, 6, 'all', False, 'sp-id'),
     ('bf16x3', 64, 16, 'all', False, 'sig-1'), ('fp32', 64, 16, 'all', False, 'tanh-relu'),
     ('bf16x3', 33, 1, 'all', True, 'sp-id'), ('tf32', 17, 6, 'all', False, 'sig-1')]))
def test_stepwise_passes_vs_fp64(cuda, path, O, A, regime, trained, nets):
    """The minibatch gradient kernels + osb_optim_fused (launch per minibatch), PPO clip loss, every network."""
    w1, we = _epoch_case(cuda, path, O, A, 7, 0, regime, 1024, seed=O + A, trained=trained, nets=nets)
    print(f'[{path} O={O} A={A} {regime}{" " + nets if nets else ""}] one step worst block l2 {w1:.2e}; epoch ' +
          ', '.join(f'{k} {v:.2e}' for k, v in we.items()))


@pytest.mark.timeout(600)
@pytest.mark.parametrize('precision,fused', [(0, False), (1, False), (2, False), (2, True)])
def test_ppo_epoch_kl_stop_then_second_epoch(cuda, precision, fused):
    """UpdateEngine.ppo_epoch with clipping active (critics): a first epoch stopped by the KL after one of three
    passes (adam_step = 1 x n_mb), then a second epoch of two passes continuing the same Adam state
    (adam_step = 3 x n_mb), vs ppo_epoch64 with the state passed back in."""
    O, A, N, T, batch = 60, 8, 32, 112, 1024
    theta, data, _ = _regime_data(O, A, N, T, 'critics', 21)
    rng = np.random.default_rng(22)
    perms = np.stack([rng.permutation(N * T) for _ in range(5)])
    _, max_norm, coef = REGIMES['critics']
    lrs = (LRS[0], LRS[1], LRS[1])       # ppo_epoch takes one critic learning rate
    kw = dict(net_mask=7, loss_kind=0, batch_size=batch, critic_norm_coef=coef, max_grad_norm=max_norm, lrs=lrs,
              clip=0.2, entropy_coef=0.01)
    s1, r1, p1 = o64.ppo_epoch64(theta, data, MOMENTS, perms[:3], LAM, update_iters=3, target_kl=1e-12,
                                 kl_early_stop=True, **kw)
    s2, r2, p2 = o64.ppo_epoch64(None, data, MOMENTS, perms[3:], LAM, update_iters=2, kl_early_stop=False,
                                 state=s1, **kw)
    assert p1 == 1 and p2 == 2
    n_mb = -(-N * T // batch)
    path = {0: 'fp32', 1: 'tf32', 2: 'x3_fused' if fused else 'bf16x3'}[precision]
    lib, _, _ = _lib()
    saved = os.environ.pop('OSB_X3_NO_FUSE', None)
    if not fused:
        os.environ['OSB_X3_NO_FUSE'] = '1'
    try:
        agent, buf, eng = _engine_case(cuda, O, A, N, T, theta, data)
        lag = torch.tensor([LAM, 0, 0, 0], dtype=torch.float32, device=cuda)
        rows = torch.as_tensor(np.stack([_rows(p, N, T) for p in perms])).to(cuda)
        ekw = dict(loss_kind=0, lagrange=lag, net_mask=7, batch_size=batch, clip=0.2, entropy_coef=0.01,
                   critic_norm_coef=coef, max_grad_norm=max_norm, lr_actor=lrs[0], lr_critic=lrs[1],
                   precision=precision)
        launches = lib.osb_launch_count()
        eng.ppo_epoch(update_iters=3, target_kl=1e-12, kl_early_stop=True, perm=rows[:3].contiguous(), **ekw)
        torch.cuda.synchronize()
        launches = lib.osb_launch_count() - launches
        # the persistent kernel is one launch per pass (plus the KL evaluation); the stepwise path launches a gradient
        # kernel and an optimiser kernel for every minibatch of every pass (no-ops after the stop)
        assert launches < 2 * 3 * n_mb if fused else launches >= 2 * 3 * n_mb, (path, launches)
        got1 = _host(agent)
        kls = eng.kl_state.cpu().numpy()
        assert int(kls[1]) == 1 and kls[2] == 1.0, kls
        assert (got1['step'] == n_mb).all(), got1['step']
        _compare_stats(path, eng, r1, 7, 0.01)
        w1 = _compare_epoch(path, got1, s1, theta, O, A, 7)
        eng.ppo_epoch(update_iters=2, target_kl=0.0, kl_early_stop=False, perm=rows[3:].contiguous(), **ekw)
        torch.cuda.synchronize()
    finally:
        os.environ.pop('OSB_X3_NO_FUSE', None)
        if saved is not None:
            os.environ['OSB_X3_NO_FUSE'] = saved
    got2 = _host(agent)
    assert (got2['step'] == 3 * n_mb).all(), got2['step']
    _compare_stats(path, eng, r2, 7, 0.01)
    w2 = _compare_epoch(path, got2, s2, theta, O, A, 7)
    print(f'[{path}] epoch 1 (KL stop) ' + ', '.join(f'{k} {v:.2e}' for k, v in w1.items()) +
          '; epoch 2 ' + ', '.join(f'{k} {v:.2e}' for k, v in w2.items()))
