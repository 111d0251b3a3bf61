"""GPU: the natural-gradient pieces of CPO / PCPO / TRPO / TRPOLag / RCPO / OnCRPO / NaturalPG / TRPOPID -- the
Fisher-vector product, the conjugate-gradient solve, the full-batch surrogate gradient, the old-policy means and the
line-search evaluation -- through UpdateEngine exactly as the algorithms call them, in every precision, against the
float64 reference (oracle/fisher64.py, itself pinned to the unmodified reference in test_natural_gradient_ref_cpu).

The advantages are raw and the buffer's moments non-trivial ({mean_r, std_r + 1e-8, mean_c, 1} = MOMENTS), so the
on-load standardisation of every update and evaluation kernel is checked against (adv_r - mean_r) / std_r and
adv_c - mean_c; the PPO-side minibatch kernels and a whole bf16x3 PPO-Lag epoch are checked the same way.

Shapes reach the ragged last tile, the scalar row gather (obs dim % 4 != 0), A = 1, the A > 8 instantiation of the
bf16x3 FVP backward, more 128-row tiles than CTAs in the FVP / gradient kernels (> 132 on an H100 SXM) and in the
evaluation kernels (> 264), and obs dims > 64 (K-chunked layer 1 on tf32 tiles; the bf16x3 mode falls
back to the fp32 tiles there and is held to the fp32 bars).  Each case prints its worst error."""
import functools
import time

import numpy as np
import pytest
import torch

from oracle import actor_critic as oac
from oracle import fisher64 as f64
from oracle import learner as ol
from test_update_gpu import _rand_data, _rows, _setup
from test_update_x3_gpu import _oracle_grad

pytestmark = pytest.mark.gpu

MOMENTS = [0.37, 2.3, -0.41, 1.0]
LAM = 0.37
DAMPING = 0.1
LOSS_RATIO, LOSS_COST = 1, 3

SHAPES = [
    (12, 3, 8, 24),        # the golden shape of test_update_gpu::test_fvp_cg_eval_golden
    (17, 6, 9, 31),        # O % 4 != 0: scalar row gather; ragged last tile
    (33, 1, 50, 11),       # A = 1
    (45, 9, 300, 70),      # A = 9: A > 8 template of the bf16x3 FVP backward; 165 tiles > 132 CTAs
    (64, 16, 100, 50),     # largest bf16x3 dims
    (60, 8, 512, 80),      # 320 tiles: several tiles per CTA in FVP / gradient / evaluation
    (111, 8, 40, 30),      # obs dims > 64: K-chunked layer 1 (tf32); bf16x3 takes the fp32 tiles
    (376, 8, 64, 40),
]
PRECISIONS = [0, 1, 2]     # engine.precision: fp32 FMA tiles, tf32 wgmma tiles, split-bf16 wgmma tiles

# fp32 and bf16x3: the bars test_update_gpu / test_update_x3_gpu apply to the same arithmetic; tf32: the bars of
# test_update_tc_gpu
_EXACT = dict(l2=1e-4, rtol=2e-4, atol=2e-5, mu=2e-6, s_rtol=1e-4, s_atol=1e-6, kl_rtol=1e-3, kl_atol=1e-8, one=1e-5)
BARS = {'fp32': _EXACT, 'bf16x3': _EXACT,
        'tf32': dict(l2=5e-3, rtol=None, atol=None, mu=3e-3, s_rtol=2e-2, s_atol=2e-3, kl_rtol=2e-2, kl_atol=2e-3,
                     one=2e-3)}


def _raw(data):
    """Standard-normal advantages -> raw advantages whose moments are MOMENTS (approximately)."""
    out = dict(data)
    out['adv_r'] = (data['adv_r'] * np.float32(MOMENTS[1]) + np.float32(MOMENTS[0])).astype(np.float32)
    out['adv_c'] = (data['adv_c'] + np.float32(MOMENTS[2])).astype(np.float32)
    return out


def _standardised(data):
    out = dict(data)
    out['adv_r'] = ((data['adv_r'].astype(np.float64) - MOMENTS[0]) / MOMENTS[1]).astype(np.float32)
    out['adv_c'] = (data['adv_c'].astype(np.float64) - MOMENTS[2]).astype(np.float32)
    return out


@functools.lru_cache(maxsize=None)
def _case(O, A, N, T):
    """Env-major batch with raw advantages, the actor block of theta and a direction vector (float32)."""
    rng = np.random.default_rng(1000 + 7 * O + N)
    theta = oac.init_theta(O, A, seed=O + A)
    data = _raw(_rand_data(rng, N, T, O, A, theta))
    Pa = oac.layout(O, A)['actor']['size']
    return theta, theta[:Pa].copy(), data, rng.standard_normal(Pa).astype(np.float32)


@functools.lru_cache(maxsize=None)
def _ref_fvp(O, A, N, T):
    _, th, data, vec = _case(O, A, N, T)
    return f64.fvp64(th, vec, data['obs'], DAMPING)


@functools.lru_cache(maxsize=None)
def _ref_grad(O, A, N, T, kind):
    _, th, data, _ = _case(O, A, N, T)
    return f64.surrogate_grad64(th, data, MOMENTS, LAM, kind)


def _engine(cuda, O, A, N, T, precision):
    theta, _, data, _ = _case(O, A, N, T)
    agent, buf, eng = _setup(cuda, data, N, T, O, A, theta)
    buf.adv_moments.copy_(torch.tensor(MOMENTS))
    eng.precision = precision
    path = 'bf16x3' if eng._x3() else 'tf32' if eng._tc() else 'fp32'
    if precision == 2 and O > 64:
        assert path == 'fp32'       # split-bf16 tiles cover obs dims <= 64; beyond, the fp32 tiles
    return agent, buf, eng, path


def _slab(buf, key):
    x = buf.data[key].cpu().numpy()
    return x.reshape(x.shape[0] * x.shape[1], *x.shape[2:])


def _check_blocks(what, got, want, O, A, bar, per_block=True):
    """Per parameter block of the actor: l2-relative error, and for the fp32-level paths elementwise
    rtol / atol relative to the block's largest entry.  Returns the worst l2-relative error."""
    got = np.asarray(got, np.float64)
    worst = 0.0
    for name, (off, shape) in oac.layout(O, A)['actor']['entries'].items():
        n = int(np.prod(shape))
        g, w = got[off:off + n], want[off:off + n]
        rel = float(np.linalg.norm(g - w) / (np.linalg.norm(w) + 1e-300))
        worst = max(worst, rel)
        print(f'  {what} {name}: l2-rel {rel:.2e}  max-err/scale {np.abs(g - w).max() / np.abs(w).max():.2e}')
        if per_block:
            assert rel < bar['l2'], (what, name, rel)
        if bar['rtol'] is not None:
            np.testing.assert_allclose(g, w, rtol=bar['rtol'], atol=bar['atol'] * np.abs(w).max(), err_msg=f'{what} {name}')
    total = float(np.linalg.norm(got - want) / np.linalg.norm(want))
    print(f'{what}: worst block l2-rel {worst:.2e}, whole-vector l2-rel {total:.2e}')
    assert total < bar['l2'], (what, total)
    return worst


@pytest.mark.timeout(300)
@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('O,A,N,T', SHAPES)
def test_fvp_vs_fp64(cuda, O, A, N, T, precision):
    """UpdateEngine.fvp (F v + damping v) vs the double-backward Hessian of the mean KL."""
    agent, buf, eng, path = _engine(cuda, O, A, N, T, precision)
    vec = torch.as_tensor(_case(O, A, N, T)[3]).to(cuda)
    out = torch.zeros_like(vec)
    eng.fvp(vec, out, DAMPING)
    torch.cuda.synchronize()
    print(f'[{path}]')
    _check_blocks('fvp', out.cpu().numpy(), _ref_fvp(O, A, N, T), O, A, BARS[path])


@pytest.mark.timeout(300)
@pytest.mark.parametrize('precision', PRECISIONS)
def test_fvp_strided_vs_fp64(cuda, precision):
    """fvp_sample_freq = 3: the FVP over slab rows 0, 3, 6, ..."""
    O, A, N, T = 64, 16, 100, 50
    agent, buf, eng, path = _engine(cuda, O, A, N, T, precision)
    _, th, _, vec = _case(O, A, N, T)
    out = torch.zeros(eng.Pa, device=cuda)
    eng.fvp(torch.as_tensor(vec).to(cuda), out, DAMPING, stride=3)
    torch.cuda.synchronize()
    want = f64.fvp64(th, vec, _slab(buf, 'obs')[::3], DAMPING)
    print(f'[{path}]')
    _check_blocks('fvp stride 3', out.cpu().numpy(), want, O, A, BARS[path])


@pytest.mark.timeout(300)
@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('O,A,N,T', SHAPES)
def test_actor_loss_grad_vs_fp64(cuda, O, A, N, T, precision):
    """UpdateEngine.actor_loss_grad: the full-batch ratio surrogate (Lagrangian mix) and cost surrogate, both signs,
    gradient and loss value, vs float64 autograd on the standardised advantages."""
    agent, buf, eng, path = _engine(cuda, O, A, N, T, precision)
    bar = BARS[path]
    lag = torch.tensor([LAM], dtype=torch.float32, device=cuda)
    eng.snapshot_old_policy()
    print(f'[{path}]')
    for kind, name in ((LOSS_RATIO, 'ratio'), (LOSS_COST, 'cost')):
        want, want_loss = _ref_grad(O, A, N, T, name)
        for sign in (-1.0, 1.0):
            g = torch.zeros(eng.Pa, device=cuda)
            loss = float(eng.actor_loss_grad(kind, lag, g, sign))
            _check_blocks(f'grad {name} sign {sign:+.0f}', g.cpu().numpy(), sign * want, O, A, bar,
                          per_block=path != 'tf32')
            print(f'  loss {name}: {loss:.7f} vs {want_loss:.7f}  rel {abs(loss - want_loss) / abs(want_loss):.2e}')
            np.testing.assert_allclose(loss, want_loss, rtol=bar['s_rtol'], atol=bar['s_atol'], err_msg=name)


@pytest.mark.timeout(300)
@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('O,A,N,T', SHAPES)
def test_old_policy_and_evaluate_vs_fp64(cuda, O, A, N, T, precision):
    """snapshot_old_policy vs the float64 mean; evaluate of the unchanged actor (KL 0) and of theta + 0.02 v (KL,
    surrogates, mean ratio); at the policy's own log-probs the unchanged actor has ratio 1."""
    agent, buf, eng, path = _engine(cuda, O, A, N, T, precision)
    bar = BARS[path]
    _, th, data, vec = _case(O, A, N, T)
    lag = torch.tensor([LAM], dtype=torch.float32, device=cuda)
    eng.snapshot_old_policy()
    obs, act = _slab(buf, 'obs'), _slab(buf, 'act')
    mu = eng.mu_old.cpu().numpy().reshape(-1, A)
    want_mu = f64.mean64(th, obs)
    print(f'[{path}] mu_old max-err {np.abs(mu - want_mu).max():.2e}')
    np.testing.assert_allclose(mu, want_mu, rtol=0, atol=bar['mu'])
    np.testing.assert_array_equal(eng.logstd_old.cpu().numpy(), th[:A])
    ev0 = eng.evaluate(agent.theta, lag)
    assert abs(ev0['kl']) < 1e-9, ev0['kl']
    th2 = (th + np.float32(0.02) * vec).astype(np.float32)
    theta2 = agent.theta.clone()
    theta2[: eng.Pa] = torch.as_tensor(th2).to(cuda)
    got = eng.evaluate(theta2, lag)
    want = f64.eval64(th2, th, data, MOMENTS, LAM)
    for k in ('kl', 'loss', 'loss_r', 'loss_c', 'ratio'):
        print(f'  {k}: {got[k]:.8g} vs {want[k]:.8g}  rel {abs(got[k] - want[k]) / abs(want[k]):.2e}')
        rtol, atol = (bar['kl_rtol'], bar['kl_atol']) if k == 'kl' else (bar['s_rtol'], bar['s_atol'])
        np.testing.assert_allclose(got[k], want[k], rtol=rtol, atol=atol, err_msg=k)
    buf.data['logp'].copy_(torch.as_tensor(f64.logp64(th, obs, act).astype(np.float32)).view_as(buf.data['logp']))
    ev1 = eng.evaluate(agent.theta, lag)
    print(f'  own log-probs: kl {ev1["kl"]:.1e}  ratio - 1 {ev1["ratio"] - 1:.1e}')
    assert abs(ev1['kl']) < 1e-9 and abs(ev1['ratio'] - 1.0) < bar['one'], ev1


def _fvp_ref(th, obs):
    return lambda v: f64.fvp64(th, v, obs, DAMPING)


@pytest.mark.timeout(300)
@pytest.mark.parametrize('precision', [0, 2])
@pytest.mark.parametrize('O,A,N,T', [(12, 3, 8, 24), (60, 8, 512, 80)])
def test_conjugate_gradients_vs_fp64(cuda, O, A, N, T, precision):
    """conjugate_gradients(b, 15, damping 0.1) on b = -grad of the reward surrogate vs the float64 CG on fvp64."""
    agent, buf, eng, path = _engine(cuda, O, A, N, T, precision)
    _, th, data, _ = _case(O, A, N, T)
    b = (-_ref_grad(O, A, N, T, 'ratio')[0]).astype(np.float32)
    x = eng.conjugate_gradients(torch.as_tensor(b).to(cuda), 15, DAMPING)
    torch.cuda.synchronize()
    want, steps, _ = f64.cg64(_fvp_ref(th, data['obs']), b, 15)
    got = x.cpu().numpy()
    print(f'[{path}] cg: l2-rel {np.linalg.norm(got - want) / np.linalg.norm(want):.2e}  '
          f'max-err {np.abs(got - want).max():.2e}  |x|_max {np.abs(want).max():.2e}  steps {steps}')
    np.testing.assert_allclose(got, want, rtol=5e-3, atol=2e-5)
    assert int(eng.cg_scalars[2]) == steps


@pytest.mark.timeout(300)
@pytest.mark.parametrize('precision', PRECISIONS)
def test_conjugate_gradients_edges(cuda, precision):
    """b = 0: x = 0 after one step with the done flag set.  A residual tolerance between two well-separated residual
    norms of the float64 solve stops the device solve after the same number of steps."""
    O, A, N, T = 12, 3, 8, 24
    agent, buf, eng, path = _engine(cuda, O, A, N, T, precision)
    x = eng.conjugate_gradients(torch.zeros(eng.Pa, device=cuda), 15, DAMPING)
    sc = eng.cg_scalars.cpu().numpy()
    assert torch.isfinite(x).all() and not x.any() and np.isfinite(sc).all()
    assert sc[1] == 1.0 and sc[2] == 1.0, sc
    _, th, data, _ = _case(O, A, N, T)
    b = (-_ref_grad(O, A, N, T, 'ratio')[0]).astype(np.float32)
    _, _, norms = f64.cg64(_fvp_ref(th, data['obs']), b, 15, residual_tol=0.0)
    # first step k >= 2 whose residual is below half of every earlier one: tol = geometric mean of the two
    k = next(k for k in range(1, len(norms)) if norms[k] < 0.5 * min(norms[:k]))
    tol = float(np.sqrt(norms[k] * min(norms[:k])))
    want, steps, _ = f64.cg64(_fvp_ref(th, data['obs']), b, 15, residual_tol=tol)
    assert steps == k + 1 < 15
    x = eng.conjugate_gradients(torch.as_tensor(b).to(cuda), 15, DAMPING, residual_tol=tol)
    sc = eng.cg_scalars.cpu().numpy()
    print(f'[{path}] early stop: tol {tol:.3e} steps {steps}, device {sc[2]:.0f} (done {sc[1]:.0f})')
    assert sc[1] == 1.0 and int(sc[2]) == steps
    rel = float(np.linalg.norm(x.cpu().numpy() - want) / np.linalg.norm(want))
    assert rel < (5e-2 if path == 'tf32' else 5e-3), rel


@pytest.mark.timeout(300)
def test_headline_size_bf16x3_vs_fp64(cuda):
    """The bench.py --algo CPO batch (4096 envs x 128 steps = 524 288 rows, obs 60 / act 8) on split-bf16 tiles:
    FVP, both surrogate gradients and the line-search evaluation against the chunked float64 reference."""
    from omnisafe_b200.algorithms.engine import UpdateEngine
    from omnisafe_b200.common.buffer import VectorOnPolicyBuffer
    from omnisafe_b200.models import ConstraintActorCritic
    from test_update_gpu import _model_cfgs

    N, T, O, A = 4096, 128, 60, 8
    g = torch.Generator(device=cuda).manual_seed(11)
    agent = ConstraintActorCritic(O, A, _model_cfgs(3e-4, 3e-4), epochs=1, device=cuda)
    theta = oac.init_theta(O, A, seed=1)
    agent.load_flat(theta)
    buf = VectorOnPolicyBuffer(O, A, T, 0.99, 0.95, 0.95, 'gae', 0.0, True, True, num_envs=N, device=cuda)
    r = lambda *s: torch.randn(*s, generator=g, device=cuda)   # noqa: E731
    d = buf.data
    d['obs'].copy_(r(T, N, O)); d['act'].copy_(r(T, N, A) * 0.5)
    d['adv_r'].copy_(MOMENTS[0] + MOMENTS[1] * r(T, N)); d['adv_c'].copy_(MOMENTS[2] + r(T, N))
    d['target_value_r'].copy_(r(T, N)); d['target_value_c'].copy_(r(T, N))
    noise = 0.05 * r(T, N)
    buf.adv_moments.copy_(torch.tensor(MOMENTS))
    eng = UpdateEngine(agent, buf)
    eng.precision = 2
    assert eng._x3()
    Pa = eng.Pa
    th = theta[:Pa].copy()
    t0 = time.perf_counter()
    data = {k: _slab(buf, k) for k in ('obs', 'act', 'adv_r', 'adv_c')}
    data['logp'] = (f64.logp64(th, data['obs'], data['act']) + noise.reshape(-1).double().cpu().numpy()).astype(np.float32)
    d['logp'].copy_(torch.as_tensor(data['logp']).view(T, N))
    vec = np.random.default_rng(5).standard_normal(Pa).astype(np.float32)
    want_fvp = f64.fvp64(th, vec, data['obs'], DAMPING)
    want_r, loss_r = f64.surrogate_grad64(th, data, MOMENTS, LAM, 'ratio')
    want_c, loss_c = f64.surrogate_grad64(th, data, MOMENTS, LAM, 'cost')
    th2 = (th + np.float32(0.02) * vec).astype(np.float32)
    want_ev = f64.eval64(th2, th, data, MOMENTS, LAM)
    want_mu = f64.mean64(th, data['obs'])
    print(f'float64 reference at {N * T} rows: {time.perf_counter() - t0:.1f} s')
    bar = BARS['bf16x3']
    out = torch.zeros(Pa, device=cuda)
    eng.fvp(torch.as_tensor(vec).to(cuda), out, DAMPING)
    torch.cuda.synchronize()
    _check_blocks('fvp', out.cpu().numpy(), want_fvp, O, A, bar)
    lag = torch.tensor([LAM], dtype=torch.float32, device=cuda)
    eng.snapshot_old_policy()
    mu = eng.mu_old.cpu().numpy().reshape(-1, A)
    print(f'mu_old max-err {np.abs(mu - want_mu).max():.2e}')
    np.testing.assert_allclose(mu, want_mu, rtol=0, atol=bar['mu'])
    for kind, sign, want, want_loss, name in ((LOSS_RATIO, -1.0, want_r, loss_r, 'ratio'),
                                              (LOSS_COST, 1.0, want_c, loss_c, 'cost')):
        gv = torch.zeros(Pa, device=cuda)
        loss = float(eng.actor_loss_grad(kind, lag, gv, sign))
        _check_blocks(f'grad {name}', gv.cpu().numpy(), sign * want, O, A, bar)
        print(f'  loss {name}: {loss:.7f} vs {want_loss:.7f}')
        np.testing.assert_allclose(loss, want_loss, rtol=bar['s_rtol'], atol=bar['s_atol'], err_msg=name)
    theta2 = agent.theta.clone()
    theta2[:Pa] = torch.as_tensor(th2).to(cuda)
    got = eng.evaluate(theta2, lag)
    for k in ('kl', 'loss', 'loss_r', 'loss_c', 'ratio'):
        print(f'  {k}: {got[k]:.8g} vs {want_ev[k]:.8g}  rel {abs(got[k] - want_ev[k]) / abs(want_ev[k]):.2e}')
        rtol, atol = (bar['kl_rtol'], bar['kl_atol']) if k == 'kl' else (bar['s_rtol'], bar['s_atol'])
        np.testing.assert_allclose(got[k], want_ev[k], rtol=rtol, atol=atol, err_msg=k)


# ---- advantage moments in the PPO-side kernels ---------------------------------------------------------------------

@pytest.mark.timeout(300)
@pytest.mark.parametrize('loss_kind', [0, 1, 3])
@pytest.mark.parametrize('fn', ['osb_minibatch_grad', 'osb_minibatch_grad_tc', 'osb_minibatch_grad_x3'])
def test_minibatch_grad_moments_vs_autograd(cuda, fn, loss_kind):
    """The minibatch gradient kernels standardise raw advantages with the buffer's moments: vs oracle autograd on
    the standardised advantages, at the bars of test_update_gpu (fp32), test_update_tc_gpu and test_update_x3_gpu."""
    from omnisafe_b200._lib import current_stream, lib, ptr

    O, A, N, T = 60, 8, 64, 40
    rng = np.random.default_rng(77 + loss_kind)
    theta = oac.init_theta(O, A, seed=5)
    data = _raw(_rand_data(rng, N, T, O, A, theta))
    agent, buf, eng = _setup(cuda, data, N, T, O, A, theta)
    buf.adv_moments.copy_(torch.tensor(MOMENTS))
    B = N * T
    lag = torch.tensor([LAM], dtype=torch.float32, device=cuda)
    perm_em = rng.permutation(B)
    start, count = 3, B - 10
    perm = torch.as_tensor(_rows(perm_em, N, T)).to(cuda)
    coef = 1e-3
    d = buf.data
    getattr(lib(), fn)(ptr(agent.theta), O, A, ptr(d['obs']), ptr(d['act']), ptr(d['logp']), ptr(d['adv_r']),
                       ptr(d['adv_c']), ptr(d['target_value_r']), ptr(d['target_value_c']), ptr(eng.mu_old),
                       ptr(buf.adv_moments), ptr(perm), B, 0, start, count, loss_kind, 0.2, 0.01, 1.0, 0.0, ptr(lag),
                       ptr(eng.logstd_old), 7, ptr(eng.gpart), ptr(eng.stats_part), 0, current_stream())
    nb = lib().osb_update_grid_blocks(count) if fn == 'osb_minibatch_grad' else lib().osb_tc_grid_blocks(count, 7)
    lib().osb_grad_reduce(ptr(eng.gpart), ptr(eng.stats_part), nb, O, A, ptr(agent.theta), ptr(agent.grad), coef, 7,
                          ptr(eng.sumsq_part), ptr(agent.adam_step), ptr(eng.train_stats), 0, current_stream())
    torch.cuda.synchronize()
    got = agent.grad.cpu().numpy()
    ts = eng.train_stats.cpu().numpy().reshape(3, 8)
    want, loss = _oracle_grad(theta, O, A, _standardised(data), torch.as_tensor(perm_em[start:start + count]), LAM,
                              loss_kind, coef)
    lay = oac.layout(O, A)
    tc = fn.endswith('_tc')
    worst = 0.0
    for net in ol.NETS:
        s, n = lay[net]['start'], lay[net]['size']
        for name, (off, shape) in lay[net]['entries'].items():
            m = int(np.prod(shape))
            w, g = want[off:off + m], got[off:off + m]
            rel = float(np.linalg.norm(g - w) / (np.linalg.norm(w) + 1e-30))
            worst = max(worst, rel)
            if tc:
                cos = float((g * w).sum() / (np.linalg.norm(g) * np.linalg.norm(w) + 1e-30))
                tol = 2e-2 if (net == 'actor' and loss_kind == 0) else 5e-3   # PPO clip flips near the boundary
                assert rel < tol and cos > 0.9999, (net, name, rel, cos)
            elif fn.endswith('_x3'):
                assert rel < 1e-4, (net, name, rel)
        if not tc:
            scale = np.abs(want[s:s + n]).max()
            np.testing.assert_allclose(got[s:s + n], want[s:s + n], rtol=2e-4, atol=2e-5 * max(scale, 1e-3), err_msg=net)
    print(f'{fn} kind {loss_kind}: worst block l2-rel {worst:.2e}, loss {ts[0, 0]:.6f}')
    ent = 0.01 * (0.5 + 0.5 * np.log(2 * np.pi)) if loss_kind == 0 else 0.0
    np.testing.assert_allclose(ts[0, 0], loss + ent, rtol=5e-3 if tc else 1e-3, atol=1e-4)


@pytest.mark.timeout(300)
def test_ppolag_epoch_x3_moments_vs_oracle(cuda):
    """One whole PPO-Lag update epoch on the persistent bf16x3 kernel (64 x 32 rows, batch 512, 3 passes) on raw
    advantages with non-trivial moments vs Learner.update_ppo on the standardised advantages."""
    rng = np.random.default_rng(31)
    N, T, O, A = 64, 32, 60, 8
    theta = oac.init_theta(O, A, seed=2)
    data = _raw(_rand_data(rng, N, T, O, A, theta))
    B = N * T
    perms_em = np.stack([rng.permutation(B) for _ in range(3)])
    L = ol.Learner(theta, O, A)
    L.update_ppo(_standardised(data), perms_em, LAM, batch_size=512, clip=0.2, critic_norm_coef=0.001,
                 max_grad_norm=40.0, kl_early_stop=False)
    agent, buf, eng = _setup(cuda, data, N, T, O, A, theta)
    buf.adv_moments.copy_(torch.tensor(MOMENTS))
    lag = torch.tensor([LAM, 0, 0, 0], dtype=torch.float32, device=cuda)
    perms = torch.as_tensor(np.stack([_rows(p_, N, T) for p_ in perms_em])).to(cuda)
    eng.ppo_epoch(loss_kind=0, lagrange=lag, net_mask=7, batch_size=512, update_iters=3, clip=0.2,
                  critic_norm_coef=0.001, max_grad_norm=40.0, lr_actor=3e-4, lr_critic=3e-4, target_kl=10.0,
                  kl_early_stop=False, perm=perms, precision=2)
    torch.cuda.synchronize()
    got, want = agent.theta.cpu().numpy(), L.flat()
    bad = ~np.isclose(got, want, rtol=5e-4, atol=5e-6)
    print(f'epoch: {bad.sum()} elements off, max |diff| {np.abs(got - want).max():.2e}, '
          f'|diff| / |step| {np.linalg.norm(got - want) / np.linalg.norm(want - theta):.2e}')
    assert bad.mean() < 1e-3 and np.abs(got - want).max() < 2e-2, (bad.sum(), np.abs(got - want).max())
