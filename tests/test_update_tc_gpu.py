"""GPU: the wgmma (TF32) variant of the fused minibatch kernel vs autograd and vs the exact-fp32
path.  Tolerance: TF32 keeps 10 mantissa bits, so gradients agree to ~1e-2 of their scale (stated
here; the fp32 FMA path is the 1e-5 parity path)."""
import numpy as np
import pytest
import torch

from oracle import actor_critic as oac
from oracle import learner as ol
from test_update_gpu import _rand_data, _rows, _setup

pytestmark = pytest.mark.gpu


@pytest.mark.timeout(120)
@pytest.mark.parametrize('O,A,N,T,loss_kind', [(60, 8, 20, 13, 0), (60, 8, 64, 40, 0), (17, 6, 9, 31, 3), (64, 16, 16, 24, 1), (60, 8, 512, 80, 0),
                                                (111, 8, 40, 30, 1), (376, 8, 33, 12, 3), (128, 4, 300, 9, 1), (65, 8, 20, 7, 0)])   # obs dims > 64: K-chunked layer 1
def test_tc_grad_vs_autograd(cuda, O, A, N, T, loss_kind):
    from omnisafe_b200._lib import current_stream, lib, ptr

    rng = np.random.default_rng(O + N)
    theta = oac.init_theta(O, A, seed=5)
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
    lib().osb_minibatch_grad_tc(ptr(agent.theta), O, A, ptr(d['obs']), ptr(d['act']), ptr(d['logp']),
                                ptr(d['adv_r']), ptr(d['adv_c']), ptr(d['target_value_r']), ptr(d['target_value_c']),
                                ptr(eng.mu_old), ptr(buf.adv_moments), ptr(perm), B, 0, start, count, loss_kind, 0.2, 0.01,
                                1.0, 0.0, ptr(lag), ptr(eng.logstd_old), 7, ptr(eng.gpart), ptr(eng.stats_part), 0, current_stream())
    nb = lib().osb_tc_grid_blocks(count, 7)
    lib().osb_grad_reduce(ptr(eng.gpart), ptr(eng.stats_part), nb, O, A, ptr(agent.theta), ptr(agent.grad),
                          coef, 7, ptr(eng.sumsq_part), ptr(agent.adam_step), ptr(eng.train_stats), 0,
                          current_stream())
    torch.cuda.synchronize()
    got = agent.grad.cpu().numpy()
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
    bad = 0
    for net in ol.NETS:
        for name, (off, shape) in lay[net]['entries'].items():
            n = int(np.prod(shape))
            w, g = want[off:off + n], got[off:off + n]
            scale = max(np.abs(w).max(), 1e-6)
            err = np.abs(g - w).max() / scale
            cos = float((g * w).sum() / (np.linalg.norm(g) * np.linalg.norm(w) + 1e-30))
            rel = float(np.linalg.norm(g - w) / (np.linalg.norm(w) + 1e-30))
            print(f'{net}.{name}: max-err/scale {err:.2e}  l2-rel {rel:.2e}  cos {cos:.6f}')
            tol = 2e-2 if (net == 'actor' and loss_kind == 0) else 5e-3   # PPO clip flips near the boundary
            bad += (rel > tol) or (cos < 0.9999)
    assert bad == 0


@pytest.mark.timeout(120)
def test_tc_epoch_close_to_fp32_epoch(cuda):
    """A whole PPO-Lag update epoch in TF32 mode lands next to the exact-fp32 epoch."""
    rng = np.random.default_rng(3)
    N, T, O, A = 64, 32, 60, 8
    theta = oac.init_theta(O, A, seed=2)
    data = _rand_data(rng, N, T, O, A, theta)
    B = N * T
    perms = torch.as_tensor(np.stack([_rows(rng.permutation(B), N, T) for _ in range(3)])).to(cuda)
    out = []
    for prec in (0, 1):
        agent, buf, eng = _setup(cuda, data, N, T, O, A, theta)
        lag = torch.tensor([0.2, 0, 0, 0], dtype=torch.float32, device=cuda)
        eng.ppo_epoch(loss_kind=0, lagrange=lag, net_mask=7, batch_size=512, update_iters=3, clip=0.2,
                      critic_norm_coef=0.001, max_grad_norm=40.0, lr_actor=3e-4, lr_critic=3e-4,
                      target_kl=10.0, kl_early_stop=False, perm=perms, precision=prec)
        torch.cuda.synchronize()
        out.append(agent.theta.cpu().numpy())
    delta = out[0] - theta
    diff = out[1] - out[0]
    assert np.isfinite(out[1]).all()
    assert np.linalg.norm(diff) < 0.15 * np.linalg.norm(delta), (np.linalg.norm(diff), np.linalg.norm(delta))


@pytest.mark.timeout(120)
@pytest.mark.parametrize('O', [60, 111, 376])
def test_tc_actor_eval_matches_fp32_eval(cuda, O):
    rng = np.random.default_rng(9)
    N, T, A = 96, 50, 8
    theta = oac.init_theta(O, A, seed=4)
    data = _rand_data(rng, N, T, O, A, theta)
    agent, buf, eng = _setup(cuda, data, N, T, O, A, theta)
    eng.precision = 0
    eng.snapshot_old_policy()
    mu0 = eng.mu_old.clone()
    th2 = agent.theta.clone()
    th2[: eng.Pa] += 0.02 * torch.randn(eng.Pa, device=cuda)
    lag = torch.tensor([0.3], dtype=torch.float32, device=cuda)
    ref = eng.evaluate(th2, lag)
    eng.precision = 1
    eng.snapshot_old_policy()
    torch.cuda.synchronize()
    np.testing.assert_allclose(eng.mu_old.cpu().numpy(), mu0.cpu().numpy(), rtol=0, atol=3e-3)
    eng.mu_old.copy_(mu0)
    got = eng.evaluate(th2, lag)
    for k in ('kl', 'loss', 'loss_c', 'loss_r', 'ratio'):
        np.testing.assert_allclose(got[k], ref[k], rtol=2e-2, atol=2e-3, err_msg=k)


@pytest.mark.timeout(120)
@pytest.mark.parametrize('O,A,N,T,stride', [(60, 8, 64, 40, 1), (17, 6, 9, 31, 1), (64, 16, 100, 50, 3), (60, 8, 512, 80, 1),
                                             (111, 8, 40, 30, 1), (376, 8, 64, 40, 2)])
def test_tc_fvp_vs_fp32_fvp(cuda, O, A, N, T, stride):
    """Tensor-core Fisher-vector product (tangent kernel + TC backward) vs the exact-fp32 FVP kernel.  Both are
    checked against the float64 double-backward FVP at these and more shapes in
    test_natural_gradient_gpu::test_fvp_vs_fp64.  Tolerance 5e-3 l2-relative."""
    from omnisafe_b200._lib import current_stream, lib, ptr

    rng = np.random.default_rng(O * 7 + N)
    theta = oac.init_theta(O, A, seed=11)
    data = _rand_data(rng, N, T, O, A, theta)
    agent, buf, eng = _setup(cuda, data, N, T, O, A, theta)
    Pa = eng.Pa
    vec = torch.as_tensor(rng.standard_normal(Pa).astype(np.float32)).to(cuda)
    out32 = torch.zeros(Pa, device=cuda)
    outtc = torch.zeros(Pa, device=cuda)
    eng.precision = 0
    eng.fvp(vec, out32, 0.1, stride)
    eng.precision = 1
    eng.fvp(vec, outtc, 0.1, stride)
    torch.cuda.synchronize()
    a, b = out32.cpu().numpy(), outtc.cpu().numpy()
    assert np.isfinite(b).all()
    lay = oac.layout(O, A)['actor']['entries']
    for name, (off, shape) in lay.items():
        n = int(np.prod(shape))
        rel = np.linalg.norm(a[off:off + n] - b[off:off + n]) / (np.linalg.norm(a[off:off + n]) + 1e-30)
        print(f'{name}: l2-rel {rel:.2e}')
        assert rel < 5e-3, name


@pytest.mark.timeout(120)
@pytest.mark.parametrize('loss_kind', [1, 3])
def test_tc_full_batch_actor_grad(cuda, loss_kind):
    """actor_loss_grad (natural_pg.py:L150-157) in tensor-core mode -- a single network spread over one
    CTA per SM -- vs the exact-fp32 kernel."""
    rng = np.random.default_rng(21)
    N, T, O, A = 300, 70, 60, 8          # 165 tiles of 128 rows: more tiles than CTAs, ragged tail
    theta = oac.init_theta(O, A, seed=4)
    data = _rand_data(rng, N, T, O, A, theta)
    agent, buf, eng = _setup(cuda, data, N, T, O, A, theta)
    lag = torch.tensor([0.2], dtype=torch.float32, device=cuda)
    g32 = torch.zeros(eng.Pa, device=cuda)
    gtc = torch.zeros(eng.Pa, device=cuda)
    eng.snapshot_old_policy()
    eng.precision = 0
    l32 = eng.actor_loss_grad(loss_kind, lag, g32)
    eng.precision = 1
    ltc = eng.actor_loss_grad(loss_kind, lag, gtc)
    torch.cuda.synchronize()
    a, b = g32.cpu().numpy(), gtc.cpu().numpy()
    rel = np.linalg.norm(a - b) / np.linalg.norm(a)
    print('l2-rel', rel, float(l32), float(ltc))
    assert rel < 5e-3
    assert abs(float(l32) - float(ltc)) < 1e-3 * max(1.0, abs(float(l32)))


@pytest.mark.timeout(120)
@pytest.mark.parametrize('N,T', [(64, 40), (300, 70)])
def test_tc_focops_vs_fp32_kernel(cuda, N, T):
    """FOCOPS loss (first_order/focops.py:L62-108, two passes for the [b,1] x [b] broadcast) on the
    tensor-core tiles vs the exact-fp32 kernel (golden-checked against the reference in
    test_agent_gpu / test_update_gpu).  KL-mask flips at the eta boundary bound the agreement: 2e-2."""
    from omnisafe_b200._lib import current_stream, lib, ptr

    O, A = 60, 8
    rng = np.random.default_rng(N)
    theta = oac.init_theta(O, A, seed=9)
    data = _rand_data(rng, N, T, O, A, theta)
    agent, buf, eng = _setup(cuda, data, N, T, O, A, theta)
    eng.precision = 0
    eng.snapshot_old_policy()
    agent.theta[: eng.Pa].add_(torch.as_tensor(rng.standard_normal(eng.Pa).astype(np.float32) * 0.02).to(cuda))
    B = N * T
    lag = torch.tensor([0.3], dtype=torch.float32, device=cuda)
    perm = torch.as_tensor(rng.permutation(B).astype(np.int32)).to(cuda)
    start, count = 5, B - 9
    d = buf.data
    grads, stats = [], []
    for fn, nbf in ((lib().osb_minibatch_grad, lambda: lib().osb_update_grid_blocks(count)),
                    (lib().osb_minibatch_grad_tc, lambda: lib().osb_tc_grid_blocks(count, 7))):
        eng.train_stats.zero_()
        fn(ptr(agent.theta), O, A, ptr(d['obs']), ptr(d['act']), ptr(d['logp']), ptr(d['adv_r']), ptr(d['adv_c']),
           ptr(d['target_value_r']), ptr(d['target_value_c']), ptr(eng.mu_old), ptr(buf.adv_moments), ptr(perm), B, 0,
           start, count, 2, 0.2, 0.01, 1.5, 0.02, ptr(lag), ptr(eng.logstd_old), 7, ptr(eng.gpart),
           ptr(eng.stats_part), 0, current_stream())
        lib().osb_grad_reduce(ptr(eng.gpart), ptr(eng.stats_part), nbf(), O, A, ptr(agent.theta), ptr(agent.grad),
                              0.0, 7, ptr(eng.sumsq_part), ptr(agent.adam_step), ptr(eng.train_stats), 0,
                              current_stream())
        torch.cuda.synchronize()
        grads.append(agent.grad.cpu().numpy().copy())
        stats.append(eng.train_stats.cpu().numpy().copy())
    a, b = grads
    Pa = eng.Pa
    rel_actor = np.linalg.norm(a[:Pa] - b[:Pa]) / np.linalg.norm(a[:Pa])
    rel_critics = np.linalg.norm(a[Pa:] - b[Pa:]) / np.linalg.norm(a[Pa:])
    print('actor l2-rel', rel_actor, 'critics', rel_critics, stats[0][:8], stats[1][:8])
    assert rel_actor < 2e-2 and rel_critics < 5e-3
    assert abs(stats[0][0] - stats[1][0]) < 2e-2 * max(1.0, abs(stats[0][0]))
