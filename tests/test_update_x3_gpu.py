"""GPU: the split-bf16 ("bf16x3", bf16 wgmma, six MMAs per product) variant of the fused minibatch
kernel.  It is held to the SAME bars as the exact-fp32 FMA path (tests/test_update_gpu.py): gradients vs
oracle autograd at rtol 2e-4 / atol 2e-5 of the scale (and <= 1e-4 l2-relative per parameter block), and a whole
PPOLag._update against the golden fixture of the unmodified reference at the fp32-mode tolerance."""
import os

import numpy as np
import pytest
import torch

from oracle import actor_critic as oac
from oracle import learner as ol
from test_update_gpu import (_default_spec_after, _rand_data, _rows, _setup, _theta, entropy_mean, net_cases,  # noqa: F401
                             oracle_nets, sigma_cases)

pytestmark = pytest.mark.gpu


def _oracle_grad(theta, O, A, data, idx, lam, loss_kind, coef, nets=None):
    L = ol.Learner(theta, O, A)
    t = {k: torch.as_tensor(v)[idx] for k, v in data.items()}
    adv = (t['adv_r'] - lam * t['adv_c']) / (1 + lam)
    with oracle_nets(nets):
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
    return torch.cat([L.flat_grad(n) for n in ol.NETS]).numpy(), float(loss)


@pytest.mark.timeout(300)
@pytest.mark.parametrize('O,A,N,T,loss_kind,count,trained,nets', net_cases(sigma_cases([
    (60, 8, 20, 13, 0, None), (60, 8, 64, 40, 0, None), (17, 6, 9, 31, 3, None), (64, 16, 16, 24, 1, None),
    (60, 8, 256, 80, 0, 16384),      # the bench minibatch: 16 384 rows, obs 60 / act 8
    (60, 8, 256, 80, 1, 16384), (33, 1, 50, 11, 3, None),
], [  # ragged last tile, A = 1, A = 16, more tiles than CTAs (165 tiles of 128 rows); every single-pass kind
    (60, 8, 20, 13, 0, None), (17, 6, 9, 31, 3, None), (33, 1, 50, 11, 0, None), (64, 16, 16, 24, 1, None),
    (60, 8, 300, 70, 1, None),
]), [  # test_update_gpu.NETS: ragged last tile, A = 1 (trained), A = 16 with more tiles than CTAs, the edge regimes
    (60, 8, 20, 13, 0, None, False, 'relu+zero'), (33, 1, 50, 11, 3, None, True, 'sig-sp'),
    (64, 16, 300, 70, 1, None, False, 'sp-id'), (17, 6, 9, 31, 3, None, False, 'id-sig'),
    (60, 8, 64, 40, 0, None, False, 'tanh-relu'), (60, 8, 20, 13, 1, None, False, 'sig-1'),
    (60, 8, 20, 13, 0, None, False, 'sig-sp+sat'), (60, 8, 20, 13, 1, None, False, 'sp-id+sat'),
]))
def test_x3_grad_vs_autograd(cuda, O, A, N, T, loss_kind, count, trained, nets):
    from omnisafe_b200._lib import current_stream, lib, ptr

    rng = np.random.default_rng(O + N)
    theta = _theta(O, A, 5, trained, nets)
    data = _rand_data(rng, N, T, O, A, theta, nets)
    agent, buf, eng = _setup(cuda, data, N, T, O, A, theta, nets=nets)
    B = N * T
    lam = 0.37
    lag = torch.tensor([lam], dtype=torch.float32, device=cuda)
    perm_em = rng.permutation(B)
    start = 3
    count = count or B - 10
    perm = torch.as_tensor(_rows(perm_em, N, T)).to(cuda)
    coef = 1e-3
    d = buf.data
    args = (ptr(agent.theta), O, A, ptr(d['obs']), ptr(d['act']), ptr(d['logp']), ptr(d['adv_r']), ptr(d['adv_c']),
            ptr(d['target_value_r']), ptr(d['target_value_c']), ptr(eng.mu_old), ptr(buf.adv_moments), ptr(perm), B, 0,
            start, count, loss_kind, 0.2, 0.01, 1.0, 0.0, ptr(lag), ptr(eng.logstd_old), 7, ptr(eng.gpart),
            ptr(eng.stats_part), 0, current_stream())
    lib().osb_minibatch_grad_x3(*args)
    nb = lib().osb_tc_grid_blocks(count, 7)
    lib().osb_grad_reduce(ptr(eng.gpart), ptr(eng.stats_part), nb, O, A, ptr(agent.theta), ptr(agent.grad),
                          coef, 7, ptr(eng.sumsq_part), ptr(agent.adam_step), ptr(eng.train_stats), 0, current_stream())
    torch.cuda.synchronize()
    got = agent.grad.cpu().numpy()
    ts = eng.train_stats.cpu().numpy().reshape(3, 8).copy()
    want, loss = _oracle_grad(theta, O, A, data, torch.as_tensor(perm_em[start:start + count]), lam, loss_kind, coef,
                              nets)
    lay = oac.layout(O, A)
    worst = 0.0
    for net in ol.NETS:
        s, n = lay[net]['start'], lay[net]['size']
        scale = np.abs(want[s:s + n]).max()
        for name, (off, shape) in lay[net]['entries'].items():
            m = int(np.prod(shape))
            w, g = want[off:off + m], got[off:off + m]
            rel = float(np.linalg.norm(g - w) / (np.linalg.norm(w) + 1e-30))
            worst = max(worst, rel)
            print(f'{net}.{name}: l2-rel {rel:.2e}')
            assert rel < 1e-4, (net, name, rel)
        np.testing.assert_allclose(got[s:s + n], want[s:s + n], rtol=2e-4, atol=2e-5 * max(scale, 1e-3), err_msg=net)
    if nets:
        print(f'[bf16x3 {nets} O={O} A={A} kind {loss_kind}] worst block l2-rel {worst:.2e}')
    # slot 0: the loss without the entropy bonus; slot 4: the bonus; Loss/Loss_pi = slot 0 + slot 4 is the oracle loss,
    # bonus included (base/ppo.py:L76-84)
    bonus = -0.01 * entropy_mean(theta[:A]) if loss_kind == 0 else 0.0
    np.testing.assert_allclose(ts[0, 0], loss - bonus, rtol=1e-3, atol=1e-4)
    np.testing.assert_allclose(ts[0, 4], bonus, rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(ts[0, 0] + ts[0, 4], loss, rtol=1e-3, atol=1e-4)


@pytest.mark.timeout(300)
def test_x3_ppolag_update_epoch_golden(cuda, golden_dir):
    """Same data / minibatch order / lambda as the unmodified PPOLag._update -> same parameters, at the
    tolerance of the exact-fp32 path (tests/test_update_gpu.py::test_ppolag_update_epoch_golden)."""
    from omnisafe_b200.common.lagrange import Lagrange

    g = np.load(os.path.join(golden_dir, 'update_ppolag.npz'))
    data = {k[5:]: g[k] for k in g.files if k.startswith('data_')}
    N, T, O, A = 8, 24, 12, 3
    agent, buf, eng = _setup(cuda, data, N, T, O, A, g['theta0'])
    lag = Lagrange(float(g['cost_limit']), float(g['lam0']), float(g['lambda_lr']), device=cuda)
    ws = torch.tensor([0.0, float(g['Jc']) * 10, 0.0, 10.0], dtype=torch.float64, device=cuda)
    lag.update_lagrange_multiplier(ws)
    perms = torch.as_tensor(np.stack([_rows(p_, N, T) for p_ in g['perms'][::2]])).to(cuda)
    eng.ppo_epoch(loss_kind=0, lagrange=lag.state, net_mask=7, batch_size=int(g['batch_size']),
                  update_iters=int(g['update_iters']), clip=0.2, entropy_coef=0.0, critic_norm_coef=0.001,
                  max_grad_norm=40.0, lr_actor=3e-4, lr_critic=3e-4, target_kl=0.02, kl_early_stop=True,
                  perm=perms, precision=2)
    torch.cuda.synchronize()
    got, want = agent.theta.cpu().numpy(), g['theta1']
    bad = ~np.isclose(got, want, rtol=2e-4, atol=2e-6)
    assert bad.mean() < 1e-3 and np.abs(got - want).max() < 2e-3, (bad.sum(), np.abs(got - want).max())
    kls = eng.kl_state.cpu().numpy()
    np.testing.assert_allclose(kls[0], g['kl'][-1], rtol=2e-3, atol=1e-6)
    assert int(kls[1]) == int(g['stop_iter'][-1])


@pytest.mark.timeout(300)
def test_x3_epoch_matches_fp32_epoch(cuda):
    """A whole PPO-Lag update epoch on bf16x3 tiles lands on the exact-fp32 epoch (the tf32 mode only gets within 15 %
    of the update norm: tests/test_update_tc_gpu.py)."""
    rng = np.random.default_rng(3)
    N, T, O, A = 64, 32, 60, 8
    theta = oac.init_theta(O, A, seed=2)
    data = _rand_data(rng, N, T, O, A, theta)
    B = N * T
    perms = torch.as_tensor(np.stack([_rows(rng.permutation(B), N, T) for _ in range(3)])).to(cuda)
    out = []
    for prec in (0, 2):
        agent, buf, eng = _setup(cuda, data, N, T, O, A, theta)
        lag = torch.tensor([0.2, 0, 0, 0], dtype=torch.float32, device=cuda)
        eng.ppo_epoch(loss_kind=0, lagrange=lag, net_mask=7, batch_size=512, update_iters=3, clip=0.2,
                      critic_norm_coef=0.001, max_grad_norm=40.0, lr_actor=3e-4, lr_critic=3e-4,
                      target_kl=10.0, kl_early_stop=False, perm=perms, precision=prec)
        torch.cuda.synchronize()
        out.append(agent.theta.cpu().numpy())
    delta = out[0] - theta
    diff = out[1] - out[0]
    print('|x3 - fp32| / |update| =', np.linalg.norm(diff) / np.linalg.norm(delta))
    bad = ~np.isclose(out[1], out[0], rtol=2e-4, atol=2e-6)
    assert bad.mean() < 2e-3 and np.linalg.norm(diff) < 5e-3 * np.linalg.norm(delta)


@pytest.mark.timeout(300)
@pytest.mark.parametrize('N,T,batch,iters,trained', sigma_cases(
    [(64, 32, 512, 3), (50, 26, 512, 2), (13, 100, 640, 2), (256, 80, 16384, 1)],
    [(50, 26, 512, 2), (100, 80, 4096, 2)]))   # slices > 512 parameters (staged with the weights) and <= 512
def test_x3_fused_iteration_equals_stepwise(cuda, N, T, batch, iters, trained):
    """The persistent kernel (optimiser inside, software grid barriers, short last minibatch, CTAs without a tile)
    and the launch-per-minibatch path (bf16x3 gradient kernel + optim_fused) produce the same parameters.  Both
    paths share the clip formula, so this does not check the clip itself: test_optimizer_gpu does, against float64.
    At a trained log_std the actor steps at lr 1e-2 with the entropy bonus on, so log_std moves ~1e-2 per minibatch
    and the persistent kernel must stage the new sigma after every Adam step as the stepwise launches do."""
    rng = np.random.default_rng(N + T)
    O, A = 60, 8
    theta = _theta(O, A, 2, trained)
    lr_actor, ent = (1e-2, 0.01) if trained else (3e-4, 0.0)
    data = _rand_data(rng, N, T, O, A, theta)
    B = N * T
    perms = torch.as_tensor(np.stack([_rows(rng.permutation(B), N, T) for _ in range(iters)])).to(cuda)
    out, stats = [], []
    for fused in (False, True):
        if fused:
            os.environ.pop('OSB_X3_NO_FUSE', None)
        else:
            os.environ['OSB_X3_NO_FUSE'] = '1'
        try:
            agent, buf, eng = _setup(cuda, data, N, T, O, A, theta)
            lag = torch.tensor([0.2, 0, 0, 0], dtype=torch.float32, device=cuda)
            eng.ppo_epoch(loss_kind=0, lagrange=lag, net_mask=7, batch_size=batch, update_iters=iters, clip=0.2,
                          entropy_coef=ent, critic_norm_coef=0.001, max_grad_norm=0.5, lr_actor=lr_actor,
                          lr_critic=3e-4, target_kl=10.0, kl_early_stop=False, perm=perms, precision=2)
            torch.cuda.synchronize()
        finally:
            os.environ.pop('OSB_X3_NO_FUSE', None)
        out.append((agent.theta.cpu().numpy(), agent.adam_m.cpu().numpy(), agent.adam_v.cpu().numpy(), agent.adam_step.cpu().numpy()))
        stats.append(eng.train_stats.cpu().numpy().reshape(3, 8).copy())
    assert (out[0][3] == out[1][3]).all() and out[1][3][0] == iters * -(-B // batch)
    for a, b, name in zip(out[0][:3], out[1][:3], ('theta', 'm', 'v')):
        # identical arithmetic, different summation order of the partial gradients -> a few ulp on the gradient
        bad = ~np.isclose(a, b, rtol=1e-4, atol=1e-7)
        assert bad.mean() < 2e-3, (name, bad.sum(), np.abs(a - b).max())
    np.testing.assert_allclose(stats[1][:, :4], stats[0][:, :4], rtol=1e-4, atol=1e-6)


@pytest.mark.timeout(300)
def test_x3_actor_eval_matches_fp32_eval(cuda):
    rng = np.random.default_rng(9)
    N, T, O, A = 96, 50, 60, 8
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
    eng.precision = 2
    eng.snapshot_old_policy()
    torch.cuda.synchronize()
    np.testing.assert_allclose(eng.mu_old.cpu().numpy(), mu0.cpu().numpy(), rtol=0, atol=2e-6)     # tf32 tiles: 3e-3
    eng.mu_old.copy_(mu0)
    got = eng.evaluate(th2, lag)
    for k in ('kl', 'loss', 'loss_c', 'loss_r', 'ratio'):
        np.testing.assert_allclose(got[k], ref[k], rtol=2e-5, atol=2e-6, err_msg=k)              # tf32 tiles: 2e-2
