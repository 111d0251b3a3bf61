"""GPU parity: fused minibatch forward/backward, optimiser, KL evaluation, Lagrange multiplier,
Fisher-vector product and CG vs the oracle and vs golden fixtures of the unmodified reference.

NETS is the table of non-tanh network specs the float64 suites (this file, test_update_tc_gpu, test_update_x3_gpu,
test_natural_gradient_gpu, test_optimizer_gpu, test_two_pass_loss_gpu) add to their tanh cases; a case's `nets` is a key
of NETS, optionally with an edge regime of the data: '+sat' (layer-1 pre-activations spread over about +-100) or '+zero'
(relu units at z = +-0 exactly), see _rand_data."""
import contextlib
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from oracle import actor_critic as oac
from oracle import learner as ol

pytestmark = pytest.mark.gpu

# (actor activation, critic activation, actor widths, critic widths)
NETS = {
    'relu': ('relu', 'relu', (64, 64), (64, 64)),                  # a single non-tanh instantiation
    'sig-sp': ('sigmoid', 'softplus', (24, 40), (8, 64)),          # ACT_MIXED; masks differ by layer and by network
    'sp-id': ('softplus', 'identity', (40, 24), (64, 8)),          # ACT_MIXED with the widths reversed
    'id-sig': ('identity', 'sigmoid', (64, 64), (33, 17)),         # a masked critic behind an unmasked actor
    'tanh-relu': ('tanh', 'relu', (64, 64), (64, 64)),             # the precision's tanh inside the mixed variant
    'sig-1': ('sigmoid', 'sigmoid', (1, 63), (63, 1)),             # extreme widths
}
SAT_RANGE = 100.0      # '+sat': the largest |layer-1 pre-activation| of every network


@pytest.fixture(autouse=True)
def _default_spec_after():
    """Launches made directly through the C ABI read the process-wide spec: leave the default (tanh, 64 wide) behind."""
    yield
    from omnisafe_b200.models.actor_critic import set_net_spec

    set_net_spec(0, 0, (64, 64), (64, 64))


def _spec(nets):
    """(NETS entry or None, edge regime or '') of a case's `nets`."""
    if nets is None:
        return None, ''
    key, _, edge = nets.partition('+')
    return NETS[key], edge


def oracle_nets(nets):
    """The oracle's network spec (oracle.actor_critic.nets) of a case; tanh 64 wide for nets=None."""
    spec, _ = _spec(nets)
    return oac.nets(*spec) if spec else contextlib.nullcontext()


def net_cases(cases, new):
    """Parameter sets of a test that gains a trailing `nets` argument: `cases` (pytest.params, e.g. sigma_cases) keep
    their ids with nets=None; each tuple of `new` ends in (..., nets) and gets the id of its values joined by '-'."""
    return ([pytest.param(*c.values, None, id=c.id) for c in cases]
            + [pytest.param(*c, id='-'.join(map(str, c))) for c in new])


def _model_cfgs(lr_actor=3e-4, lr_critic=3e-4, nets=None):
    aa, ca, ah, ch = _spec(nets)[0] or ('tanh', 'tanh', (64, 64), (64, 64))
    return NS(actor=NS(hidden_sizes=list(ah), activation=aa, lr=lr_actor),
              critic=NS(hidden_sizes=list(ch), activation=ca, lr=lr_critic),
              actor_type='gaussian_learning', linear_lr_decay=False, weight_initialization_mode='kaiming_uniform')


def _setup(dev, data, N, T, O, A, theta, lr_actor=3e-4, lr_critic=3e-4, nets=None):
    """Build agent + slab buffer from env-major `data` (as VectorOnPolicyBuffer.get() returns it); the agent's network
    spec is the one the following direct C-ABI launches use."""
    from omnisafe_b200.algorithms.engine import UpdateEngine
    from omnisafe_b200.common.buffer import VectorOnPolicyBuffer
    from omnisafe_b200.models import ConstraintActorCritic

    agent = ConstraintActorCritic(O, A, _model_cfgs(lr_actor, lr_critic, nets), epochs=1, device=dev)
    agent.load_flat(theta)
    agent.apply_net_spec()
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


def _theta(O, A, seed, trained, nets=None):
    spec, _ = _spec(nets)
    widths = dict(actor_hidden=spec[2], critic_hidden=spec[3]) if spec else {}
    return oac.init_theta(O, A, seed=seed, log_std=oac.trained_log_std(A, seed) if trained else None, **widths)


def _edge(theta, obs, O, A, nets):
    """The edge regime of `nets`, applied to theta's layer 1 (in place) and to obs (in place):
      sat:  every network's W1 and b1 scaled so that its float64 pre-activations over `obs` reach +-SAT_RANGE: past
            softplus's threshold 20, past z = -87 where sigmoid's 1 / (1 + e^-z) underflows, and sigmoid outputs
            within float32 rounding of 1, whose derivative h (1 - h) comes from the stored h;
      zero: every 5th row of obs all zeros and 8 entries of every network's b1 exactly 0, so those units see z = +-0:
            relu'(0) is 0 in torch and [h > 0] in the kernels."""
    spec, edge = _spec(nets)
    if not edge:
        return
    views = oac.unflatten(theta, O, A)
    if edge == 'zero':
        obs[::5] = 0.0
        for net in views.values():
            net['b1'][3:64:8] = 0.0
        return
    assert edge == 'sat', edge
    x = torch.as_tensor(obs, dtype=torch.float64)
    for net, width in zip(views.values(), (spec[2][0], spec[3][0], spec[3][0])):
        z = torch.nn.functional.linear(x, net['w1'][:width].double(), net['b1'][:width].double())
        s = SAT_RANGE / -float(z.min())
        net['w1'].mul_(s)
        net['b1'].mul_(s)
        z = torch.nn.functional.linear(x, net['w1'][:width].double(), net['b1'][:width].double())
        assert float(z.min()) < -0.99 * SAT_RANGE and float(z.max()) > 0.5 * SAT_RANGE, (float(z.min()), float(z.max()))
        assert (z.abs() < 5).float().mean() > 0.02, 'no units left in the unsaturated range'


def relu_kinks(theta, obs, O, A, nets, net):
    """Fraction of the relu units of `net` ('actor', 'reward_critic', 'cost_critic'), over the rows of `obs` and both
    hidden layers, whose float64 pre-activation z lies within tf32 rounding of 0: |z| < 2^-10 (sum_k |w_k x_k| + |b|)
    (both operands of every product rounded to 10 mantissa bits).  The tf32 tiles may put such a unit on the other side
    of relu's kink, which moves the sample's whole contribution through that unit: a flip, not a rounding error."""
    spec, _ = _spec(nets)
    p = {k: v.double() for k, v in oac.unflatten(np.asarray(theta, np.float32), O, A)[net].items()}
    act, (a1, a2) = (spec[0], spec[2]) if net == 'actor' else (spec[1], spec[3])
    if act != 'relu':
        return 0.0
    h, near, total = torch.as_tensor(np.asarray(obs, np.float64)), 0, 0
    for w, b, rows, cols in ((p['w1'], p['b1'], a1, O), (p['w2'], p['b2'], a2, a1)):
        w, b = w[:rows, :cols], b[:rows]
        z = h @ w.T + b
        near += int((z.abs() < 2.0 ** -10 * (h.abs() @ w.abs().T) + b.abs() * 2.0 ** -10).sum())
        total += z.numel()
        h = torch.relu(z)
    return near / total


# tf32 tiles at '+sat': a layer's inputs reach |h| ~ 100 (softplus, identity), and a tf32 operand carries 2^-11 of its
# own magnitude, not of the result's; the fp32 and bf16x3 tiles meet their 1e-4 bars on the same data, so the
# activations are right.  Measured on an H100 (700 W): worst block l2-rel 9.6e-3 (test_update_tc_gpu, sp-id, the
# identity critic's b2) and whole-vector 5.5e-3 (test_natural_gradient_gpu, the sp-id actor's ratio surrogate).
TF32_SAT_L2 = 2e-2


def tf32_bar(l2, min_cos, theta, obs, O, A, nets, net):
    """The tf32 bars (l2-relative, cosine) of `net`'s gradient for a case of `nets`: the tanh bars, raised for relu
    units near the kink to l2 sqrt(f) and cosine 1 - f with f = relu_kinks (one flipped unit-row is one term of a sum
    of f^-1 such terms; measured on an H100 (700 W) at f = 2.5e-3 to 6.7e-3: l2 0.1 to 0.53 sqrt(f)), and to
    TF32_SAT_L2 at '+sat'."""
    f = relu_kinks(theta, obs, O, A, nets, net) if nets else 0.0
    if f:
        l2, min_cos = max(l2, float(np.sqrt(f))), min(min_cos, 1.0 - f)
    if nets and _spec(nets)[1] == 'sat':
        l2 = max(l2, TF32_SAT_L2)
    return l2, min_cos


def _rand_data(rng, N, T, O, A, theta, nets=None):
    """Random batch at the policy `theta` (under the network spec of `nets`); an edge regime of `nets` edits theta's
    layer 1 in place first (_edge)."""
    B = N * T
    obs = rng.standard_normal((B, O)).astype(np.float32)
    eps = rng.standard_normal((B, A)).astype(np.float32)
    _edge(theta, obs, O, A, nets)
    with oracle_nets(nets):
        act, v_r, v_c, logp = oac.step(theta, obs, eps, O, A)
    logp = (logp + 0.3 * rng.standard_normal(B)).astype(np.float32)   # push ratios across the clip range
    return {'obs': obs, 'act': act, 'logp': logp,
            'adv_r': rng.standard_normal(B).astype(np.float32), 'adv_c': rng.standard_normal(B).astype(np.float32),
            'target_value_r': rng.standard_normal(B).astype(np.float32),
            'target_value_c': rng.standard_normal(B).astype(np.float32)}


@pytest.mark.parametrize('O,A,N,T,loss_kind,trained,nets', net_cases(sigma_cases(
    [(60, 8, 20, 13, 0), (60, 8, 32, 8, 1), (17, 6, 9, 31, 3), (111, 8, 16, 10, 0), (376, 8, 7, 20, 0)],
    # ragged last tile, A = 1, A = 16 with more tiles than CTAs, obs dims > 64; every single-pass kind
    [(60, 8, 20, 13, 0), (17, 6, 9, 31, 3), (33, 1, 50, 11, 0), (64, 16, 300, 70, 1), (111, 8, 16, 10, 1)]), [
    # NETS: ragged last tile, A = 1 (trained), A = 16 with more tiles than CTAs, obs dims > 64, the edge regimes
    (60, 8, 20, 13, 0, False, 'sig-sp'), (33, 1, 50, 11, 0, True, 'sp-id'), (64, 16, 300, 70, 1, False, 'id-sig'),
    (111, 8, 16, 10, 3, False, 'sig-1'), (17, 6, 9, 31, 3, True, 'tanh-relu'), (60, 8, 20, 13, 1, False, 'relu+zero'),
    (60, 8, 20, 13, 0, False, 'sig-sp+sat'), (60, 8, 20, 13, 1, False, 'sp-id+sat')]))
def test_minibatch_grad_vs_autograd(cuda, O, A, N, T, loss_kind, trained, nets):
    from omnisafe_b200._lib import current_stream, lib, ptr

    rng = np.random.default_rng(O + N)
    theta = _theta(O, A, 5, trained, nets)
    data = _rand_data(rng, N, T, O, A, theta, nets)
    agent, buf, eng = _setup(cuda, data, N, T, O, A, theta, nets=nets)
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
    want = torch.cat([L.flat_grad(n) for n in ol.NETS]).numpy()
    lay = oac.layout(O, A)
    worst = 0.0
    for net in ol.NETS:
        s, n = lay[net]['start'], lay[net]['size']
        scale = np.abs(want[s:s + n]).max()
        np.testing.assert_allclose(got[s:s + n], want[s:s + n], rtol=2e-4, atol=2e-5 * max(scale, 1e-3), err_msg=net)
        if nets:      # the suite's 1e-4 l2 bar per parameter block
            for name, (off, shape) in lay[net]['entries'].items():
                w, g = want[off:off + int(np.prod(shape))], got[off:off + int(np.prod(shape))]
                rel = float(np.linalg.norm(g - w) / (np.linalg.norm(w) + 1e-30))
                worst = max(worst, rel)
                assert rel < 1e-4 or not w.any() and not g.any(), (net, name, rel)
    if nets:
        print(f'[fp32 {nets} O={O} A={A} kind {loss_kind}] worst block l2-rel {worst:.2e}')
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
