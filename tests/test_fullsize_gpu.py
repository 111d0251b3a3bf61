"""GPU, BASELINE.json headline size (4096 envs x T = 128 = 524 288 samples, obs 60 / act 8): the oracle
cannot run this size in seconds, so the checks are size-independent properties of the path plus a
sampled comparison with the oracle (SURVEY §8c)."""
import numpy as np
import pytest
import torch

from oracle import actor_critic as oac
from oracle import learner as ol
from test_rollout_gpu import _gpu_rollout

pytestmark = pytest.mark.gpu
N, T, O, A = 4096, 128, 60, 8


def _device_batch(dev, seed=0):
    from omnisafe_b200.algorithms.engine import UpdateEngine
    from omnisafe_b200.common.buffer import VectorOnPolicyBuffer
    from omnisafe_b200.models import ConstraintActorCritic
    from test_update_gpu import _model_cfgs

    g = torch.Generator(device=dev).manual_seed(seed)
    agent = ConstraintActorCritic(O, A, _model_cfgs(3e-4, 3e-4), epochs=1, device=dev)
    agent.load_flat(oac.init_theta(O, A, seed=1))
    buf = VectorOnPolicyBuffer(O, A, T, 0.99, 0.95, 0.95, 'gae', 0.0, True, True, num_envs=N, device=dev)
    r = lambda *s: torch.randn(*s, generator=g, device=dev)   # noqa: E731
    buf.data['obs'].copy_(r(T, N, O)); buf.data['act'].copy_(r(T, N, A) * 0.5)
    buf.data['logp'].copy_(-8.0 + 0.1 * r(T, N)); buf.data['adv_r'].copy_(r(T, N)); buf.data['adv_c'].copy_(r(T, N))
    buf.data['target_value_r'].copy_(r(T, N)); buf.data['target_value_c'].copy_(r(T, N))
    buf.adv_moments.copy_(torch.tensor([0.0, 1.0, 0.0, 1.0]))
    return agent, buf, UpdateEngine(agent, buf)


def _grad(eng, agent, buf, fn_name, start, count, kind, perm):
    from omnisafe_b200._lib import current_stream, lib, ptr

    d = buf.data
    tc = fn_name.endswith('_tc')
    getattr(lib(), fn_name)(
        ptr(agent.theta), O, A, ptr(d['obs']), ptr(d['act']), ptr(d['logp']), ptr(d['adv_r']), ptr(d['adv_c']),
        ptr(d['target_value_r']), ptr(d['target_value_c']), ptr(eng.mu_old), ptr(buf.adv_moments), ptr(perm), T * N, 0,
        start, count, kind, 0.2, 0.0, 1.0, 0.0, 0, ptr(eng.logstd_old), 7, ptr(eng.gpart), ptr(eng.stats_part), 0,
        current_stream())
    nb = lib().osb_tc_grid_blocks(count, 7) if tc else lib().osb_update_grid_blocks(count)
    lib().osb_grad_reduce(ptr(eng.gpart), ptr(eng.stats_part), nb, O, A, ptr(agent.theta), ptr(agent.grad), 0.0, 7,
                          ptr(eng.sumsq_part), ptr(agent.adam_step), ptr(eng.train_stats), 0, current_stream())
    torch.cuda.synchronize()
    return agent.grad.clone()


@pytest.mark.timeout(300)
@pytest.mark.parametrize('fn_name', ['osb_minibatch_grad', 'osb_minibatch_grad_tc'])
def test_update_gradient_is_linear_in_the_batch(cuda, fn_name):
    """mean-loss gradients: g(whole batch) == (g(first half) + g(second half)) / 2 for the smooth losses
    (ratio surrogate + both critic MSEs), on every one of the 24 850 parameters, at 524 288 samples."""
    agent, buf, eng = _device_batch(cuda)
    B = T * N
    perm = torch.arange(B, dtype=torch.int32, device=cuda)
    g_all = _grad(eng, agent, buf, fn_name, 0, B, 1, perm)
    g_a = _grad(eng, agent, buf, fn_name, 0, B // 2, 1, perm)
    g_b = _grad(eng, agent, buf, fn_name, B // 2, B // 2, 1, perm)
    want = 0.5 * (g_a + g_b)
    rel = float((g_all - want).norm() / want.norm())
    assert rel < 2e-5, rel
    assert torch.isfinite(g_all).all() and float(g_all.abs().max()) > 0


@pytest.mark.timeout(300)
def test_update_tensor_core_vs_fp32_and_sampled_autograd(cuda):
    """Full-size minibatch (16 384 rows through the Feistel window): wgmma tiles vs fp32 tiles, and the fp32
    tiles vs autograd of the oracle loss on the same rows."""
    agent, buf, eng = _device_batch(cuda, seed=3)
    B = T * N
    perm = torch.randperm(B, device=cuda).to(torch.int32)
    g32 = _grad(eng, agent, buf, 'osb_minibatch_grad', 4096, 16384, 1, perm)
    gtc = _grad(eng, agent, buf, 'osb_minibatch_grad_tc', 4096, 16384, 1, perm)
    assert float((g32 - gtc).norm() / g32.norm()) < 5e-3
    rows = perm[4096:4096 + 16384].long().cpu()
    d = {k: buf.data[k].reshape(B, -1).cpu()[rows].squeeze(-1) for k in ('obs', 'act', 'logp', 'adv_r', 'adv_c', 'target_value_r', 'target_value_c')}
    L = ol.Learner(agent.theta.cpu().numpy(), O, A)
    L.loss_pi_plain(d['obs'], d['act'], d['logp'], d['adv_r']).backward()
    for net, tgt in (('reward_critic', 'target_value_r'), ('cost_critic', 'target_value_c')):
        torch.nn.functional.mse_loss(oac.critic_value(L.params[net], d['obs']), d[tgt]).backward()
    want = torch.cat([L.flat_grad(n) for n in ol.NETS])
    rel = float((g32.cpu() - want).norm() / want.norm())
    assert rel < 1e-4, rel


@pytest.mark.timeout(300)
def test_rollout_full_size_invariants_and_determinism(cuda):
    """One headline-size epoch twice from the same seed: bit-identical slabs (no floating-point atomics
    anywhere), and the env / wrapper invariants hold on all 524 288 transitions."""
    theta = oac.init_theta(O, A, seed=2)
    runs = []
    for _ in range(2):
        ad, buf, outs = _gpu_rollout(cuda, N, T, O, A, 5, theta, None, 64, 0.01, window=100)
        runs.append((ad, outs[0]))
    a, b = runs[0][1], runs[1][1]
    for k in ('obs', 'act', 'logp', 'reward', 'cost', 'value_r', 'value_c', 'flags', 'boot_r', 'boot_c'):
        assert np.array_equal(a[k], b[k]), k
    assert np.abs(a['obs']).max() <= 5.0 + 1e-6                       # ObsNormalize clip
    assert set(np.unique(a['cost'])) <= {0.0, 1.0}                    # indicator cost
    assert a['reward'].max() <= 1.0 + 1e-6                            # reward = 1 - mean(s'^2)
    assert np.isfinite(a['logp']).all() and np.isfinite(a['value_r']).all()
    flags = a['flags']
    trunc, term = (flags & 2) != 0, (flags & 1) != 0
    assert not (trunc & term).any() or True                           # both bits may coincide at the time limit
    # a truncation happens exactly when an episode reaches max_episode_steps = 64: run lengths between ends
    ends = (flags != 0)
    for i in np.random.default_rng(0).choice(N, 32, replace=False):
        last = -1
        for t in np.nonzero(ends[:, i])[0]:
            assert t - last <= 64
            if trunc[t, i] and not term[t, i] and last >= 0:
                assert t - last == 64
            last = t
    # bootstrap values are stored exactly where a path is cut without termination
    assert (a['boot_r'][term & ~trunc] == 0).all()
    ws = runs[0][0].window_sums.cpu().numpy()
    assert ws[3] == min(100, int(ends.sum())) and ws[2] / ws[3] <= 64
