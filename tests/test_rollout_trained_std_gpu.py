"""GPU: the rollout kernels' sampling at a trained policy std, row by row against float64, and with the std moved between
epochs.

At the reference's initial log_std = 0, sigma, 2 sigma^2 and log sigma are 1, 2 and 0 for every action, so a kernel
that takes the wrong action's sigma, stages sigma for some actions only or leaves out -log sigma writes the same slabs as
a correct one.  Here the actor's log_std is oracle.actor_critic.trained_log_std(A) (distinct per action, not monotone,
sigma 0.20 to 1.49), and every row the kernel stored is checked on its own in float64:

  act   = mu64(obs) + exp(log_std) eps          mu64: the actor MLP in float64 on the stored (normalised) row
  logp  = sum_a (-eps_a^2 / 2 - log_std_a - log(2 pi) / 2)
  value = the float64 critics on the same row

with eps the supplied noise (parity mode) or oracle/philox.py's draw at the adapter's noise seed (fast mode).  The
log-probability form does not depend on mu -- the kernel forms the action and its log-probability from one mu -- so one
fp32-level bar holds in every precision and tests the sigma algebra alone.  Because each row stands alone, the check does
not follow the trajectory, and holds where a fp32 replay of a tf32 epoch drifts.

Bars: act and values 2e-5 (fp32 tiles, bf16x3) and 5e-3 (tf32); logp 2e-5 relative + 5e-5 absolute in all three.
Largest deviations from float64 seen on an H100 80GB HBM3 (700 W) over the cases of this file (printed at the end of
a run with -s):
  fp32     act 7.4e-7, values 3.1e-7, logp 3.3e-6
  tf32     act 4.2e-4, values 3.9e-4, logp 5.0e-6
  bf16x3   act 1.1e-6, values 8.4e-7, logp 5.0e-6

The second part writes a new theta into agent.theta in place between two epochs, as the optimiser does (log_std becomes
trained_log_std + log_std_shift, every weight moves), and holds both epochs to the oracle and to the float64 rows: the
fp32 tiles read log_std per step, the persistent tensor-core kernel stages sigma once per launch, the per-step launch once
per step, and the registered-env act kernel reads it through the pointer a CUDA graph bakes in."""
import numpy as np
import pytest
import torch

import external_envs as xe
from oracle import actor_critic as oac
from oracle import philox
from oracle import rollout as orollout
from oracle.normalizer import Normalizer as ONormalizer
from oracle.synthetic_env import SyntheticBoxEnv as OEnv
from test_rollout_dims_gpu import SEED, _check, _rollout, _safety_adapter, _sm_count
from test_rollout_gpu import _model_cfgs

pytestmark = pytest.mark.gpu

RTC = 128
FP32_TOL = dict(rtol=2e-5, atol=2e-5)
TF32_TOL = dict(rtol=5e-3, atol=5e-3)
LOGP_TOL = dict(rtol=2e-5, atol=5e-5)
HALF_LOG_2PI = 0.5 * np.log(2.0 * np.pi)
DEVIATIONS = {}                           # precision -> largest deviation from float64 per slab, over the module


@pytest.fixture(scope='module', autouse=True)
def _report_deviations():
    yield
    for p, d in sorted(DEVIATIONS.items()):
        print(f'\nlargest deviation from float64 at precision {p}: ' + ', '.join(f'{k} {v:.1e}' for k, v in d.items()))


def trained_theta(On, A, seed):
    return oac.init_theta(On, A, seed=seed, log_std=oac.trained_log_std(A))


def moved_theta(theta, On, A, seed):
    """theta after some optimiser steps: log_std = trained_log_std + log_std_shift, every weight and bias moved."""
    rng = np.random.default_rng(seed)
    out = (theta + 0.02 * rng.standard_normal(theta.shape)).astype(np.float32)
    off = oac.layout(On, A)['actor']['entries']['log_std'][0]
    out[off:off + A] = oac.trained_log_std(A) + oac.log_std_shift(A)
    return out


def check_rows(sl, eps, theta, On, A, precision, what=''):
    """Every stored row of act, logp, value_r and value_c against float64 on the stored obs row."""
    nets = oac.unflatten(torch.as_tensor(np.asarray(theta, np.float64)), On, A)
    obs = torch.as_tensor(sl['obs'].astype(np.float64))
    assert obs.shape[-1] == On
    e = np.asarray(eps, np.float64)
    with torch.no_grad():
        mu = oac.mlp(nets['actor'], obs).numpy()
        v_r = oac.critic_value(nets['reward_critic'], obs).numpy()
        v_c = oac.critic_value(nets['cost_critic'], obs).numpy()
    log_std = nets['actor']['log_std'].numpy()
    want = {'act': mu + np.exp(log_std) * e, 'value_r': v_r, 'value_c': v_c,
            'logp': (-0.5 * e * e - log_std - HALF_LOG_2PI).sum(-1)}
    tol = TF32_TOL if precision == 1 else FP32_TOL
    for k, w in want.items():
        np.testing.assert_allclose(sl[k], w, **(LOGP_TOL if k == 'logp' else tol), err_msg=f'{what} {k}')
    seen = DEVIATIONS.setdefault(precision, {})
    for k, w in want.items():
        seen[k] = max(seen.get(k, 0.0), float(np.abs(sl[k] - w).max()))


def fast_eps(ad, N, T, A, epochs):
    return [philox.rollout_eps(ad.noise_seed, N, T, e, A) for e in range(epochs)]


def _synthetic(dev, N, T, O, A, theta, eps, precision, tmax=5, tp=0.05):
    """Two epochs of the fused rollout (launch shape asserted by _rollout); the noise each epoch used."""
    ad, _, outs = _rollout(dev, N, T, O, A, theta, eps, tmax, tp, precision)
    return outs, (list(eps) if eps is not None else fast_eps(ad, N, T, A, 2))


# ---- float64 rows of the kernels' own slabs --------------------------------------------------------------------------

@pytest.mark.parametrize('precision', [0, 1, 2])
@pytest.mark.parametrize('A', [1, 2, 3, 7, 8, 9, 16])
def test_rows_action_dims(cuda, A, precision):
    """Every lane layout: one action per lane on the fp32 tiles (a second trip for A > 8), action pairs from one Philox
    block for A <= 8 on the tensor-core tiles (odd A leaves half a pair idle), one action per lane for A > 8."""
    N, T, O = 129, 8, 60
    theta = trained_theta(O, A, seed=A)
    eps = np.random.default_rng(300 + A).standard_normal((2, T, N, A)).astype(np.float32)
    outs, eps = _synthetic(cuda, N, T, O, A, theta, eps, precision)
    for e, sl in enumerate(outs):
        check_rows(sl, eps[e], theta, O, A, precision, f'epoch {e}')


@pytest.mark.parametrize('precision', [0, 1, 2])
@pytest.mark.parametrize('A', [3, 16])
@pytest.mark.parametrize('O', [60, 64, 65, 111])
def test_rows_obs_dims(cuda, O, A, precision):
    """O = 64 is the widest input of the tensor-core tiles; O = 65 and 111 take the fp32 tiles in every precision."""
    N, T = 129, 8
    theta = trained_theta(O, A, seed=O + A)
    eps = np.random.default_rng(O * 7 + A).standard_normal((2, T, N, A)).astype(np.float32)
    outs, eps = _synthetic(cuda, N, T, O, A, theta, eps, precision)
    for e, sl in enumerate(outs):
        check_rows(sl, eps[e], theta, O, A, precision, f'epoch {e}')


@pytest.mark.parametrize('precision', [0, 1, 2])
@pytest.mark.parametrize('A', [1, 8, 9, 16])
def test_rows_fast_mode(cuda, A, precision):
    """In-kernel Philox noise, the rows held to float64 at oracle/philox.py's normals, two epochs."""
    N, T, O = 129, 8, 60
    theta = trained_theta(O, A, seed=50 + A)
    outs, eps = _synthetic(cuda, N, T, O, A, theta, None, precision)
    for e, sl in enumerate(outs):
        check_rows(sl, eps[e], theta, O, A, precision, f'fast epoch {e}')


@pytest.mark.timeout(300)
@pytest.mark.parametrize('fast', [False, True])
@pytest.mark.parametrize('precision', [1, 2])
@pytest.mark.parametrize('A', [3, 16])
def test_rows_per_step_launch(cuda, A, precision, fast):
    """N = 6000: more tensor-core CTAs than SMs, so one launch per step, each staging sigma again."""
    N, T, O = 6000, 5, 60
    assert -(-N // RTC) * 3 > _sm_count(cuda)
    theta = trained_theta(O, A, seed=70 + A)
    eps = None if fast else np.random.default_rng(400 + A).standard_normal((2, T, N, A)).astype(np.float32)
    outs, eps = _synthetic(cuda, N, T, O, A, theta, eps, precision, tmax=3, tp=0.02)
    for e, sl in enumerate(outs):
        check_rows(sl, eps[e], theta, O, A, precision, f'epoch {e}')


@pytest.mark.parametrize('precision', [0, 1, 2])
@pytest.mark.parametrize('O', [63, 64])
@pytest.mark.parametrize('kind', ['PPOSaute', 'PPOSimmerPID'])
def test_rows_safety_column(cuda, kind, O, precision):
    """The safety state is input column O: O = 63 stays on the tensor-core tiles, O = 64 takes the fp32 tiles."""
    from omnisafe_b200.common.buffer import VectorOnPolicyBuffer
    from omnisafe_b200.models import ConstraintActorCritic

    N, T, A = 129, 12, 3
    ad = _safety_adapter(cuda, kind, N, O, A, 6, 0.03)
    ad.precision = precision
    theta = trained_theta(O + 1, A, seed=O)
    eps = np.random.default_rng(O + 1).standard_normal((2, T, N, A)).astype(np.float32)
    agent = ConstraintActorCritic(O + 1, A, _model_cfgs(), epochs=1, device=cuda)
    agent.load_flat(theta)
    buf = VectorOnPolicyBuffer(O + 1, A, T, 0.99, 0.95, 0.95, 'gae', 0.0, True, True, num_envs=N, device=cuda)
    for e in range(2):
        ad.rollout(T, agent, buf, eps=torch.as_tensor(eps[e]).to(cuda))
        torch.cuda.synchronize()
        sl = {k: v.cpu().numpy() for k, v in buf.data.items() if v is not None}
        assert (sl['obs'][..., O] != 1).any()                       # the safety column is live
        check_rows(sl, eps[e], theta, O + 1, A, precision, f'epoch {e}')


@pytest.mark.parametrize('precision', [0, 1, 2])
@pytest.mark.parametrize('A', [1, 16])
def test_rows_early_terminated(cuda, A, precision):
    """The EarlyTerminated cost rule reads the sampled action 0."""
    from test_saute_gpu import _early_rollout

    N, T, O = 256, 30, 17
    theta = trained_theta(O, A, seed=40 + A)
    eps = np.random.default_rng(A + 5).standard_normal((T, N, A)).astype(np.float32)
    _, buf = _early_rollout(cuda, N, T, O, A, 3, theta, eps, 6, 0.03, 1.0, precision)
    sl = {k: v.cpu().numpy() for k, v in buf.data.items() if v is not None}
    assert (sl['reward'] == 0).sum() > 100                              # the rule fires
    check_rows(sl, eps, theta, O, A, precision)


@pytest.fixture(scope='module')
def graph_envs():
    from omnisafe_b200.envs import CMDP, Box, ENV_REGISTRY, env_register
    from test_external_graph_gpu import GRAPH_WIDE_ID, _graph_envs

    xe.register(CMDP, Box, env_register, ENV_REGISTRY.support_envs())
    if GRAPH_WIDE_ID not in ENV_REGISTRY.support_envs():
        for cls in _graph_envs(CMDP, Box):
            env_register(cls)
    return GRAPH_WIDE_ID


@pytest.mark.parametrize('precision', [0, 1, 2])
@pytest.mark.parametrize('graph', [False, True])
@pytest.mark.parametrize('A', [3, 9])
def test_rows_registered_env(cuda, monkeypatch, graph_envs, A, graph, precision):
    """osb_ext_act on the graph-safe WideBox, eager and under CUDA-graph replay (epoch 1 captures, epoch 2 replays)."""
    from test_external_graph_gpu import _run

    N, T, O, E = 100, 8, 45, 3
    theta = trained_theta(O, A, seed=90 + A)
    eps = np.random.default_rng(A).standard_normal((E, T, N, A)).astype(np.float32)
    ad, _, outs = _run(monkeypatch, cuda, graph_envs, N, T, O, A, 5, theta, eps, precision, E, graph)
    assert ad.captures == (1 if graph else 0)
    for e, sl in enumerate(outs):
        check_rows(sl, eps[e], theta, O, A, precision, f'epoch {e}')


# ---- sigma moves between epochs --------------------------------------------------------------------------------------

@pytest.mark.timeout(300)
@pytest.mark.parametrize('path,precision,N', [('fp32-tiles', 0, 129), ('persistent', 1, 129), ('persistent', 2, 129),
                                              ('per-step', 2, 6000)])
@pytest.mark.parametrize('A', [3, 9])
def test_sigma_moves_between_epochs(cuda, A, path, precision, N):
    """Epoch 1 at theta1, then theta2 written into agent.theta in place, epoch 2: both against the oracle (which takes
    sigma from the theta of each epoch) and against the float64 rows."""
    from omnisafe_b200._lib import lib
    from omnisafe_b200.adapter.onpolicy_adapter import OnPolicyAdapter
    from omnisafe_b200.common.buffer import VectorOnPolicyBuffer
    from omnisafe_b200.models import ConstraintActorCritic
    from test_rollout_gpu import _cfgs

    T, O, tmax, tp = 6, 60, 4, 0.05
    thetas = [trained_theta(O, A, seed=110 + A)]
    thetas.append(moved_theta(thetas[0], O, A, seed=A))
    eps = np.random.default_rng(500 + A).standard_normal((2, T, N, A)).astype(np.float32)
    ad = OnPolicyAdapter('SyntheticBox-v0', N, SEED, _cfgs(True, 16, obs_dim=O, act_dim=A, max_episode_steps=tmax,
                                                             term_prob=tp), device=cuda)
    ad.precision = precision
    agent = ConstraintActorCritic(O, A, _model_cfgs(), epochs=1, device=cuda)
    agent.load_flat(thetas[0])
    buf = VectorOnPolicyBuffer(O, A, T, 0.99, 0.95, 0.95, 'gae', 0.0, True, True, num_envs=N, device=cuda)
    env, onorm, window = OEnv(N, O, A, max_episode_steps=tmax, seed=SEED, term_prob=tp), ONormalizer((O,)), []
    before = lib().osb_launch_count()
    for e in range(2):
        agent.theta.copy_(torch.as_tensor(thetas[e]).to(cuda))
        ad.rollout(T, agent, buf, eps=torch.as_tensor(eps[e]).to(cuda))
        torch.cuda.synchronize()
        sl = {k: v.cpu().numpy() for k, v in buf.data.items() if v is not None}
        _check(sl, orollout.rollout_epoch(env, onorm, thetas[e], T, eps[e], window=window), precision)
        check_rows(sl, eps[e], thetas[e], O, A, precision, f'epoch {e}')
    persistent = lib().osb_launch_count() - before < 2 * (T + 1)
    assert persistent == (path == 'persistent')


@pytest.mark.parametrize('precision', [0, 2])
@pytest.mark.parametrize('A', [3, 9])
def test_sigma_moves_registered_env(cuda, monkeypatch, graph_envs, A, precision):
    """Epochs 0 and 1 at theta1 (eager, then capture and replay), theta2 written in place, epoch 2 replays: the graph's
    slabs equal the eager run's bit for bit, and both follow the oracle and the float64 rows at each theta."""
    from test_external_graph_gpu import _adapter, _state
    from test_external_env_gpu import _compare

    N, T, O, E = 100, 8, 45, 3
    theta1 = trained_theta(O, A, seed=120 + A)
    thetas = [theta1, theta1, moved_theta(theta1, O, A, seed=A + 1)]
    eps = np.random.default_rng(600 + A).standard_normal((E, T, N, A)).astype(np.float32)
    runs = {}
    for graph in (True, False):
        ad, agent, buf = _adapter(monkeypatch, cuda, graph_envs, N, T, O, A, 5, thetas[0], precision, graph)
        outs = []
        for e in range(E):
            agent.theta.copy_(torch.as_tensor(thetas[e]).to(cuda))
            ad.rollout(T, agent, buf, eps=torch.as_tensor(eps[e]).to(cuda))
            torch.cuda.synchronize()
            outs.append(_state(ad, buf))
        assert ad.captures == (1 if graph else 0)
        runs[graph] = outs
    for e, (x, y) in enumerate(zip(runs[True], runs[False])):
        assert x.keys() == y.keys()
        for k in x:
            assert np.array_equal(x[k], y[k]), f'epoch {e}: {k} differs between graph and eager'
    lo, hi = xe.wide_box_bounds(A)
    scale = orollout.action_scale
    monkeypatch.setattr(orollout, 'action_scale', lambda act: scale(act, lo, hi))
    env, norm = xe.WideBoxOracle(N, O, A, 7, seed=5), ONormalizer((O,))
    for e, sl in enumerate(runs[True]):
        _compare(sl, orollout.rollout_epoch(env, norm, thetas[e], T, eps[e]))
        check_rows(sl, eps[e], thetas[e], O, A, precision, f'epoch {e}')


# ---- the unmodified reference at a trained sigma ---------------------------------------------------------------------

GOLDEN_TOL = [(0, 2e-5), (2, 2e-5), (1, 5e-3)]


@pytest.mark.parametrize('precision,tol', GOLDEN_TOL)
@pytest.mark.parametrize('A', [3, 9])
def test_trained_std_golden(cuda, golden_dir, A, precision, tol):
    """rollout_ppolag_trained.npz: one epoch of the reference on the synthetic env with log_std = trained_log_std(A)."""
    from test_external_env_gpu import _check_golden
    from test_oracle_golden import trained_golden
    from test_rollout_gpu import _gpu_rollout

    g = trained_golden(golden_dir, A)
    N, T, O = int(g['N']), int(g['T']), int(g['O'])
    ad, buf, outs = _gpu_rollout(cuda, N, T, O, A, int(g['seed']), g['theta'], g['eps'][None], int(g['tmax']),
                                 float(g['term_prob']), window=10, precision=precision)
    check_rows(outs[0], g['eps'], g['theta'], O, A, precision)
    _check_golden(ad, buf, outs[0], g, tol)


@pytest.mark.parametrize('precision,tol', GOLDEN_TOL)
@pytest.mark.parametrize('graph', [False, True])
def test_trained_std_external_golden(cuda, monkeypatch, golden_dir, graph_envs, graph, precision, tol):
    """rollout_external_trained.npz: two epochs of the reference on WideBox at a trained log_std; under graph replay the
    second epoch is the first replay."""
    from test_external_env_gpu import _check_golden
    from test_external_graph_gpu import _adapter

    g = np.load(f'{golden_dir}/rollout_external_trained.npz')
    N, T, O, A, E = int(g['N']), int(g['T']), int(g['O']), int(g['A']), int(g['epochs_rolled'])
    env_id = graph_envs if graph else xe.WIDE_BOX_ID
    ad, agent, buf = _adapter(monkeypatch, cuda, env_id, N, T, O, A, int(g['seed']), g['theta'], precision, graph,
                              max_episode_steps=int(g['tmax']))
    eps = g['eps'].reshape(E, T, N, A)
    for e in range(E):
        ad.rollout(T, agent, buf, eps=torch.as_tensor(eps[e]).to(cuda))
    torch.cuda.synchronize()
    assert ad.captures == (1 if graph else 0)
    sl = {k: v.cpu().numpy() for k, v in buf.data.items() if v is not None}
    check_rows(sl, eps[-1], g['theta'], O, A, precision)
    _check_golden(ad, buf, sl, g, tol)
