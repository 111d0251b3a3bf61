"""GPU: the rollout kernels at every branch of the action dimension and at the obs-dim tile boundary, and the in-kernel
Philox noise pinned to oracle/philox.py.

The sampling code of the step kernels branches on A: the fp32 tiles give each env 8 lanes and loop a = q, q + 8 (A > 8
takes a second trip), the tensor-core tiles give each lane an action pair drawn from one Philox block for A <= 8 (odd A
leaves half a pair idle; A = 1, 2 leave most lanes idle) and one action per lane for A > 8.  The tensor-core tiles take
a network input of at most 64 columns, so O = 63 with the Saute / Simmer safety column still runs on them and O = 64
with it falls back to the fp32 tiles.  Both launch shapes of the tensor-core tiles run: the persistent kernel (every CTA
resident, one launch per epoch) and one launch per step (N = 6000: more CTAs than SMs).

Fast mode (no `eps`) draws the noise in the kernels.  Each fast-mode case is run a second time with `eps` computed by
oracle/philox.py at the adapter's noise seed, env gid and global step epoch_index * T + t: both runs must give the same
slabs within a few fp32 ulp (the accuracy of the kernels' logf / sincosf), so the kernels draw exactly the reference's
normal for each (env, step, component), and a second epoch draws new ones.  On an H100 (700 W) the largest action
deviation seen in fp32 and bf16x3 was 7.2e-7 (log_std = 0, so that is the normal's own deviation), 0.18 of FAST_TOL.

Cases whose id ends in '-trained' run the same checks with the actor's log_std at oracle.actor_critic.trained_log_std(A)
(sigma 0.20 to 1.49, distinct per action), where a sigma taken from the wrong action or staged for some actions only no
longer looks right."""
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from itertools import product

import external_envs as xe
from oracle import evaluator as eval_oracle
from oracle import philox
from oracle import rollout as orollout
from oracle.normalizer import Normalizer as ONormalizer
from oracle.synthetic_env import SyntheticBoxEnv as OEnv
from test_rollout_gpu import _compare, _gpu_rollout, _model_cfgs
from test_update_gpu import _theta, sigma_cases

pytestmark = pytest.mark.gpu

SEED = 9
RTC = 128                                 # envs per tensor-core tile
A_SWEEP = [1, 2, 3, 7, 8, 9, 12, 16]
FAST_TOL = dict(rtol=1e-6, atol=1e-6)     # fast-mode slabs vs the same rollout fed the oracle's noise


def _sm_count(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


def _persistent_expected(dev, N, On, precision):
    """The launch shape the epoch should take: tensor-core tiles (tf32 / bf16x3, network input <= 64) with every CTA of
    the env tiles x three networks resident."""
    return precision in (1, 2) and On <= 64 and -(-N // RTC) * 3 <= _sm_count(dev)


def _rollout(dev, N, T, O, A, theta, eps, tmax, term_prob, precision, epochs=2, window=16):
    """_gpu_rollout plus the launch shape it took: a persistent epoch is a handful of launches, one launch per step is
    more than T + 1 of them."""
    from omnisafe_b200._lib import lib

    before = lib().osb_launch_count()
    ad, buf, outs = _gpu_rollout(dev, N, T, O, A, SEED, theta, eps, tmax, term_prob, window=window, epochs=epochs,
                                 precision=precision)
    launches = lib().osb_launch_count() - before
    persistent = launches < epochs * (T + 1)
    assert persistent == _persistent_expected(dev, N, O, precision), (launches, epochs, T)
    return ad, buf, outs


def _compare_tf32(sl, ref):
    """The bars of test_rollout_gpu.py::test_rollout_tensor_core_mode for the TF32 GEMMs."""
    tol = dict(rtol=5e-3, atol=5e-3)
    assert np.array_equal(sl['flags'], ref['flags'])
    for k, r in (('obs', 'obs'), ('act', 'act'), ('value_r', 'val_r'), ('value_c', 'val_c'), ('reward', 'rew')):
        np.testing.assert_allclose(sl[k], ref[r], **tol, err_msg=k)
    np.testing.assert_allclose(sl['logp'], ref['logp'], rtol=5e-3, atol=2e-2)
    assert (sl['cost'] != ref['cost']).mean() < 5e-3
    need = ((ref['flags'] != 0) | (np.arange(ref['flags'].shape[0])[:, None] == ref['flags'].shape[0] - 1)) \
        & ((ref['flags'] & 1) == 0)
    np.testing.assert_allclose(sl['boot_r'][need], ref['boot_r'][need], **tol)
    np.testing.assert_allclose(sl['boot_c'][need], ref['boot_c'][need], **tol)


def _check(sl, ref, precision):
    if precision == 1:
        _compare_tf32(sl, ref)
    else:
        _compare(sl, ref, tol=2e-5)


def _check_window(ad, window, W, precision):
    """The episode ring (the last W finished episodes in order) and window_sums (its float64 column sums and count)."""
    w = np.array(window[-W:], np.float32).reshape(-1, 3)
    meta, ring, ws = ad.ep_meta.cpu().numpy(), ad.ep_ring.cpu().numpy(), ad.window_sums.cpu().numpy()
    cnt, head = int(meta[0]), int(meta[1])
    assert cnt == len(w) and cnt > 0
    order = [(head - cnt + i) % W for i in range(cnt)]
    tol = 5e-3 if precision == 1 else 2e-5
    np.testing.assert_allclose(ring[0][order], w[:, 0], rtol=tol, atol=tol)
    np.testing.assert_array_equal(ring[2][order], w[:, 2])
    if precision != 1:
        np.testing.assert_array_equal(ring[1][order], w[:, 1])
    assert ws[3] == cnt
    np.testing.assert_allclose(ws[:3], ring[:, :cnt].astype(np.float64).sum(1), rtol=1e-12, atol=1e-9)


def _oracle_epochs(N, T, O, A, theta, eps, tmax, term_prob, epochs=2, **kw):
    env = OEnv(N, O, A, max_episode_steps=tmax, seed=SEED, term_prob=term_prob)
    onorm, window = ONormalizer((O,)), []
    refs = [orollout.rollout_epoch(env, onorm, theta, T, eps[e], window=window, **kw) for e in range(epochs)]
    return refs, window


# ---- a. action-dimension sweep against the oracle --------------------------------------------------------------------

@pytest.mark.parametrize('A,precision,trained', sigma_cases(list(product(A_SWEEP, [0, 1, 2])),
                                                          list(product([1, 2, 3, 8, 9, 16], [0, 1, 2]))))
def test_action_dims_vs_oracle(cuda, A, precision, trained):
    """Every A from 1 to 16 that takes a different lane layout, two epochs (normaliser, episode counters and window
    carry over), ragged env tiles, terminations and truncations; fp32 tiles and the persistent tensor-core kernel."""
    N = 129 if A % 2 else 50
    T, O, tmax, tp, W = 10, 60, 4, 0.05, 16
    theta = _theta(O, A, A, trained)
    eps = np.random.default_rng(100 + A).standard_normal((2, T, N, A)).astype(np.float32)
    ad, _, outs = _rollout(cuda, N, T, O, A, theta, eps, tmax, tp, precision, window=W)
    refs, window = _oracle_epochs(N, T, O, A, theta, eps, tmax, tp)
    for sl, ref in zip(outs, refs):
        _check(sl, ref, precision)
    assert (refs[1]['flags'] & 1).any() and (refs[1]['flags'] & 2).any()
    _check_window(ad, window, W, precision)


@pytest.mark.timeout(300)
@pytest.mark.parametrize('A,precision,trained', sigma_cases(list(product([1, 9, 16], [1, 2])),
                                                          [(1, 2), (9, 1), (9, 2), (16, 2)]))
def test_action_dims_per_step_launch(cuda, A, precision, trained):
    """N = 6000 is more CTAs (47 tiles x 3 networks) than the H100 has SMs: the tensor-core tiles run one launch per
    step, where the step index and the noise pointer come from the host instead of the persistent loop."""
    N, T, O, tmax, tp, W = 6000, 5, 60, 3, 0.02, 64
    assert -(-N // RTC) * 3 > _sm_count(cuda)
    theta = _theta(O, A, 20 + A, trained)
    eps = np.random.default_rng(200 + A).standard_normal((2, T, N, A)).astype(np.float32)
    ad, _, outs = _rollout(cuda, N, T, O, A, theta, eps, tmax, tp, precision, window=W)
    refs, window = _oracle_epochs(N, T, O, A, theta, eps, tmax, tp)
    for sl, ref in zip(outs, refs):
        _check(sl, ref, precision)
    _check_window(ad, window, W, precision)


# ---- b. obs-dim boundaries ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize('O,A,precision,trained', sigma_cases(list(product([2, 63, 64, 65], [2, 16], [0, 1, 2])),
                                                            list(product([63, 64, 65], [2, 16], [0, 2]))
                                                            + [(64, 16, 1), (65, 16, 1)]))
def test_obs_dim_boundaries(cuda, O, A, precision, trained):
    """O = 64 is the widest input of the tensor-core tiles (one K chunk), O = 65 the narrowest that falls back to the
    fp32 tiles; O = 2 leaves most of the chunk as padding."""
    N, T, tmax, tp, W = 50, 8, 5, 0.05, 16
    theta = _theta(O, A, O + A, trained)
    eps = np.random.default_rng(O * 31 + A).standard_normal((2, T, N, A)).astype(np.float32)
    ad, _, outs = _rollout(cuda, N, T, O, A, theta, eps, tmax, tp, precision, window=W)
    refs, window = _oracle_epochs(N, T, O, A, theta, eps, tmax, tp)
    for sl, ref in zip(outs, refs):
        _check(sl, ref, precision)
    _check_window(ad, window, W, precision)


def _safety_adapter(dev, kind, N, O, A, tmax, tp):
    from omnisafe_b200.adapter.saute_adapter import SauteAdapter
    from omnisafe_b200.adapter.simmer_adapter import SimmerAdapter

    algo = dict(obs_normalize=True, reward_normalize=False, cost_normalize=False, safety_budget=2.0, saute_gamma=0.999,
                max_ep_len=float(tmax), unsafe_reward=-0.5)
    control = None
    if kind == 'PPOSimmerPID':
        algo['upper_budget'] = 5.0
        control = NS(kp=0.0005, ki=0.00001, kd=0.0, polyak=0.995)
    cfgs = NS(algo_cfgs=NS(**algo), logger_cfgs=NS(window_lens=16), control_cfgs=control,
              env_cfgs=dict(obs_dim=O, act_dim=A, max_episode_steps=tmax, term_prob=tp))
    cls = SimmerAdapter if kind == 'PPOSimmerPID' else SauteAdapter
    return cls('SyntheticBox-v0', N, SEED, cfgs, device=dev)


SAFETY_CASES = list(product(['PPOSaute', 'PPOSimmerPID'], [63, 64], [0, 2]))


@pytest.mark.parametrize('kind,O,precision,trained', sigma_cases(SAFETY_CASES, SAFETY_CASES))
def test_safety_column_at_tile_boundary(cuda, kind, O, precision, trained):
    """The safety state z is the network's column O: with O = 63 the input is 64 wide and stays on the tensor-core
    tiles, with O = 64 it is 65 wide and takes the fp32 tiles.  Against the oracle's Saute / Simmer semantics."""
    from omnisafe_b200._lib import lib
    from omnisafe_b200.common.buffer import VectorOnPolicyBuffer
    from omnisafe_b200.models import ConstraintActorCritic

    N, T, A, tmax, tp = 129, 12, 2, 6, 0.03
    ad = _safety_adapter(cuda, kind, N, O, A, tmax, tp)
    ad.precision = precision
    theta = _theta(O + 1, A, O, trained)
    eps = np.random.default_rng(O).standard_normal((2, T, N, A)).astype(np.float32)
    agent = ConstraintActorCritic(O + 1, A, _model_cfgs(), epochs=1, device=cuda)
    agent.load_flat(theta)
    buf = VectorOnPolicyBuffer(O + 1, A, T, 0.99, 0.95, 0.95, 'gae', 0.0, True, True, num_envs=N, device=cuda)
    saute = {'budget': ad._safety_budget, 'gamma': ad._saute_gamma, 'unsafe_reward': ad._unsafe_reward,
             'z0': ad._safety_init()}
    if kind == 'PPOSimmerPID':
        assert saute['z0'] < 1.0
    refs, window = _oracle_epochs(N, T, O, A, theta, eps, tmax, tp, saute=saute)
    before = lib().osb_launch_count()
    for e in range(2):
        ad.rollout(T, agent, buf, eps=torch.as_tensor(eps[e]).to(cuda))
        torch.cuda.synchronize()
        sl = {k: v.cpu().numpy() for k, v in buf.data.items() if v is not None}
        assert sl['obs'].shape == (T, N, O + 1)
        _compare(sl, refs[e], tol=2e-5)
    persistent = lib().osb_launch_count() - before < 2 * (T + 1)
    assert persistent == _persistent_expected(cuda, N, O + 1, precision)
    assert (refs[1]['rew'] == np.float32(ad._unsafe_reward)).any()          # the unsafe branch is exercised
    _check_window(ad, window, 16, precision)


@pytest.mark.parametrize('A,precision,trained', sigma_cases(list(product([1, 16], [0, 2])), list(product([1, 16], [0, 2]))))
def test_early_terminated_action_dims(cuda, A, precision, trained):
    """The EarlyTerminated cost rule reads action 0 of the sampled action in the kernel: A = 1 (a single component)
    and A = 16 (two components per lane)."""
    from test_saute_gpu import _early_rollout

    N, T, O, tmax, tp, limit = 256, 30, 17, 6, 0.03, 1.0
    theta = _theta(O, A, 40 + A, trained)
    eps = np.random.default_rng(A).standard_normal((T, N, A)).astype(np.float32)
    ad, buf = _early_rollout(cuda, N, T, O, A, 3, theta, eps, tmax, tp, limit, precision)
    env = OEnv(N, O, A, max_episode_steps=tmax, seed=3, term_prob=tp)
    early = {'cost_limit': limit, 'acc': np.zeros(N, np.float32)}
    ref = orollout.rollout_epoch(env, ONormalizer((O,)), theta, T, eps, early=early)
    sl = {k: v.cpu().numpy() for k, v in buf.data.items() if v is not None}
    _compare(sl, ref, tol=2e-5)
    assert (ref['rew'] == 0).sum() > 100                               # the rule fires
    np.testing.assert_array_equal(ad._cost_logger.cpu().numpy(), early['acc'])    # the accumulator left for the next epoch


# ---- c. fast-mode noise pinned to the reference ------------------------------------------------------------------------

def _assert_same_slabs(fast, parity, what, tf32=False):
    """Every slab of the fast-mode run (and, on registered envs, the normaliser state and the episode window) against
    the run fed the oracle's noise, epoch by epoch.  The normaliser sums observations, which reach 1e3 on WideBox, so its
    state is held relative to the array's largest entry.

    TF32 rounds the GEMM inputs to 10 mantissa bits: once a 1-ulp difference of the noise has moved an observation,
    it can cross a rounding boundary and move the next step's mean by ~1e-4.  At precision 1 only the first step of the
    first epoch, whose inputs are identical, is held to FAST_TOL; the rest is held to the TF32 bars of the oracle tests,
    still far below the spread of a wrongly drawn normal."""
    for e, (x, y) in enumerate(zip(fast, parity)):
        assert x.keys() == y.keys()
        for k in x:
            msg = f'{what} epoch {e}: {k}'
            if np.issubdtype(x[k].dtype, np.integer):
                np.testing.assert_array_equal(x[k], y[k], err_msg=msg)
            elif k.startswith('norm_') or k == 'window_sums':
                np.testing.assert_allclose(x[k], y[k], rtol=FAST_TOL['rtol'],
                                           atol=FAST_TOL['atol'] * max(1.0, float(np.abs(y[k]).max())), err_msg=msg)
            elif tf32 and k == 'cost':
                assert (x[k] != y[k]).mean() < 5e-3, msg
            elif tf32:
                np.testing.assert_allclose(x[k], y[k], rtol=5e-3, atol=2e-2 if k == 'logp' else 5e-3, err_msg=msg)
            else:
                np.testing.assert_allclose(x[k], y[k], **FAST_TOL, err_msg=msg)
    if tf32:
        for k in ('act', 'logp'):
            np.testing.assert_allclose(fast[0][k][0], parity[0][k][0], **FAST_TOL, err_msg=f'{what} step 0: {k}')


FAST_SHAPES = [(0, 129), (1, 129), (2, 129), (1, 6000), (2, 6000)]


@pytest.mark.timeout(300)
@pytest.mark.parametrize('A,precision,N,trained', sigma_cases(
    [(A, *s) for A, s in product([1, 2, 3, 8, 9, 16], FAST_SHAPES)],
    [(A, *s) for A, s in product([1, 3, 9, 16], [(0, 129), (1, 129), (2, 129), (2, 6000)])]))
def test_fast_mode_noise_matches_oracle(cuda, A, precision, N, trained):
    """Fast mode against the same rollout fed oracle/philox.py's noise, two epochs, the fp32 tiles, the persistent
    tensor-core kernel (N = 129) and its per-step launch (N = 6000)."""
    T, O, tmax, tp = (8, 60, 5, 0.05) if N < 1000 else (5, 60, 3, 0.02)
    theta = _theta(O, A, 60 + A, trained)
    ad, _, fast = _rollout(cuda, N, T, O, A, theta, None, tmax, tp, precision)
    eps = np.stack([philox.rollout_eps(ad.noise_seed, N, T, e, A) for e in range(2)])
    _, _, parity = _rollout(cuda, N, T, O, A, theta, eps, tmax, tp, precision)
    _assert_same_slabs(fast, parity, 'synthetic env', tf32=precision == 1)
    assert not np.array_equal(fast[0]['act'], fast[1]['act'])


# ---- d. fast mode on registered envs -----------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def graph_envs():
    from omnisafe_b200.envs import CMDP, Box, ENV_REGISTRY, env_register
    from test_external_graph_gpu import GRAPH_WIDE_ID, _graph_envs

    xe.register(CMDP, Box, env_register, ENV_REGISTRY.support_envs())
    if GRAPH_WIDE_ID not in ENV_REGISTRY.support_envs():
        for cls in _graph_envs(CMDP, Box):
            env_register(cls)
    return GRAPH_WIDE_ID


REGISTERED_CASES = list(product([3, 9], [False, True], [0, 2]))


@pytest.mark.parametrize('A,graph,precision,trained', sigma_cases(REGISTERED_CASES, REGISTERED_CASES))
def test_fast_mode_noise_registered_env(cuda, monkeypatch, graph_envs, A, graph, precision, trained):
    """The act kernel of the external-env path draws at act_global_step: the host's epoch_index * T + t when eager,
    the device epoch counter under graph replay (epoch 1 captures and replays, epoch 2 replays)."""
    from test_external_graph_gpu import _run

    N, T, O, E = 100, 8, 45, 3
    theta = _theta(O, A, 80 + A, trained)
    ad, _, fast = _run(monkeypatch, cuda, graph_envs, N, T, O, A, 5, theta, None, precision, E, graph)
    eps = np.stack([philox.rollout_eps(ad.noise_seed, N, T, e, A) for e in range(E)])
    ad2, _, parity = _run(monkeypatch, cuda, graph_envs, N, T, O, A, 5, theta, eps, precision, E, graph)
    assert ad.captures == ad2.captures == (1 if graph else 0)
    _assert_same_slabs(fast, parity, 'WideBox graph' if graph else 'WideBox eager')
    assert (fast[-1]['flags'] & 1).any() and (fast[-1]['flags'] & 2).any()


# ---- e. evaluation kernel ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize('precision', ['fp32', 'bf16x3'])
@pytest.mark.parametrize('A', [1, 16])
def test_evaluator_action_dims(cuda, tmp_path, A, precision, capsys):
    """osb_eval_synthetic's deterministic action at A = 1 and 16 against oracle/evaluator.py, 256 envs."""
    from omnisafe_b200 import Evaluator
    from test_evaluate_gpu import random_case, write_run

    O, E, n = 60, 256, 300
    cfg, pi, norm = random_case(O, A, seed=A)
    ev = Evaluator()
    ev.load_saved(write_run(tmp_path, cfg, pi, norm, precision), 'epoch-0.pt')
    rets, costs = ev.evaluate(num_episodes=n, cost_criteria=0.99, num_envs=E)
    capsys.readouterr()
    r, c, ln, nz = eval_oracle.evaluate(pi, norm, cfg['env_cfgs'], n, 0.99, num_envs=E)
    np.testing.assert_array_equal(ev.episode_lengths, ln)
    np.testing.assert_allclose(rets, r, rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(costs, c, rtol=1e-4, atol=1e-4)
    assert int(ev.normalizer.count[0]) == nz.count
    np.testing.assert_allclose(ev.normalizer.mean.cpu().numpy(), nz.mean, rtol=1e-4, atol=1e-4)
    assert ev.last_actions.shape[-1] == A
