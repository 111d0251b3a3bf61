"""GPU: the persistent rollout epoch (one cooperative launch, every CTA folding the normaliser sums into its own copy of
the running statistics, actor CTAs on tiles of 64 envs) against one launch per step (OSB_ROLLOUT_PER_STEP=1: the last CTA of each launch folds them
into NormState, every tile 128 envs), bit for bit.

Both paths run the same tensor-core forward and per-env arithmetic on the same seed and in-kernel Philox noise, so every
slab, the env state, every normaliser tensor and the episode window must be identical after each of two epochs (the
second one starts from the statistics the first one left in NormState).  The cases cover ragged env tiles, the largest
N whose CTAs are all resident, network inputs of 17 to 64 columns, one action, an action pair layout and A > 8, the
Saute safety column and the EarlyTerminated cost rule, in tf32 and bf16x3."""
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from test_rollout_gpu import _model_cfgs
from test_update_gpu import _theta, sigma_cases

pytestmark = pytest.mark.gpu

RTA, RTC = 64, 128      # envs per actor tile of the persistent kernel, per critic tile (and per tile of every step)
T, TMAX, TP, SEED = 12, 5, 0.05, 4


def _largest_n(dev):
    """The largest N whose CTAs (ceil(N / 64) actor tiles and ceil(N / 128) tiles per critic) are all resident."""
    sm = torch.cuda.get_device_properties(dev).multi_processor_count
    return max(n for n in range(RTC, 64 * sm, 64) if -(-n // RTA) + 2 * -(-n // RTC) <= sm)


def _adapter(dev, kind, N, O, A):
    from omnisafe_b200.adapter.early_terminated_adapter import EarlyTerminatedAdapter
    from omnisafe_b200.adapter.onpolicy_adapter import OnPolicyAdapter
    from omnisafe_b200.adapter.saute_adapter import SauteAdapter

    algo = dict(obs_normalize=True, reward_normalize=False, cost_normalize=False)
    env = dict(obs_dim=O, act_dim=A, max_episode_steps=TMAX, term_prob=TP)
    if kind == 'PPOSaute':
        algo.update(safety_budget=2.0, saute_gamma=0.999, max_ep_len=float(TMAX), unsafe_reward=-0.5)
        cls = SauteAdapter
    elif kind == 'PPOEarlyTerminated':
        algo.update(cost_limit=1.0)
        cls = EarlyTerminatedAdapter
    else:
        cls = OnPolicyAdapter
    return cls('SyntheticBox-v0', N, SEED, NS(algo_cfgs=NS(**algo), logger_cfgs=NS(window_lens=16), env_cfgs=env),
               device=dev)


def _epochs(dev, kind, N, O, A, precision, per_step, monkeypatch, trained=False):
    """Two rollout epochs; the state after each, and the number of launches they took."""
    from omnisafe_b200._lib import lib
    from omnisafe_b200.common.buffer import VectorOnPolicyBuffer
    from omnisafe_b200.models import ConstraintActorCritic

    if per_step:
        monkeypatch.setenv('OSB_ROLLOUT_PER_STEP', '1')
    else:
        monkeypatch.delenv('OSB_ROLLOUT_PER_STEP', raising=False)
    On = O + (kind == 'PPOSaute')
    ad = _adapter(dev, kind, N, O, A)
    ad.precision = precision
    agent = ConstraintActorCritic(On, A, _model_cfgs(), epochs=1, device=dev)
    agent.load_flat(_theta(On, A, O + A, trained))
    buf = VectorOnPolicyBuffer(On, A, T, 0.99, 0.95, 0.95, 'gae', 0.0, True, True, num_envs=N, device=dev)
    nz, env = ad._obs_normalizer, ad._env
    before = lib().osb_launch_count()
    states = []
    for _ in range(2):
        ad.rollout(T, agent, buf)
        torch.cuda.synchronize()
        st = {f'slab.{k}': v for k, v in buf.data.items() if v is not None}
        st.update({f'env.{k}': getattr(env, k) for k in env._STATE})
        st.update({f'norm.{k}': getattr(nz, k) for k in nz._STATE})
        st.update({'ep_ring': ad.ep_ring, 'ep_meta': ad.ep_meta, 'window_sums': ad.window_sums})
        if kind == 'PPOSaute':
            st['safety'] = ad.safety
        if kind == 'PPOEarlyTerminated':
            st['cost_acc'] = ad._cost_logger
        states.append({k: v.cpu().numpy().copy() for k, v in st.items()})
    return states, lib().osb_launch_count() - before


CASES = [   # kind, N, O, A
    ('PPOLag', 4096, 60, 8),
    ('PPOLag', 4000, 17, 1),
    ('PPOLag', 100, 64, 16),
    ('PPOLag', 'largest', 60, 8),
    ('PPOSaute', 4000, 63, 8),
    ('PPOEarlyTerminated', 4096, 17, 16),
    ('PPOEarlyTerminated', 100, 60, 1),
]


TRAINED = [c for c in CASES if c[1] in (4096, 100) or c[0] == 'PPOSaute']     # sigma per action pair, per lane, z


@pytest.mark.parametrize('kind,N,O,A,precision,trained', sigma_cases([(*c, p) for c in CASES for p in (1, 2)],
                                                                     [(*c, p) for c in TRAINED for p in (1, 2)]))
def test_persistent_epoch_matches_per_step(cuda, monkeypatch, kind, N, O, A, precision, trained):
    if N == 'largest':
        N = _largest_n(cuda)
    ref, launches_ref = _epochs(cuda, kind, N, O, A, precision, True, monkeypatch, trained)
    got, launches = _epochs(cuda, kind, N, O, A, precision, False, monkeypatch, trained)
    assert launches_ref > 2 * (T + 1) and launches < 2 * (T + 1), (launches_ref, launches)
    for e in range(2):
        assert got[e].keys() == ref[e].keys()
        for k in ref[e]:
            assert np.array_equal(got[e][k], ref[e][k]), f'epoch {e}: {k}'
    assert (ref[1]['slab.flags'] != 0).any() and ref[1]['norm.count'][0] > 2 * T * N
