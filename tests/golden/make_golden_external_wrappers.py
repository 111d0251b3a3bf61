"""Generate tests/golden/rollout_external_wrappers.npz and rollout_external_autoreset.npz: two epochs of the UNMODIFIED
reference OnPolicyAdapter.rollout (PPOLag) with a single env, as upstream supports it, on test CMDPs of
tests/wrapper_envs.py that never reset themselves and declare the wrappers, so that the reference wraps them in
TimeLimit and AutoReset (online_adapter.py:L120-131):

- rollout_external_wrappers.npz: WrappedBox-v0, both wrappers, a small max_episode_steps; the env raises its own
  truncated now and then (TimeLimit discards it) and sometimes terminates in the step the limit hits;
- rollout_external_autoreset.npz: AutoResetBox-v0, AutoReset only, the env's own truncation ending episodes.

In both an episode is still running at the epoch boundary.

    python tests/golden/make_golden_external_wrappers.py

Like make_golden.py it needs the reference sources (imported through oracle/ref_shim.py) and runs on the CPU; only its
output is committed.  Besides the slabs it stores the env's own terminated / truncated flags of every step (env_term /
env_trunc), which the tests use to check the fixture's coverage.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))          # tests/ (wrapper_envs)
import make_golden as mg  # noqa: E402  (installs the reference shim)

import external_envs as xe  # noqa: E402
import wrapper_envs as we  # noqa: E402
from gymnasium.spaces import Box  # noqa: E402  (shim)
from omnisafe.envs.core import CMDP, env_register, support_envs  # noqa: E402


def gen(env_id, fname, seed=45, T=64, O=45, A=3, tmax=4, epochs_rolled=2):
    from omnisafe.algorithms import registry
    from omnisafe.envs.wrapper import AutoReset, TimeLimit
    from omnisafe.utils.config import get_default_kwargs_yaml
    from omnisafe.utils.tools import recursive_check_config
    import torch.distributions.normal as tdn

    N, algo_name = 1, 'PPOLag'
    we.register(CMDP, Box, env_register, support_envs())
    cfgs = get_default_kwargs_yaml(algo_name, env_id, 'on-policy')
    custom = {
        'seed': seed,
        'train_cfgs': {'vector_env_nums': N, 'total_steps': N * T * 2, 'torch_threads': 1},
        'algo_cfgs': {'steps_per_epoch': N * T, 'batch_size': 32, 'update_iters': 2},
        'logger_cfgs': {'use_tensorboard': False, 'use_wandb': False, 'log_dir': '/tmp/osb_golden_runs', 'window_lens': 10},
    }
    recursive_check_config(custom, cfgs)
    cfgs.recurisve_update(custom)
    cfgs.recurisve_update({'env_cfgs': {'obs_dim': O, 'act_dim': A, 'max_episode_steps': tmax}})
    cfgs.recurisve_update({'exp_name': f'{algo_name}-golden-wrappers', 'env_id': env_id, 'algo': algo_name})
    cfgs.train_cfgs.recurisve_update({'epochs': 2})
    algo = registry.get(algo_name)(env_id=env_id, cfgs=cfgs)
    assert not cfgs.algo_cfgs.reward_normalize and not cfgs.algo_cfgs.cost_normalize
    theta = mg._flat_theta(algo._actor_critic)
    adapter = algo._env
    chain, w = [], adapter._env
    while hasattr(w, '_env'):
        chain.append(type(w))
        w = w._env
    time_limit = bool(w.need_time_limit_wrapper)
    assert AutoReset in chain and (TimeLimit in chain) == time_limit, chain
    # the env's own flags of every step, recorded below the wrapper chain
    env_term, env_trunc = [], []
    inner_step = w.step

    def rec_step(action):
        out = inner_step(action)
        env_term.append(bool(out[3].reshape(-1)[0]))
        env_trunc.append(bool(out[4].reshape(-1)[0]))
        return out

    w.step = rec_step
    drawn, orig = [], tdn._standard_normal

    def rec(shape, dtype, device):
        e = orig(shape, dtype, device)
        drawn.append(e.clone())
        return e

    tdn._standard_normal = rec
    try:
        for e in range(epochs_rolled):
            if e > 0:
                algo._buf.get()
            adapter.rollout(steps_per_epoch=T, agent=algo._actor_critic, buffer=algo._buf, logger=algo._logger)
    finally:
        tdn._standard_normal = orig
    eps = np.stack([d.numpy() for d in drawn if tuple(d.shape) == (N, A)])
    assert eps.shape[0] == T * epochs_rolled, eps.shape
    fields = ('obs', 'act', 'reward', 'cost', 'value_r', 'value_c', 'logp', 'adv_r', 'adv_c', 'target_value_r',
              'target_value_c')
    data = {k: np.stack([b.data[k].numpy().copy() for b in algo._buf.buffers], 1) for k in fields}
    window = {k: np.array(list(algo._logger._data[k]), np.float32) for k in ('Metrics/EpRet', 'Metrics/EpCost', 'Metrics/EpLen')}
    norm = adapter._env
    while not hasattr(norm, '_obs_normalizer'):
        norm = norm._env
    nz = norm._obs_normalizer

    # the fixture must exercise what it is for (over both epochs)
    env_term = np.array(env_term).reshape(epochs_rolled, T)
    env_trunc = np.array(env_trunc).reshape(epochs_rolled, T)
    steps, done, trunc = 0, [], []
    for te, tr in zip(env_term.reshape(-1), env_trunc.reshape(-1)):
        if len(done) % T == 0:
            steps = 0
        steps += 1
        tr = steps >= tmax if time_limit else tr
        trunc.append(tr)
        done.append(te or tr)
        steps = 0 if te or tr else steps
    done, trunc = np.array(done).reshape(epochs_rolled, T), np.array(trunc).reshape(epochs_rolled, T)
    assert done.sum() >= 10 and not done[:, -1].all(), 'no episode running at the epoch boundary'
    if time_limit:
        assert (env_trunc & ~trunc & ~env_term).any(), "no truncation of the env's own that TimeLimit discards"
        assert (env_term & trunc).any(), 'no termination in the step the time limit hits'
    else:
        assert (env_trunc & ~env_term).any() and env_term.any()
    lo, hi = xe.wide_box_bounds(A)
    np.savez(os.path.join(HERE, fname), N=N, T=T, O=O, A=A, seed=seed, tmax=tmax, time_limit=int(time_limit),
             theta=theta, epochs_rolled=epochs_rolled, eps=eps, act_lo=lo, act_hi=hi, env_term=env_term,
             env_trunc=env_trunc, norm_mean=nz.mean.numpy(), norm_std=nz.std.numpy(), norm_count=int(nz._count),
             win_ret=window['Metrics/EpRet'], win_cost=window['Metrics/EpCost'], win_len=window['Metrics/EpLen'],
             **{'slab_' + k: v for k, v in data.items()})


if __name__ == '__main__':
    torch.set_num_threads(1)
    gen(we.WRAPPED_ID, 'rollout_external_wrappers.npz')
    gen(we.AUTO_RESET_ID, 'rollout_external_autoreset.npz', seed=46, tmax=64)
    print('golden fixtures written to', HERE)
