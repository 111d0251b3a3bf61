"""Generate tests/golden/rollout_external_early.npz: two epochs of the UNMODIFIED reference EarlyTerminatedAdapter.rollout
(PPOEarlyTerminated) on the WideBox test CMDP of tests/external_envs.py with a single env, as upstream supports it, and a
low cost limit, so that the cost rule cuts episodes often: on steps where the env itself terminated or truncated, and
with the accumulator carried across ordinary episode ends.

    python tests/golden/make_golden_external_early.py

Like make_golden.py it needs the reference sources (imported through oracle/ref_shim.py) and runs on the CPU; only its
output is committed.  Besides the slabs it stores the env's own terminated / truncated flags of every step (env_term /
env_trunc) and the step's accumulator before the rule (acc), which the tests use to check the fixture's coverage.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))          # tests/ (external_envs)
import make_golden as mg  # noqa: E402  (installs the reference shim)

import external_envs as xe  # noqa: E402
from gymnasium.spaces import Box  # noqa: E402  (shim)
from omnisafe.envs.core import CMDP, env_register, support_envs  # noqa: E402


def gen_rollout_external_early(fname='rollout_external_early.npz', seed=44, T=64, O=45, A=3, tmax=5, cost_limit=2.5,
                               epochs_rolled=2):
    from omnisafe.algorithms import registry
    from omnisafe.utils.config import get_default_kwargs_yaml
    from omnisafe.utils.tools import recursive_check_config
    import torch.distributions.normal as tdn

    N, algo_name = 1, 'PPOEarlyTerminated'
    xe.register(CMDP, Box, env_register, support_envs())
    cfgs = get_default_kwargs_yaml(algo_name, xe.WIDE_BOX_ID, 'on-policy')
    custom = {
        'seed': seed,
        'train_cfgs': {'vector_env_nums': N, 'total_steps': N * T * 2, 'torch_threads': 1},
        'algo_cfgs': {'steps_per_epoch': N * T, 'batch_size': 32, 'update_iters': 2, 'cost_limit': cost_limit},
        'logger_cfgs': {'use_tensorboard': False, 'use_wandb': False, 'log_dir': '/tmp/osb_golden_runs', 'window_lens': 10},
    }
    recursive_check_config(custom, cfgs)
    cfgs.recurisve_update(custom)
    cfgs.recurisve_update({'env_cfgs': {'obs_dim': O, 'act_dim': A, 'max_episode_steps': tmax}})
    cfgs.recurisve_update({'exp_name': f'{algo_name}-golden-external', 'env_id': xe.WIDE_BOX_ID, 'algo': algo_name})
    cfgs.train_cfgs.recurisve_update({'epochs': 2})
    algo = registry.get(algo_name)(env_id=xe.WIDE_BOX_ID, cfgs=cfgs)
    assert not cfgs.algo_cfgs.reward_normalize
    theta = mg._flat_theta(algo._actor_critic)
    adapter = algo._env
    # the env's own flags and the accumulator before each step's rule, recorded around the wrapper chain's step
    env_term, env_trunc, env_cost, acc = [], [], [], []
    inner_step = adapter._env.step

    def rec_step(action):
        acc.append(float(adapter._cost_logger.reshape(-1)[0]))
        out = inner_step(action)
        env_term.append(bool(out[3].reshape(-1)[0]))
        env_trunc.append(bool(out[4].reshape(-1)[0]))
        env_cost.append(float(out[2].reshape(-1)[0]))
        return out

    adapter._env.step = rec_step
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

    # the fixture must exercise what it is for (over both epochs; the slabs hold the last one)
    env_term = np.array(env_term).reshape(epochs_rolled, T)
    env_trunc = np.array(env_trunc).reshape(epochs_rolled, T)
    acc = np.array(acc, np.float32).reshape(epochs_rolled, T)
    after = (acc + np.array(env_cost, np.float32).reshape(epochs_rolled, T)).astype(np.float32)
    trig = after > np.float32(cost_limit)
    assert np.array_equal(after[-1] - acc[-1], data['cost'][:, 0])
    assert np.array_equal(data['reward'][:, 0][trig[-1]], np.zeros(int(trig[-1].sum()), np.float32))
    assert trig.sum() >= 10, int(trig.sum())
    assert (trig & env_trunc).any(), 'no trigger on a step the env truncated'
    assert (trig & env_term).any(), 'no trigger on a step the env terminated'
    carried = (env_term | env_trunc) & ~trig & (after > 0)
    assert carried.any(), 'no accumulator carried across an ordinary episode end'
    lo, hi = xe.wide_box_bounds(A)
    np.savez(os.path.join(HERE, fname), N=N, T=T, O=O, A=A, seed=seed, tmax=tmax, cost_limit=np.float32(cost_limit),
             theta=theta, epochs_rolled=epochs_rolled, eps=eps, act_lo=lo, act_hi=hi, env_term=env_term,
             env_trunc=env_trunc, acc=acc, norm_mean=nz.mean.numpy(), norm_std=nz.std.numpy(),
             norm_count=int(nz._count), win_ret=window['Metrics/EpRet'], win_cost=window['Metrics/EpCost'],
             win_len=window['Metrics/EpLen'], **{'slab_' + k: v for k, v in data.items()})


if __name__ == '__main__':
    torch.set_num_threads(1)
    gen_rollout_external_early()
    print('golden fixture written to', HERE)
