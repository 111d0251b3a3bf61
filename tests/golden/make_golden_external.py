"""Generate tests/golden/rollout_external.npz: two epochs of the UNMODIFIED reference OnPolicyAdapter.rollout (PPOLag)
on the WideBox test CMDP of tests/external_envs.py -- asymmetric per-dimension action box, observations up to ~1e3,
terminations and truncations in the same step, obs dim 45.

    python tests/golden/make_golden_external.py

Like make_golden.py it needs the reference sources (imported through oracle/ref_shim.py) and runs on the CPU; only its
output is committed.
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


def gen_rollout_external(fname='rollout_external.npz', seed=41, N=8, T=24, O=45, A=3, tmax=7, epochs_rolled=2):
    from omnisafe.algorithms import registry
    from omnisafe.utils.config import get_default_kwargs_yaml
    from omnisafe.utils.tools import recursive_check_config
    import torch.distributions.normal as tdn

    xe.register(CMDP, Box, env_register, support_envs())
    cfgs = get_default_kwargs_yaml('PPOLag', xe.WIDE_BOX_ID, 'on-policy')
    custom = {
        'seed': seed,
        'train_cfgs': {'vector_env_nums': N, 'total_steps': N * T * 2, 'torch_threads': 1},
        'algo_cfgs': {'steps_per_epoch': N * T, 'batch_size': 32, 'update_iters': 2},
        'logger_cfgs': {'use_tensorboard': False, 'use_wandb': False, 'log_dir': '/tmp/osb_golden_runs', 'window_lens': 10},
    }
    recursive_check_config(custom, cfgs)
    cfgs.recurisve_update(custom)
    cfgs.recurisve_update({'env_cfgs': {'obs_dim': O, 'act_dim': A, 'max_episode_steps': tmax}})
    cfgs.recurisve_update({'exp_name': 'PPOLag-golden-external', 'env_id': xe.WIDE_BOX_ID, 'algo': 'PPOLag'})
    cfgs.train_cfgs.recurisve_update({'epochs': 2})
    algo = registry.get('PPOLag')(env_id=xe.WIDE_BOX_ID, cfgs=cfgs)
    theta = mg._flat_theta(algo._actor_critic)
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
            algo._env.rollout(steps_per_epoch=T, agent=algo._actor_critic, buffer=algo._buf, logger=algo._logger)
    finally:
        tdn._standard_normal = orig
    eps = np.stack([d.numpy() for d in drawn if tuple(d.shape) == (N, A)])
    assert eps.shape[0] == T * epochs_rolled, eps.shape
    fields = ('obs', 'act', 'reward', 'cost', 'value_r', 'value_c', 'logp', 'adv_r', 'adv_c', 'target_value_r',
              'target_value_c')
    data = {k: np.stack([b.data[k].numpy().copy() for b in algo._buf.buffers], 1) for k in fields}
    window = {k: np.array(list(algo._logger._data[k]), np.float32) for k in ('Metrics/EpRet', 'Metrics/EpCost', 'Metrics/EpLen')}
    norm = algo._env._env
    while not hasattr(norm, '_obs_normalizer'):
        norm = norm._env
    nz = norm._obs_normalizer
    # the fixture must exercise what it is for
    core = xe.WideBoxCore(N, O, A, tmax, seed=0, device='cpu')
    assert np.abs(data['obs']).max() > 0 and float(nz.mean.abs().max()) > 10.0
    lo, hi = xe.wide_box_bounds(A)
    assert not np.allclose(lo, -hi)
    both = False
    core.reset()
    for _ in range(T * epochs_rolled):
        _, _, _, term, trunc, _, _ = core.step(torch.zeros(N, A))
        both |= bool((term & trunc).any())
    assert both, 'no step with a termination and a truncation at once'
    np.savez(os.path.join(HERE, fname), N=N, T=T, O=O, A=A, seed=seed, tmax=tmax, theta=theta,
             epochs_rolled=epochs_rolled, eps=eps, act_lo=lo, act_hi=hi,
             norm_mean=nz.mean.numpy(), norm_std=nz.std.numpy(), norm_count=int(nz._count),
             win_ret=window['Metrics/EpRet'], win_cost=window['Metrics/EpCost'], win_len=window['Metrics/EpLen'],
             **{'slab_' + k: v for k, v in data.items()})


if __name__ == '__main__':
    torch.set_num_threads(1)
    gen_rollout_external()
    print('golden fixture written to', HERE)
