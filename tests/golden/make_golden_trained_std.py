"""Generate the rollout fixtures at a trained policy std: the UNMODIFIED reference OnPolicyAdapter.rollout (PPOLag) with
the actor's log_std set to oracle.actor_critic.trained_log_std(A) before rolling out.

    python tests/golden/make_golden_trained_std.py

  rollout_ppolag_trained.npz    the synthetic env, one epoch at A = 3 and one at A = 9 (keys prefixed 'A3_' / 'A9_')
  rollout_external_trained.npz  the WideBox CMDP of tests/external_envs.py, two epochs at A = 3

At the reference's initial log_std = 0 every action has sigma = 1, so rollout_ppolag.npz and rollout_external.npz cannot
tell one action's sigma from another's.  The `_standard_normal` draws are recorded as in make_golden.py.  Like
make_golden.py it needs the reference sources (imported through oracle/ref_shim.py) and runs on the CPU; only its output
is committed.
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
from oracle import actor_critic as oac  # noqa: E402


def _set_trained_std(algo, A):
    with torch.no_grad():
        algo._actor_critic.actor.log_std.copy_(torch.as_tensor(oac.trained_log_std(A)))


def _roll(algo, N, T, A, epochs):
    """`epochs` rollouts of the reference with every standard-normal draw recorded; the slabs, the draws, the logger
    window and the observation normaliser."""
    import torch.distributions.normal as tdn

    drawn, orig = [], tdn._standard_normal

    def rec(shape, dtype, device):
        e = orig(shape, dtype, device)
        drawn.append(e.clone())
        return e

    tdn._standard_normal = rec
    try:
        for e in range(epochs):
            if e > 0:
                algo._buf.get()
            algo._env.rollout(steps_per_epoch=T, agent=algo._actor_critic, buffer=algo._buf, logger=algo._logger)
    finally:
        tdn._standard_normal = orig
    eps = np.stack([d.numpy() for d in drawn if tuple(d.shape) == (N, A)])
    assert eps.shape[0] == T * epochs, eps.shape
    fields = ('obs', 'act', 'reward', 'cost', 'value_r', 'value_c', 'logp', 'adv_r', 'adv_c', 'target_value_r',
              'target_value_c')
    data = {'slab_' + k: np.stack([b.data[k].numpy().copy() for b in algo._buf.buffers], 1) for k in fields}
    win = {k: np.array(list(algo._logger._data['Metrics/' + k]), np.float32) for k in ('EpRet', 'EpCost', 'EpLen')}
    norm = algo._env._env
    while not hasattr(norm, '_obs_normalizer'):
        norm = norm._env
    nz = norm._obs_normalizer
    return dict(eps=eps, epochs_rolled=epochs, theta=mg._flat_theta(algo._actor_critic),
                norm_mean=nz.mean.numpy(), norm_std=nz.std.numpy(), norm_count=int(nz._count),
                win_ret=win['EpRet'], win_cost=win['EpCost'], win_len=win['EpLen'], **data)


def gen_rollout_ppolag_trained(fname='rollout_ppolag_trained.npz', N=8, T=24, O=12, tmax=8, term_prob=0.05):
    out = {}
    for A, seed in ((3, 5), (9, 6)):
        algo = mg._build_algo('PPOLag', N, T, O, A, seed, tmax=tmax, term_prob=term_prob)
        _set_trained_std(algo, A)
        g = _roll(algo, N, T, A, 1)
        g['eps'] = g['eps'].reshape(T, N, A)
        out.update({f'A{A}_{k}': v for k, v in dict(g, N=N, T=T, O=O, A=A, seed=seed, tmax=tmax,
                                                      term_prob=term_prob).items()})
    np.savez(os.path.join(HERE, fname), **out)


def gen_rollout_external_trained(fname='rollout_external_trained.npz', seed=43, N=8, T=24, O=45, A=3, tmax=7,
                                 epochs=2):
    from omnisafe.algorithms import registry
    from omnisafe.utils.config import get_default_kwargs_yaml
    from omnisafe.utils.tools import recursive_check_config

    xe.register(CMDP, Box, env_register, support_envs())
    cfgs = get_default_kwargs_yaml('PPOLag', xe.WIDE_BOX_ID, 'on-policy')
    custom = {
        'seed': seed,
        'train_cfgs': {'vector_env_nums': N, 'total_steps': N * T * epochs, 'torch_threads': 1},
        'algo_cfgs': {'steps_per_epoch': N * T, 'batch_size': 32, 'update_iters': 2},
        'logger_cfgs': {'use_tensorboard': False, 'use_wandb': False, 'log_dir': '/tmp/osb_golden_runs', 'window_lens': 10},
    }
    recursive_check_config(custom, cfgs)
    cfgs.recurisve_update(custom)
    cfgs.recurisve_update({'env_cfgs': {'obs_dim': O, 'act_dim': A, 'max_episode_steps': tmax}})
    cfgs.recurisve_update({'exp_name': 'PPOLag-golden-external-trained', 'env_id': xe.WIDE_BOX_ID, 'algo': 'PPOLag'})
    cfgs.train_cfgs.recurisve_update({'epochs': epochs})
    algo = registry.get('PPOLag')(env_id=xe.WIDE_BOX_ID, cfgs=cfgs)
    _set_trained_std(algo, A)
    g = _roll(algo, N, T, A, epochs)
    lo, hi = xe.wide_box_bounds(A)
    np.savez(os.path.join(HERE, fname), N=N, T=T, O=O, A=A, seed=seed, tmax=tmax, act_lo=lo, act_hi=hi, **g)


if __name__ == '__main__':
    torch.set_num_threads(1)
    gen_rollout_ppolag_trained()
    gen_rollout_external_trained()
    print('golden fixtures written to', HERE)
