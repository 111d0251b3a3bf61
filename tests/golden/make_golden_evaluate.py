"""Generate tests/golden/evaluate_*.npz: the UNMODIFIED reference Evaluator (omnisafe/evaluator.py, `load_saved` +
`evaluate`) on checkpoints in the reference format ('pi', 'obs_normalizer') of the synthetic env (RefSyntheticBox of
make_golden.py):

- ppolag: terminations and truncations;
- pposaute: the safety state z crosses 0;
- ppoearly: PPOEarlyTerminated with cost_criteria 0.99, episodes cut by the cost rule;
- widebox: PPOLag on the WideBox registered env of tests/external_envs.py (asymmetric action box, |obs| up to 1e3,
  terminations and truncations), through tests/eval_envs.py.

    python tests/golden/make_golden_evaluate.py

Like make_golden.py it needs the reference sources (imported through oracle/ref_shim.py) and runs on the CPU; only its
outputs are committed.  Each fixture holds the run's config.json text, the checkpoint's tensors, the per-episode returns,
costs and lengths and the normaliser after the evaluation.
"""
from __future__ import annotations

import contextlib
import io
import json
import os
import re
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))          # tests/ (external_envs, eval_envs)
import make_golden  # noqa: E402,F401  (installs the reference shim, registers RefSyntheticBox)

import eval_envs  # noqa: E402
from omnisafe.envs.core import CMDP, env_register, support_envs  # noqa: E402

from omnisafe.common.normalizer import Normalizer  # noqa: E402
from omnisafe.evaluator import Evaluator  # noqa: E402
from omnisafe.models.actor.actor_builder import ActorBuilder  # noqa: E402
from gymnasium.spaces import Box  # noqa: E402  (shim)

CASES = {
    # name: (algo, env_cfgs, algo_cfgs, num_episodes, cost_criteria)
    'ppolag': ('PPOLag', dict(obs_dim=12, act_dim=3, max_episode_steps=8, term_prob=0.15, cost_threshold=0.0),
               dict(obs_normalize=True), 6, 1.0),
    'pposaute': ('PPOSaute', dict(obs_dim=10, act_dim=4, max_episode_steps=9, term_prob=0.05, cost_threshold=-0.05),
                 dict(obs_normalize=True, safety_budget=2.0, saute_gamma=0.999, max_ep_len=9, unsafe_reward=-1.0), 4, 1.0),
    'ppoearly': ('PPOEarlyTerminated', dict(obs_dim=12, act_dim=3, max_episode_steps=10, term_prob=0.0,
                                            cost_threshold=-0.1),
                 dict(obs_normalize=True, cost_limit=3.0), 5, 0.99),
    'widebox': ('PPOLag', dict(obs_dim=45, act_dim=3, max_episode_steps=7), dict(obs_normalize=True), 6, 1.0),
}


def _checkpoint(name, O, A, saute, seed):
    gen = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    obs_space = Box(-10.0, 10.0, (O + int(saute),))
    scale = (10.0 ** (torch.arange(O) % 4)).float() if name == 'widebox' else torch.ones(O)
    actor = ActorBuilder(obs_space=obs_space, act_space=Box(-1.0, 1.0, (A,)), hidden_sizes=[64, 64],
                         activation='tanh', weight_initialization_mode='kaiming_uniform').build_actor('gaussian_learning')
    with torch.no_grad():   # a trained-looking policy: large enough weights that the actions move the state
        for p in actor.parameters():
            p.mul_(3.0)
    norm = Normalizer((O,), clip=5)
    for k in range(4):
        norm.normalize((torch.rand(16, O, generator=gen) * 2 - 1) * (0.5 + k) * scale)
    return {'pi': actor.state_dict(), 'obs_normalizer': norm.state_dict()}


def gen(name, seed):
    algo, env_cfgs, algo_cfgs, num_episodes, crit = CASES[name]
    O, A = env_cfgs['obs_dim'], env_cfgs['act_dim']
    saute = 'Saute' in algo or 'Simmer' in algo
    cfg = {
        'algo': algo, 'env_id': eval_envs.WIDE_BOX_EVAL_ID if name == 'widebox' else 'SyntheticBox-v0', 'seed': seed, 'env_cfgs': env_cfgs, 'algo_cfgs': algo_cfgs,
        'model_cfgs': {'actor_type': 'gaussian_learning', 'weight_initialization_mode': 'kaiming_uniform',
                       'actor': {'hidden_sizes': [64, 64], 'activation': 'tanh'}},
    }
    ckpt = _checkpoint(name, O, A, saute, seed)
    with tempfile.TemporaryDirectory() as d:
        os.makedirs(os.path.join(d, 'torch_save'))
        with open(os.path.join(d, 'config.json'), 'w', encoding='utf-8') as fh:
            json.dump(cfg, fh)
        torch.save(ckpt, os.path.join(d, 'torch_save', 'epoch-0.pt'))
        ev = Evaluator()
        ev.load_saved(save_dir=d, model_name='epoch-0.pt')
        out = io.StringIO()
        with contextlib.redirect_stdout(out):
            rets, costs = ev.evaluate(num_episodes=num_episodes, cost_criteria=crit)
        norm = ev._env
        while not hasattr(norm, '_obs_normalizer'):
            norm = norm._env
        nz = norm._obs_normalizer
    lens = [float(x) for x in re.findall(r'Episode length: ([0-9.]+)', out.getvalue())]
    assert len(lens) == num_episodes
    # the fixture must exercise what it is for
    if name == 'widebox':
        assert float(nz.mean.abs().max()) > 10.0 and min(lens) < env_cfgs['max_episode_steps'], lens
    if name == 'ppolag':
        assert min(lens) < env_cfgs['max_episode_steps'] and max(lens) == env_cfgs['max_episode_steps'], lens
    if name == 'ppoearly':
        assert min(lens) < env_cfgs['max_episode_steps'], lens
    if name == 'pposaute':
        b = algo_cfgs['safety_budget'] * (1 - 0.999 ** 9) / (1 - 0.999) / 9
        assert max(costs) / b > 1.0, 'z never crossed 0'
    np.savez(os.path.join(HERE, f'evaluate_{name}.npz'), config=json.dumps(cfg), num_episodes=num_episodes,
             cost_criteria=crit, ret=np.array(rets), cost=np.array(costs), length=np.array(lens),
             norm_mean=nz.mean.numpy(), norm_std=nz.std.numpy(), norm_sumsq=nz._sumsq.numpy(), norm_count=int(nz._count),
             **{'pi_' + k: v.numpy() for k, v in ckpt['pi'].items()},
             **{'norm0' + k: v.numpy() for k, v in ckpt['obs_normalizer'].items()})
    print(name, 'lengths', lens, 'returns', rets, 'costs', costs)


if __name__ == '__main__':
    torch.set_num_threads(1)
    eval_envs.register(CMDP, Box, env_register, support_envs())
    for i, name in enumerate(CASES):
        gen(name, seed=71 + i)
    print('golden fixtures written to', HERE)
