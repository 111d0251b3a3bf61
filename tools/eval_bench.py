"""Time `Evaluator.evaluate`: O = 60, A = 8, episodes of 64 steps (no terminations), bf16x3.

    python tools/eval_bench.py [--out DIR]
    python tools/eval_bench.py --registered [--graph] [--out DIR]

Default, the synthetic env: the time per evaluation step with one env (the reference's loop shape) and the episodes per
second with 4096 envs.  --registered: the same dynamics as a registered env stepped in PyTorch (TorchBox of
tools/external_env_bench.py), 4096 envs, evaluation env-steps/s and episodes/s; --graph uses its graph-safe variant and
times it eagerly (OSB_NO_GRAPH=1) and replayed from CUDA graphs, alternating, three calls each.  One JSON line, with the
card's name and power limit read in the same run.  Times are host wall-clock around whole `evaluate` calls (each ends in
a device synchronisation when it reads the results), after one warm-up call.
"""
from __future__ import annotations

import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def make_run(d: str, O: int = 60, A: int = 8, T: int = 64, env_id: str = 'SyntheticBox-v0') -> None:
    rng = np.random.default_rng(0)
    pi = {'log_std': torch.full((A,), -0.5), 'mean.0.weight': torch.as_tensor(rng.uniform(-0.3, 0.3, (64, O)), dtype=torch.float32),
          'mean.0.bias': torch.zeros(64), 'mean.2.weight': torch.as_tensor(rng.uniform(-0.2, 0.2, (64, 64)), dtype=torch.float32),
          'mean.2.bias': torch.zeros(64), 'mean.4.weight': torch.as_tensor(rng.uniform(-0.3, 0.3, (A, 64)), dtype=torch.float32),
          'mean.4.bias': torch.zeros(A)}
    norm = {'_mean': torch.zeros(O), '_sumsq': torch.full((O,), 999.0), '_std': torch.ones(O), '_var': torch.ones(O),
            '_count': torch.tensor(1000), '_clip': torch.full((O,), 5.0)}
    os.makedirs(os.path.join(d, 'torch_save'))
    cfg = {'algo': 'PPOLag', 'env_id': env_id, 'train_cfgs': {'matmul_precision': 'bf16x3'},
           'env_cfgs': {'obs_dim': O, 'act_dim': A, 'max_episode_steps': T}, 'algo_cfgs': {'obs_normalize': True}}
    with open(os.path.join(d, 'config.json'), 'w', encoding='utf-8') as fh:
        json.dump(cfg, fh)
    torch.save({'pi': pi, 'obs_normalizer': norm}, os.path.join(d, 'torch_save', 'epoch-0.pt'))


def timed(ev, **kw) -> float:
    with contextlib.redirect_stdout(io.StringIO()):
        ev.evaluate(**kw)                       # warm-up: module load, attributes, accumulator images
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ev.evaluate(**kw)
        torch.cuda.synchronize()
    return time.perf_counter() - t0


def gpu_name_power() -> str:
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return smi[0] if smi else 'unknown'


def registered(graph: bool) -> dict:
    """4096 envs of TorchBox (graph: TorchBoxGraph), 4 episodes each: evaluation env-steps/s and episodes/s."""
    from external_env_bench import ENV_ID, GRAPH_ENV_ID, register_torch_box

    from omnisafe_b200 import Evaluator

    register_torch_box()
    E, T, per_env = 4096, 64, 4
    nE = E * per_env
    res = {'envs': E, 'episode_steps': T, 'episodes': nE}
    with tempfile.TemporaryDirectory() as d:
        make_run(d, T=T, env_id=GRAPH_ENV_ID if graph else ENV_ID)
        ev = Evaluator()
        ev.load_saved(d, 'epoch-0.pt')
        modes = ('eager', 'graph') if graph else ('eager',)
        times = {m: [] for m in modes}
        for _ in range(3 if graph else 1):
            for m in modes:
                if m == 'eager':
                    os.environ['OSB_NO_GRAPH'] = '1'
                else:
                    os.environ.pop('OSB_NO_GRAPH', None)
                times[m].append(timed(ev, num_episodes=nE, num_envs=E))
        os.environ.pop('OSB_NO_GRAPH', None)
    for m, ts in times.items():
        t = float(np.median(ts))
        res[f'{m}_s'] = ts
        res[f'{m}_env_steps_per_s'] = E * per_env * T / t
        res[f'{m}_episodes_per_s'] = nE / t
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--registered', action='store_true', help='the synthetic dynamics as a registered PyTorch env')
    ap.add_argument('--graph', action='store_true', help='with --registered: the graph-safe env, eager vs graph')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('tools/eval_bench.py measures on a CUDA device; none is visible')
    if args.graph and not args.registered:
        raise SystemExit('--graph needs --registered')
    if args.registered:
        res = {'mode': 'registered-graph' if args.graph else 'registered', **registered(args.graph),
               'gpu': gpu_name_power(), 'torch_device': torch.cuda.get_device_name(0)}
        emit(res, args.out)
        return
    from omnisafe_b200 import Evaluator

    T = 64
    with tempfile.TemporaryDirectory() as d:
        make_run(d, T=T)
        ev = Evaluator()
        ev.load_saved(d, 'epoch-0.pt')
        n1 = 10
        t1 = timed(ev, num_episodes=n1, num_envs=1)
        nE = 4096 * 4
        tE = timed(ev, num_episodes=nE, num_envs=4096)
    res = {'e1_step_us': t1 / (n1 * T) * 1e6, 'e4096_episodes_per_s': nE / tE, 'e4096_steps': 4 * T,
           'gpu': gpu_name_power(), 'torch_device': torch.cuda.get_device_name(0)}
    emit(res, args.out)


def emit(res: dict, out: str | None) -> None:
    line = json.dumps(res)
    print(line)
    if out:
        os.makedirs(out, exist_ok=True)
        name = 'eval_bench_%s.json' % res['mode'] if 'mode' in res else 'eval_bench.json'
        with open(os.path.join(out, name), 'w', encoding='utf-8') as fh:
            fh.write(line + '\n')


if __name__ == '__main__':
    main()
