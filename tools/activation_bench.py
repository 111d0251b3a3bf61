"""Cost of the hidden activations on the bench workload (PPOLag, SyntheticBox-v0 obs60/act8, 4096 envs x T=128).

    python tools/activation_bench.py [--parent DIR] [--rounds R] [--steps K] [--warmup W] [--bench-args ARGS]
                                     [--epochs E] [--out FILE]

1. With --parent (a checkout of another commit, built): `bench.py --gpus 1 --steps K --warmup W` of that checkout and
   of this one, alternated R times in one process tree, so that both see the same card and the same neighbours.  The
   tanh epoch is the benchmark's own workload.
2. Device time of one training epoch (rollout + GAE + update, CUDA events around `train_epoch`) per activation pair
   (actor, critics), in bf16x3 (the benchmark's arithmetic) and tf32, E epochs after 3 warm-up epochs.
The card's name and power limit are read in the same run and printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAIRS = [('tanh', 'tanh'), ('identity', 'identity'), ('relu', 'relu'), ('sigmoid', 'sigmoid'), ('softplus', 'softplus'),
         ('softplus', 'relu')]


def card() -> str:
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True, check=True)
    return q.stdout.strip().splitlines()[0]


def bench_line(tree: str, steps: int, warmup: int, extra: list[str]) -> dict:
    out = subprocess.run([sys.executable, 'bench.py', '--gpus', '1', '--steps', str(steps), '--warmup', str(warmup), *extra],
                         cwd=tree, capture_output=True, text=True, check=True).stdout
    return json.loads([ln for ln in out.splitlines() if ln.startswith('{')][-1])


def epoch_times(epochs: int) -> list[dict]:
    sys.path.insert(0, ROOT)
    import torch

    import bench
    import omnisafe_b200

    rows = []
    for prec in ('bf16x3', 'tf32'):
        for aa, ca in PAIRS:
            cfg = bench._custom_cfgs(1, tempfile.mkdtemp(), epochs + 4, precision=prec)
            cfg['model_cfgs'] = {'actor': {'activation': aa}, 'critic': {'activation': ca}}
            algo = omnisafe_b200.Agent('PPOLag', 'SyntheticBox-v0', custom_cfgs=cfg).agent
            for _ in range(3):
                algo.train_epoch()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(epochs):
                algo.train_epoch()
            e1.record()
            torch.cuda.synchronize()
            rows.append({'precision': prec, 'actor': aa, 'critic': ca, 'epoch_ms': e0.elapsed_time(e1) / epochs})
            print(f'{prec:7s} actor {aa:8s} critics {ca:8s}: {rows[-1]["epoch_ms"]:8.3f} ms / epoch', flush=True)
            del algo
    return rows


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument('--parent', help='a built checkout of the commit to compare bench.py against')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--epochs', type=int, default=10)
    ap.add_argument('--bench-args', default='', help='more bench.py arguments, e.g. "--no-cpu-baseline"')
    ap.add_argument('--out', help='write the results as JSON to this file')
    args = ap.parse_args()
    res = {'card': card()}
    print('card (name, power limit, max SM clock):', res['card'], flush=True)
    if args.parent:
        res['bench'] = {'parent': [], 'this': []}
        for r in range(args.rounds):
            for name, tree in (('parent', args.parent), ('this', ROOT)):
                line = bench_line(tree, args.steps, args.warmup, args.bench_args.split())
                res['bench'][name].append(line['value'])
                print(f'round {r} {name:6s}: {line["value"]:.4g} {line["unit"]}', flush=True)
    res['epochs'] = epoch_times(args.epochs)
    if args.out:
        with open(args.out, 'w', encoding='utf-8') as fh:
            json.dump(res, fh, indent=1)


if __name__ == '__main__':
    main()
