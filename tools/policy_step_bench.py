"""Throughput of the policy-step kernel (ConstraintActorCritic.step: actor sample + log-prob + both critics in one
osb_policy_step launch) per precision, observation width and batch size, launched eagerly and replayed from a CUDA
graph.  Eager and graph runs alternate `--repeats` times; each run times `--iters` back-to-back launches (or replays)
with CUDA events and reports microseconds per launch and rows per second.  Prints one JSON line per configuration with
the per-run values, so the spread is visible.

    python tools/policy_step_bench.py [--iters 200] [--repeats 3] [--precisions 0 1 2] [--obs 60 376]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from types import SimpleNamespace as NS

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _model(dev, O, A, precision):
    from omnisafe_b200.models import ConstraintActorCritic

    net = NS(hidden_sizes=[64, 64], activation='tanh', lr=3e-4)
    mc = NS(actor=net, critic=net, actor_type='gaussian_learning', linear_lr_decay=True,
            weight_initialization_mode='kaiming_uniform')
    m = ConstraintActorCritic(O, A, mc, epochs=1, device=dev, generator=torch.Generator().manual_seed(0))
    m.precision = precision
    return m


def _time(fn, iters: int) -> float:
    """Microseconds per call of fn over `iters` back-to-back calls on the current stream."""
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) * 1e3 / iters


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=200)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--precisions', type=int, nargs='+', default=[0, 1, 2])
    ap.add_argument('--obs', type=int, nargs='+', default=[60, 376])
    ap.add_argument('--batches', type=int, nargs='+', default=[1, 4096, 65536])
    ap.add_argument('--act', type=int, default=8)
    args = ap.parse_args()
    from omnisafe_b200._lib import lib

    dev = torch.device('cuda:0')
    A = args.act
    lib().osb_policy_prepare()
    for precision in args.precisions:
        for O in args.obs:
            m = _model(dev, O, A, precision)
            for B in args.batches:
                obs = torch.randn(B, O, device=dev).clamp_(-5, 5)
                eps = torch.randn(B, A, device=dev)

                def launch():
                    return m._launch(obs, 7, eps=eps, act=True, logp=True)

                s = torch.cuda.Stream()
                s.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(s):
                    for _ in range(3):
                        launch()
                torch.cuda.current_stream().wait_stream(s)
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    launch()
                _time(launch, 10)
                _time(g.replay, 10)
                eager, graph = [], []
                for _ in range(args.repeats):
                    eager.append(_time(launch, args.iters))
                    graph.append(_time(g.replay, args.iters))
                row = {'precision': ['fp32', 'tf32', 'bf16x3'][precision], 'O': O, 'A': A, 'B': B,
                       'eager_us': [round(x, 2) for x in eager], 'graph_us': [round(x, 2) for x in graph],
                       'eager_rows_per_s': round(B / (min(eager) * 1e-6)), 'graph_rows_per_s': round(B / (min(graph) * 1e-6)),
                       'device': torch.cuda.get_device_name(dev)}
                print(json.dumps(row), flush=True)
                del g


if __name__ == '__main__':
    main()
