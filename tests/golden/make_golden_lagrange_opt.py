"""Golden multiplier trajectories of the UNMODIFIED reference `Lagrange` (common/lagrange.py, through
oracle/ref_shim.py like make_golden.py) for every `lambda_optimizer` torch steps on a 0-d parameter.

    python tests/golden/make_golden_lagrange_opt.py

Writes lagrange_opt.npz: a recorded Jc sequence that crosses the cost limit many times, sits on it once (zero
gradient), drives lambda into the clamp at 0 and flips the gradient's sign step to step (Rprop's backtracking),
and for each optimiser and each of three settings {lambda_lr 0.035; lambda_lr 0.2; lambda_lr 0.2 with
lagrangian_upper_bound 0.5}:
- lam_<name>_<i>: lambda after every step, as the reference computes it;
- ieee_<name>_<i>: the same with Tensor.sqrt / sqrt_ / rsqrt_ correctly rounded (tests/lagrange_replay.py), the
  trajectory the device kernels reproduce bit for bit.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_shim  # noqa: E402

ref_shim.install()
from omnisafe.common.lagrange import Lagrange  # noqa: E402

from lagrange_replay import NAMES, ieee_sqrt  # noqa: E402

COST_LIMIT, LAM_INIT = 25.0, 0.001
SETTINGS = [(0.035, None), (0.2, None), (0.2, 0.5)]


def jc_sequence() -> np.ndarray:
    rng = np.random.default_rng(11)
    above = COST_LIMIT + rng.uniform(1.0, 40.0, 25)                      # lambda climbs
    below = COST_LIMIT - rng.uniform(5.0, 25.0, 20)                      # lambda falls into the clamp at 0
    flips = COST_LIMIT + rng.uniform(0.5, 8.0, 20) * np.tile([1.0, -1.0], 10)   # sign flips every step
    noisy = COST_LIMIT + 15.0 * rng.standard_normal(24)
    return np.concatenate([above, below, [COST_LIMIT], flips, noisy, above[:10]])


def run(name: str, jcs, lr: float, ub) -> np.ndarray:
    lag = Lagrange(COST_LIMIT, LAM_INIT, lr, name, ub)
    out = []
    for jc in jcs:
        lag.update_lagrange_multiplier(float(jc))
        out.append(lag.lagrangian_multiplier.item())
    return np.asarray(out, np.float32)


def main():
    torch.set_num_threads(1)
    jcs = jc_sequence()
    out = {'jc': jcs, 'cost_limit': COST_LIMIT, 'lam_init': LAM_INIT,
           'lr': np.asarray([s[0] for s in SETTINGS]), 'upper_bound': np.asarray([-1.0 if s[1] is None else s[1]
                                                                                   for s in SETTINGS])}
    for name in NAMES:
        for i, (lr, ub) in enumerate(SETTINGS):
            out[f'lam_{name}_{i}'] = run(name, jcs, lr, ub)
            with ieee_sqrt():
                out[f'ieee_{name}_{i}'] = run(name, jcs, lr, ub)
            ndiff = int((out[f'lam_{name}_{i}'] != out[f'ieee_{name}_{i}']).sum())
            print(f'{name:10s} lr={lr} ub={ub}: lambda {out[f"lam_{name}_{i}"][-1]:.6g}, '
                  f'{int((out[f"lam_{name}_{i}"] == 0).sum())} steps at 0, {ndiff} steps differ with IEEE sqrt')
    np.savez(os.path.join(HERE, 'lagrange_opt.npz'), **out)


if __name__ == '__main__':
    main()
