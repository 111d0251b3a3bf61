"""Helpers for the Lagrange-optimiser tests: upstream's multiplier loop on the CPU through torch.optim.

torch's CPU `sqrt` on fp32 is not correctly rounded (about 1 value in 150 is one ulp off), while the device
kernels take the IEEE square root.  `ieee_sqrt()` swaps Tensor.sqrt / sqrt_ / rsqrt_ for correctly rounded
versions while a reference runs, so the reference's every other fp32 rounding can be compared bit for bit.
"""
from __future__ import annotations

import contextlib

import numpy as np
import torch

NAMES = ('SGD', 'Adam', 'AdamW', 'Adamax', 'NAdam', 'RAdam', 'RMSprop', 'Rprop', 'Adagrad', 'Adadelta', 'ASGD',
         'Adafactor')


def _sqrt64(t: torch.Tensor) -> torch.Tensor:
    # the fp64 square root rounded to fp32 is the correctly rounded fp32 square root
    return torch.from_numpy(np.asarray(np.sqrt(t.detach().numpy().astype(np.float64)), np.float32)).reshape(t.shape)


@contextlib.contextmanager
def ieee_sqrt():
    saved = torch.Tensor.sqrt, torch.Tensor.sqrt_, torch.Tensor.rsqrt_

    def sqrt(t):
        return _sqrt64(t) if t.dtype == torch.float32 else saved[0](t)

    def sqrt_(t):
        return t.copy_(_sqrt64(t)) if t.dtype == torch.float32 else saved[1](t)

    def rsqrt_(t):
        return t.copy_(torch.ones_like(t) / _sqrt64(t)) if t.dtype == torch.float32 else saved[2](t)

    torch.Tensor.sqrt, torch.Tensor.sqrt_, torch.Tensor.rsqrt_ = sqrt, sqrt_, rsqrt_
    try:
        yield
    finally:
        torch.Tensor.sqrt, torch.Tensor.sqrt_, torch.Tensor.rsqrt_ = saved


def replay(name: str, jcs, cost_limit: float, lam_init: float, lr: float, upper_bound=None) -> np.ndarray:
    """Upstream's Lagrange (common/lagrange.py:L67-136): torch.optim.<name>([lambda], lr=lr); per Jc zero_grad,
    backward of -lambda * (Jc - cost_limit), step, clamp to [0, upper_bound].  lambda after every step (fp32)."""
    lam = torch.nn.Parameter(torch.as_tensor(max(lam_init, 0.0)))
    opt = getattr(torch.optim, name)([lam], lr=lr)
    out = []
    with ieee_sqrt():
        for jc in jcs:
            opt.zero_grad()
            (-lam * (float(jc) - cost_limit)).backward()
            opt.step()
            lam.data.clamp_(0.0, upper_bound)
            out.append(lam.item())
    return np.asarray(out, np.float32)
