"""Lagrange multiplier with its Adam state on the device.

Mirrors omnisafe/common/lagrange.py:L25-136 (constructor arguments, `lagrangian_multiplier`,
`update_lagrange_multiplier`).  The step itself is `osb_lagrange_update` (csrc/optim.cu): Adam on a
scalar with gradient -(Jc - cost_limit), then projection onto [0, upper_bound].
"""
from __future__ import annotations

import torch

from omnisafe_b200._lib import current_stream, lib, ptr
from omnisafe_b200.utils.train_state import restore, snapshot


class Lagrange:
    def __init__(self, cost_limit: float, lagrangian_multiplier_init: float, lambda_lr: float,
                 lambda_optimizer: str = 'Adam', lagrangian_upper_bound: float | None = None,
                 device='cuda') -> None:
        assert lambda_optimizer == 'Adam', (
            f'Optimizer={lambda_optimizer}: only Adam is implemented on the device path')
        self.cost_limit = float(cost_limit)
        self.lambda_lr = float(lambda_lr)
        self.lagrangian_upper_bound = lagrangian_upper_bound
        init_value = max(float(lagrangian_multiplier_init), 0.0)
        # state = {lambda, adam m, adam v, adam t}
        self.state = torch.tensor([init_value, 0.0, 0.0, 0.0], dtype=torch.float32, device=device)
        self.nan_flag = torch.zeros(1, dtype=torch.int32, device=device)
        self._jc_sums = None

    @property
    def lagrangian_multiplier(self) -> torch.Tensor:
        return self.state[0]

    def train_state(self) -> dict:
        """lambda and its Adam moments / step count."""
        return {'state': snapshot(self.state)[0]}

    def load_train_state(self, state: dict) -> None:
        restore(self.state, state['state'], 'Lagrange state')

    def update_lagrange_multiplier(self, Jc) -> None:   # noqa: N803  (the reference's argument name)
        """Reference signature `update_lagrange_multiplier(Jc: float)` (common/lagrange.py:L114-136): Adam step on
        lambda with gradient -(Jc - cost_limit), then projection onto [0, upper_bound].

        Overload (the training loop's fast path, no host synchronisation): a device fp64 tensor
        {sum EpRet, sum EpCost, sum EpLen, count} of the (already all-reduced) episode window, Jc = sum EpCost / count."""
        if not isinstance(Jc, torch.Tensor):
            if self._jc_sums is None:
                self._jc_sums = torch.zeros(4, dtype=torch.float64, device=self.state.device)
            self._jc_sums[1] = float(Jc)       # a NaN Jc raises the same assertion as the reference (ppo_lag.py:L74) via nan_flag
            self._jc_sums[3] = 1.0
            Jc = self._jc_sums
        assert Jc.dtype == torch.float64 and Jc.numel() >= 4, 'device fast path: fp64 {sum EpRet, sum EpCost, sum EpLen, count}'
        ub = -1.0 if self.lagrangian_upper_bound is None else float(self.lagrangian_upper_bound)
        lib().osb_lagrange_update(ptr(Jc), self.cost_limit, self.lambda_lr, ub,
                                  ptr(self.state), ptr(self.nan_flag), current_stream())
