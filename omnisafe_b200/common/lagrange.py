"""Lagrange multiplier with its optimiser state on the device.

Mirrors omnisafe/common/lagrange.py:L25-136 (constructor arguments, `lagrangian_multiplier`,
`update_lagrange_multiplier`).  The step is `torch.optim.<lambda_optimizer>(lr=lambda_lr)` on a scalar with
gradient -(Jc - cost_limit), then projection onto [0, upper_bound]: Adam is `osb_lagrange_update`, every
other optimiser torch can step on a 0-d parameter is `osb_lagrange_update_opt` (csrc/optim.cu).
"""
from __future__ import annotations

import torch

from omnisafe_b200._lib import current_stream, lib, ptr
from omnisafe_b200.utils.train_state import restore, snapshot

# kind numbers of osb_lagrange_update_opt (include/omnisafe_b200.h, OSB_LAMBDA_*)
OPT_KINDS = {'SGD': 0, 'AdamW': 1, 'Adamax': 2, 'NAdam': 3, 'RAdam': 4, 'RMSprop': 5, 'Rprop': 6,
             'Adagrad': 7, 'Adadelta': 8, 'ASGD': 9, 'Adafactor': 10}
OPT_STATE = 8   # OSB_LAMBDA_STATE
# torch.optim names that fail on the reference's multiplier as well, and why
REFUSED = {'LBFGS': 'its step needs a closure that re-evaluates the loss',
           'SparseAdam': 'it needs sparse gradients',
           'Muon': 'it only steps 2-D parameters'}


class Lagrange:
    def __init__(self, cost_limit: float, lagrangian_multiplier_init: float, lambda_lr: float,
                 lambda_optimizer: str = 'Adam', lagrangian_upper_bound: float | None = None,
                 device='cuda') -> None:
        assert hasattr(torch.optim, lambda_optimizer), f'Optimizer={lambda_optimizer} not found in torch.'
        if lambda_optimizer in REFUSED:
            raise ValueError(f'lambda_optimizer={lambda_optimizer!r} cannot step the Lagrange multiplier: '
                             f'{REFUSED[lambda_optimizer]}')
        if lambda_optimizer != 'Adam' and lambda_optimizer not in OPT_KINDS:
            raise ValueError(f'lambda_optimizer={lambda_optimizer!r} is not a torch.optim optimiser the '
                             f'multiplier can use; supported: Adam, {", ".join(OPT_KINDS)}')
        self.lambda_optimizer = lambda_optimizer
        self.cost_limit = float(cost_limit)
        self.lambda_lr = float(lambda_lr)
        self.lagrangian_upper_bound = lagrangian_upper_bound
        init_value = max(float(lagrangian_multiplier_init), 0.0)
        if lambda_optimizer == 'Adam':
            # state = {lambda, adam m, adam v, adam t}
            self.state = torch.tensor([init_value, 0.0, 0.0, 0.0], dtype=torch.float32, device=device)
        else:
            init = [init_value] + [0.0] * (OPT_STATE - 1)
            if lambda_optimizer == 'NAdam':
                init[3] = 1.0                            # mu_product
            elif lambda_optimizer == 'Rprop':
                init[2] = self.lambda_lr                 # step_size
            elif lambda_optimizer == 'ASGD':
                init[1], init[2] = self.lambda_lr, 1.0   # eta, mu
            self.state = torch.tensor(init, dtype=torch.float32, device=device)
        self.nan_flag = torch.zeros(1, dtype=torch.int32, device=device)
        self._jc_sums = None

    @property
    def lagrangian_multiplier(self) -> torch.Tensor:
        return self.state[0]

    def train_state(self) -> dict:
        """lambda and its optimiser state (Adam: moments / step count)."""
        return {'state': snapshot(self.state)[0]}

    def load_train_state(self, state: dict) -> None:
        restore(self.state, state['state'], 'Lagrange state')

    def update_lagrange_multiplier(self, Jc) -> None:   # noqa: N803  (the reference's argument name)
        """Reference signature `update_lagrange_multiplier(Jc: float)` (common/lagrange.py:L114-136): one
        optimiser step on lambda with gradient -(Jc - cost_limit), then projection onto [0, upper_bound].

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
        if self.lambda_optimizer == 'Adam':
            lib().osb_lagrange_update(ptr(Jc), self.cost_limit, self.lambda_lr, ub,
                                      ptr(self.state), ptr(self.nan_flag), current_stream())
        else:
            lib().osb_lagrange_update_opt(OPT_KINDS[self.lambda_optimizer], ptr(Jc), self.cost_limit,
                                          self.lambda_lr, ub, ptr(self.state), ptr(self.nan_flag), current_stream())
