"""PID-Lagrangian multiplier with its controller state on the device.

Mirrors omnisafe/common/pid_lagrange.py:L27-125 (constructor arguments, `lagrangian_multiplier`,
`pid_update`).  The controller step is `osb_pid_lagrange_update` (csrc/optim.cu), evaluated in fp64
like the reference's Python floats; `state[0]` holds the fp32 multiplier the update kernels read.
"""
from __future__ import annotations

import torch

from omnisafe_b200._lib import current_stream, lib, ptr
from omnisafe_b200.utils.train_state import restore, snapshot


class PIDLagrangian:
    def __init__(self, pid_kp: float, pid_ki: float, pid_kd: float, pid_d_delay: int,
                 pid_delta_p_ema_alpha: float, pid_delta_d_ema_alpha: float, sum_norm: bool,
                 diff_norm: bool, penalty_max: int, lagrangian_multiplier_init: float,
                 cost_limit: float, device='cuda') -> None:
        assert 1 <= int(pid_d_delay) <= 56, 'pid_d_delay must be in [1, 56] on the device path'
        self._cfg = (float(pid_kp), float(pid_ki), float(pid_kd), int(pid_d_delay),
                     float(pid_delta_p_ema_alpha), float(pid_delta_d_ema_alpha), int(bool(sum_norm)),
                     int(bool(diff_norm)), float(penalty_max), float(cost_limit))
        self.cost_limit = float(cost_limit)
        pid = torch.zeros(64, dtype=torch.float64)
        pid[0] = float(lagrangian_multiplier_init)   # _pid_i
        pid[4] = 1.0                                 # deque([0.0], maxlen=pid_d_delay)
        self.pid_state = pid.to(device)
        # the multiplier (= _cost_penalty) starts at 0.0 in the reference (pid_lagrange.py:L85)
        self.state = torch.zeros(4, dtype=torch.float32, device=device)
        self.nan_flag = torch.zeros(1, dtype=torch.int32, device=device)

    @property
    def lagrangian_multiplier(self) -> torch.Tensor:
        return self.state[0]

    def train_state(self) -> dict:
        """The fp64 controller terms (integral, EMAs, the derivative delay line) and the fp32 multiplier."""
        pid_state, state = snapshot(self.pid_state, self.state)
        return {'pid_state': pid_state, 'state': state}

    def load_train_state(self, state: dict) -> None:
        restore(self.pid_state, state['pid_state'], 'PID-Lagrangian controller state')
        restore(self.state, state['state'], 'PID-Lagrangian multiplier')

    def pid_update(self, window_sums: torch.Tensor) -> None:
        """`window_sums` = device fp64 {sum EpRet, sum EpCost, sum EpLen, count} of the episode window
        (already all-reduced): ep_cost_avg = sum EpCost / count."""
        lib().osb_pid_lagrange_update(ptr(window_sums), *self._cfg, ptr(self.pid_state), ptr(self.state),
                                      ptr(self.nan_flag), current_stream())

    update_lagrange_multiplier = pid_update   # the hook name the Lagrange mixin calls
