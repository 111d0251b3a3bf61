"""Safety-budget controller of the Simmer adapter: the host-side PID of omnisafe/common/simmer_agent.py:L98-186, kept on the
host because it acts once per epoch on one number per env row.  State: the previous (blurred) error, the previous clamped and
raw actions, and a window of the last 10 blurred errors for the integral term.  All arithmetic is on fp32 CPU tensors in
the reference's operation order (the budgets it produces are compared bit-for-bit with the reference's over recorded cost
sequences, tests/test_saute_gpu.py::test_simmer_controller_golden)."""
from __future__ import annotations

from collections import deque

import torch

_TINY_BUDGET = 1e-6      # lower clamp of the safety budget (simmer_agent.py:L168-173)


class SimmerPIDAgent:
    def __init__(self, cfgs, budget_bound: torch.Tensor, action_space: tuple[float, float] = (-1.0, 1.0)) -> None:
        self._gains = cfgs                       # kp, ki, kd, polyak (control_cfgs of the YAML)
        self._bound = budget_bound               # upper budget, [N, 1]
        self._lo, self._hi = action_space
        self._last_action = torch.zeros(1)
        self._last_raw = torch.zeros(1)
        self._last_err = torch.zeros(1)
        self._window: deque = deque([], maxlen=10)

    def act(self, safety_budget: torch.Tensor, observation: torch.Tensor) -> torch.Tensor:
        """One controller step: new safety budget from the current one and the observed (scaled) episode cost."""
        g = self._gains
        err = g.polyak * self._last_err + (1 - g.polyak) * (safety_budget - observation)     # polyak-blurred error
        self._window.append(err)
        integral = torch.as_tensor(sum(self._window))
        raw = g.kp * err + g.ki * integral + g.kd * (self._last_action - self._last_raw)
        step = torch.clamp(raw, min=self._lo, max=self._hi)
        new_budget = torch.clamp(safety_budget + step, _TINY_BUDGET * torch.ones_like(safety_budget), self._bound)
        self._last_action, self._last_raw, self._last_err = new_budget - safety_budget, raw, err
        return new_budget

    def train_state(self) -> dict:
        return {'last_action': self._last_action.clone(), 'last_raw': self._last_raw.clone(),
                'last_err': self._last_err.clone(), 'window': [e.clone() for e in self._window]}

    def load_train_state(self, state: dict) -> None:
        self._last_action = state['last_action'].clone()
        self._last_raw = state['last_raw'].clone()
        self._last_err = state['last_err'].clone()
        self._window = deque((e.clone() for e in state['window']), maxlen=self._window.maxlen)
