"""EarlyTerminated adapter (omnisafe/adapter/early_terminated_adapter.py:L28-98): the episode ends as soon as the accumulated
cost exceeds `algo_cfgs.cost_limit` -- reward 0, terminated = 1, env reset, accumulator cleared.  Upstream supports a single
env only (`assert num_envs == 1`, L42); here every env carries its own accumulator in the rollout kernels
(csrc/rollout.cu: EarlySpec), which reduces to the reference's behaviour for one env (tests/test_saute_gpu.py checks it
against an unmodified PPOEarlyTerminated rollout).  As upstream, the accumulator is NOT cleared by ordinary episode ends."""
from __future__ import annotations

import torch

from omnisafe_b200._lib import lib, ptr
from omnisafe_b200.adapter.onpolicy_adapter import OnPolicyAdapter
from omnisafe_b200.utils.train_state import restore, snapshot


class EarlyTerminatedAdapter(OnPolicyAdapter):
    def __init__(self, env_id: str, num_envs: int, seed: int, cfgs, device='cuda', env_id_offset: int = 0) -> None:
        super().__init__(env_id, num_envs, seed, cfgs, device=device, env_id_offset=env_id_offset)
        self._cost_limit = float(cfgs.algo_cfgs.cost_limit)
        self._cost_logger = torch.zeros(self._env.num_envs, dtype=torch.float32, device=self._device)

    def rollout(self, steps_per_epoch: int, agent, buffer, logger=None, eps=None) -> None:
        lib().osb_rollout_set_early_termination(ptr(self._cost_logger), self._cost_limit)
        try:
            super().rollout(steps_per_epoch, agent, buffer, logger, eps=eps)
        finally:
            lib().osb_rollout_set_early_termination(0, 0.0)

    def train_state(self) -> dict:
        return {**super().train_state(), 'cost_logger': snapshot(self._cost_logger)[0]}

    def load_train_state(self, state: dict) -> None:
        super().load_train_state(state)
        restore(self._cost_logger, state['cost_logger'], 'early-termination cost accumulator')
