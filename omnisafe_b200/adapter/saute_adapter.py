"""Saute adapter: safety-state augmentation inside the fused rollout.

Mirrors omnisafe/adapter/saute_adapter.py:L34-260: the networks see [normalised obs | z] (observation space one wider),
z starts at 1, z <- (z - cost / budget) / saute_gamma after every step, the stored reward becomes `unsafe_reward` once
z <= 0, z returns to 1 when an episode ends; episode returns keep the original reward.  The arithmetic runs in the
rollout kernels (csrc/rollout.cu: SauteSpec / saute_step); this class owns the safety state and the budget and switches
the mode on around `OnPolicyAdapter.rollout`.
"""
from __future__ import annotations

import numpy as np
import torch

from omnisafe_b200._lib import lib, ptr
from omnisafe_b200.adapter.onpolicy_adapter import OnPolicyAdapter
from omnisafe_b200.utils.train_state import restore, snapshot


def per_step_budget(budget: float, saute_gamma: float, max_ep_len: float) -> float:
    """saute_adapter.py:L62-68: a python-double product that lands in an fp32 tensor."""
    return float(np.float32(budget * (1 - saute_gamma ** max_ep_len) / (1 - saute_gamma) / max_ep_len))


class SauteAdapter(OnPolicyAdapter):
    def __init__(self, env_id: str, num_envs: int, seed: int, cfgs, device='cuda', env_id_offset: int = 0) -> None:
        super().__init__(env_id, num_envs, seed, cfgs, device=device, env_id_offset=env_id_offset)
        a = cfgs.algo_cfgs
        assert not getattr(a, 'reward_normalize', False), 'Reward normalization is not supported'     # saute_adapter.py:L106
        assert not getattr(a, 'cost_normalize', False), 'Cost normalization is not supported'
        self._saute_gamma = float(a.saute_gamma)
        self._unsafe_reward = float(a.unsafe_reward)
        self._max_ep_len = float(a.max_ep_len)
        self._safety_budget = per_step_budget(float(a.safety_budget), self._saute_gamma, self._max_ep_len)
        self.safety = torch.zeros(2, self._env.num_envs, dtype=torch.float32, device=self._device)   # z by step parity

    @property
    def obs_dim(self) -> int:
        """saute_adapter.py:L70-75: the observation space gains the safety state."""
        return self._env.obs_dim + 1

    def _safety_init(self) -> float:
        return 1.0                                                   # saute_adapter.py:L131

    def rollout(self, steps_per_epoch: int, agent, buffer, logger=None, eps=None) -> None:
        lib().osb_rollout_set_saute(ptr(self.safety), self._safety_budget, self._saute_gamma, self._unsafe_reward,
                                    self._safety_init())
        try:
            super().rollout(steps_per_epoch, agent, buffer, logger, eps=eps)
        finally:
            lib().osb_rollout_set_saute(0, 1.0, 1.0, 0.0, 1.0)
        self._last_buffer = buffer

    def train_state(self) -> dict:
        return {**super().train_state(), 'safety': snapshot(self.safety)[0]}

    def load_train_state(self, state: dict) -> None:
        super().load_train_state(state)
        restore(self.safety, state['safety'], 'Saute safety state')

    def ep_budget_mean(self) -> float:
        """Metrics/EpBudget (saute_adapter.py:L218-260): per finished episode the sum of the safety state after each of
        its steps (after the reset at the episode's last step), averaged over the logger window of the last epoch's
        episodes.  Computed from the slabs when the epoch is logged, not in the hot path."""
        buf = self._last_buffer
        T, N = buf.T, buf.N
        W = self.window_lens
        z_now = buf.data['obs'][..., -1]                                       # z at the beginning of step t
        z_after = torch.cat([z_now[1:], self.safety[T & 1].view(1, N)], 0)     # z after step t (post reset)
        ends = buf.data['flags'] != 0
        if not bool(ends.any()):
            return float('nan')
        csum = torch.cumsum(z_after.double(), 0)
        idx = torch.where(ends, torch.arange(T, device=ends.device).view(T, 1).expand(T, N), torch.full_like(ends, -1, dtype=torch.long))
        prev = torch.cummax(idx, 0).values
        prev = torch.cat([torch.full((1, N), -1, dtype=torch.long, device=ends.device), prev[:-1]], 0)
        base = torch.where(prev >= 0, torch.gather(csum, 0, prev.clamp(min=0)), torch.zeros_like(csum))
        per_ep = (csum - base)[ends]                                           # (step, env) order = the logger's append order
        return float(per_ep[-W:].mean())
