"""Simmer adapter (omnisafe/adapter/simmer_adapter.py:L34-131): Saute whose safety budget is moved by a PID controller
once per epoch; an epoch's reset starts the safety state at the relative budget `safety_budget / upper_budget`."""
from __future__ import annotations

import torch

from omnisafe_b200.adapter.saute_adapter import SauteAdapter, per_step_budget
from omnisafe_b200.common.simmer_agent import SimmerPIDAgent


class SimmerAdapter(SauteAdapter):
    def __init__(self, env_id: str, num_envs: int, seed: int, cfgs, device='cuda', env_id_offset: int = 0) -> None:
        super().__init__(env_id, num_envs, seed, cfgs, device=device, env_id_offset=env_id_offset)
        a = cfgs.algo_cfgs
        n = self._env.num_envs
        # fp32 [N, 1] CPU tensors like the reference's (every row equal: the controller sees one mean episode cost)
        self._budget_t = torch.ones(n, 1) * self._safety_budget
        self._upper_t = torch.ones(n, 1) * per_step_budget(float(a.upper_budget), self._saute_gamma, self._max_ep_len)
        self._rel_t = self._budget_t / self._upper_t
        self._controller = SimmerPIDAgent(cfgs.control_cfgs, budget_bound=self._upper_t)

    def _safety_init(self) -> float:
        return float(self._rel_t[0, 0])                              # simmer_adapter.py:L111

    def control_budget(self, ep_costs) -> None:
        """simmer_adapter.py:L113-131: the episode cost goes onto the per-step discounted scale, then the controller acts."""
        g, L = self._saute_gamma, self._max_ep_len
        obs = torch.as_tensor(ep_costs, dtype=torch.float32).cpu() * (1 - g ** L) / (1 - g) / L
        self._budget_t = self._controller.act(safety_budget=self._budget_t, observation=obs)
        self._rel_t = self._budget_t / self._upper_t
        self._safety_budget = float(self._budget_t[0, 0])

    def train_state(self) -> dict:
        return {**super().train_state(), 'budget': self._budget_t.clone(), 'rel': self._rel_t.clone(),
                'safety_budget': self._safety_budget, 'controller': self._controller.train_state()}

    def load_train_state(self, state: dict) -> None:
        super().load_train_state(state)
        if tuple(state['budget'].shape) != tuple(self._budget_t.shape):
            raise RuntimeError(f'training state: Simmer budget is {tuple(state["budget"].shape)}, this run has '
                               f'{tuple(self._budget_t.shape)}')
        self._budget_t, self._rel_t = state['budget'].clone(), state['rel'].clone()
        self._safety_budget = float(state['safety_budget'])
        self._controller.load_train_state(state['controller'])
