"""Test CMDPs with the optional per-env reset `reset_envs(mask)` (envs/core.py), for the EarlyTerminated rollout on
registered envs.  They keep the arithmetic of tests/external_envs.py::WideBoxCore bit for bit; `reset_envs` starts fresh
episodes for the masked envs exactly as `reset()` does for all of them, so at N = 1 the two are the same call.

- `SeededWideBox-v0`: WideBox without the hook.
- `WideBoxReset-v0`: WideBox plus `reset_envs` (a host-side check of the mask, like WideBox's own `fin.any()`).
- `GraphWideBoxReset-v0`: graph-safe, its state and its `reset_envs` output written in place, step info always complete.
- `WideBoxResetOracle`: the numpy interface of oracle/early_external.py::rollout_epoch_early.
The CMDPs are seeded with 0 at construction, as `Evaluator` builds its env without calling `set_seed`.
"""
from __future__ import annotations

import numpy as np
import torch

import external_envs as xe

SEEDED_WIDE_ID = 'SeededWideBox-v0'
RESET_WIDE_ID = 'WideBoxReset-v0'
GRAPH_RESET_WIDE_ID = 'GraphWideBoxReset-v0'


class WideBoxResetCore(xe.WideBoxCore):
    def reset_envs(self, mask):
        mask = torch.as_tensor(mask, device=self.dev).reshape(self.N)
        self.episode = torch.where(mask, self.episode + 1, self.episode)
        self.ep_step = torch.where(mask, torch.zeros_like(self.ep_step), self.ep_step)
        self.s = torch.where(mask[:, None], self._reset_values(self.episode), self.s)
        return self.s.clone()


class GraphWideBoxResetCore(xe.WideBoxCore):
    """In-place state updates (a replay reads what the previous one wrote) and a fixed reset_envs output buffer."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.rst = torch.zeros_like(self.s)
        self.resets = 0                         # reset() calls (host counter: not advanced by a graph replay)

    def reset(self):
        self.resets += 1
        self.episode += 1
        self.ep_step.zero_()
        self.s.copy_(self._reset_values(self.episode))
        return self.s

    def reset_envs(self, mask):
        self.episode.copy_(torch.where(mask, self.episode + 1, self.episode))
        self.ep_step.copy_(torch.where(mask, torch.zeros_like(self.ep_step), self.ep_step))
        self.s.copy_(torch.where(mask[:, None], self._reset_values(self.episode), self.s))
        self.rst.copy_(self.s)
        return self.rst

    def step(self, a):
        a = a.to(self.dev, torch.float32).reshape(self.N, self.A)
        sn = self.s * 0.9 + (a[:, self.idx] * 0.05) * self.scale
        reward = a[:, 0] * 0.5 - sn[:, 0] * 0.001
        cost = (sn[:, 1 % self.O] > 0).to(torch.float32)
        term = ((self.gid * 7 + self.gstep * 13) % 11) == 0
        trunc = (self.ep_step + 1) >= self.tmax
        fin = term | trunc
        self.gstep += 1
        self.episode.copy_(torch.where(fin, self.episode + 1, self.episode))
        self.s.copy_(torch.where(fin[:, None], self._reset_values(self.episode), sn))
        self.ep_step.copy_(torch.where(fin, torch.zeros_like(self.ep_step), self.ep_step + 1))
        return self.s.clone(), reward, cost, term, trunc, sn, fin


def reset_envs_cmdps(CMDP, Box):
    class SeededWideBox(xe.wide_box_cmdp(CMDP, Box)):
        _support_envs = [SEEDED_WIDE_ID]  # noqa: RUF012

        def __init__(self, env_id, **kw):
            super().__init__(env_id, **kw)
            self.set_seed(0)

    WideBox = SeededWideBox

    class WideBoxReset(WideBox):
        _support_envs = [RESET_WIDE_ID]  # noqa: RUF012

        def set_seed(self, seed):
            self._core = WideBoxResetCore(*self._kw, seed=seed, device=self._device)

        def reset_envs(self, mask):
            obs = self._core.reset_envs(mask)
            return obs[0] if self._num_envs == 1 else obs

    class GraphWideBoxReset(WideBox):
        _support_envs = [GRAPH_RESET_WIDE_ID]  # noqa: RUF012
        graph_safe = True

        def set_seed(self, seed):
            self._core = GraphWideBoxResetCore(*self._kw, seed=seed, device=self._device)

        def reset_envs(self, mask):
            return self._core.reset_envs(mask)

        def step(self, action):
            nobs, rew, cost, term, trunc, final, fin = self._core.step(torch.as_tensor(action))
            return nobs, rew, cost, term, trunc, {'final_observation': final, '_final_observation': fin}

    return SeededWideBox, WideBoxReset, GraphWideBoxReset


def register(CMDP, Box, env_register, registered_ids):
    if RESET_WIDE_ID not in registered_ids:
        for cls in reset_envs_cmdps(CMDP, Box):
            env_register(cls)


class WideBoxResetOracle(xe.WideBoxOracle):
    def __init__(self, num_envs, obs_dim, act_dim, max_episode_steps, seed):
        self.N, self.O, self.A = num_envs, obs_dim, act_dim
        self._core = WideBoxResetCore(num_envs, obs_dim, act_dim, max_episode_steps, seed, 'cpu')

    def reset_envs(self, mask):
        return self._core.reset_envs(torch.as_tensor(np.asarray(mask))).numpy()
