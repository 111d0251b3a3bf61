"""Test CMDPs for the external-env rollout (user envs stepped in PyTorch).

Imported by tests/test_external_env_gpu.py and tests/golden/make_golden_external.py.  The classes are built by factory
functions from a given `CMDP` base class and `Box` type, so the same env runs as an omnisafe_b200 CMDP on the GPU and as
a reference CMDP in the unmodified reference (which produced tests/golden/rollout_external.npz).

- `oracle_synthetic_cmdp`: the synthetic Box env of oracle/synthetic_env.py behind the CMDP contract, returning tensors
  on the env's device (the way tests/golden/make_golden.py::RefSyntheticBox wraps it).
- `wide_box_cmdp`: a torch env with an asymmetric per-dimension action box, observations up to ~1e3, terminations and
  truncations in the same step.  Every float operation is a separate elementwise fp32 op, so the CPU and CUDA runs
  produce identical bits; terminations are integer functions of the step counter.
- `WideBoxOracle`: the same env with the numpy interface oracle/rollout.py::rollout_epoch steps.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle.synthetic_env import SyntheticBoxEnv as OracleEnv

WIDE_BOX_ID = 'WideBox-v0'
ORACLE_BOX_ID = 'OracleSyntheticBox-v0'


def _unbatch(out, info, n):
    if n != 1:
        return (*out, info)
    return (*(x[0] for x in out), {k: v[0] for k, v in info.items()})


def oracle_synthetic_cmdp(CMDP, Box):
    class OracleSyntheticBox(CMDP):
        _support_envs = [ORACLE_BOX_ID]  # noqa: RUF012
        need_auto_reset_wrapper = False
        need_time_limit_wrapper = False
        need_evaluation = False

        def __init__(self, env_id, num_envs=1, device='cpu', obs_dim=60, act_dim=8, max_episode_steps=64,
                     term_prob=0.0, cost_threshold=0.0, **_):
            super().__init__(env_id)
            self._num_envs = num_envs
            self._device = torch.device(device)
            self._kw = dict(obs_dim=obs_dim, act_dim=act_dim, max_episode_steps=max_episode_steps, term_prob=term_prob,
                            cost_threshold=cost_threshold)
            self._observation_space = Box(-10.0, 10.0, (obs_dim,))
            self._action_space = Box(-1.0, 1.0, (act_dim,))
            self._env = None

        def set_seed(self, seed):
            self._env = OracleEnv(self._num_envs, seed=seed, **self._kw)

        def reset(self, seed=None, options=None):
            obs = torch.as_tensor(self._env.reset()).to(self._device)
            return (obs[0] if self._num_envs == 1 else obs), {}

        def step(self, action):
            a = torch.as_tensor(action).reshape(self._num_envs, -1).cpu().numpy()
            nobs, rew, cost, term, trunc, final, fin = self._env.step(a)
            dev = self._device
            info = {}
            if fin.any():
                info = {'final_observation': torch.as_tensor(final).to(dev), '_final_observation': torch.as_tensor(fin).to(dev)}
            out = tuple(torch.as_tensor(x).to(dev) for x in (nobs, rew, cost, term, trunc))
            return _unbatch(out, info, self._num_envs)

        def render(self):
            return None

        def close(self):
            pass

    return OracleSyntheticBox


def wide_box_bounds(act_dim):
    j = np.arange(act_dim)
    lo = (-2.0 + 0.5 * (j % 3)).astype(np.float32)       # -2, -1.5, -1, -2, ...
    hi = (0.5 + 0.75 * (j % 4)).astype(np.float32)       # 0.5, 1.25, 2, 2.75, ...
    return lo, hi


class WideBoxCore:
    """The dynamics (torch, any device).  s' = 0.9 s + 0.05 a[j mod A] scale_j with scale_j = 10^(j mod 4)."""

    def __init__(self, num_envs, obs_dim, act_dim, max_episode_steps, seed, device):
        self.N, self.O, self.A = int(num_envs), int(obs_dim), int(act_dim)
        self.tmax = int(max_episode_steps)
        self.seed = int(seed)
        self.dev = torch.device(device)
        j = torch.arange(self.O, device=self.dev)
        self.scale = (10.0 ** (j % 4)).to(torch.float32)
        self.idx = j % self.A
        self.j = j
        self.gid = torch.arange(self.N, device=self.dev)
        self.episode = torch.zeros(self.N, dtype=torch.int64, device=self.dev)
        self.ep_step = torch.zeros(self.N, dtype=torch.int64, device=self.dev)
        self.gstep = torch.zeros(self.N, dtype=torch.int64, device=self.dev)
        self.s = torch.zeros(self.N, self.O, dtype=torch.float32, device=self.dev)

    def _reset_values(self, episode):
        h = ((self.gid[:, None] * 73856093) ^ (episode[:, None] * 19349663) ^ (self.j[None, :] * 83492791)
             ^ (self.seed * 2654435761)) % 65536
        u = h.to(torch.float32) / 32768.0 - 1.0                     # exact: k / 2^15 - 1 in [-1, 1)
        return u * self.scale

    def reset(self):
        self.episode += 1
        self.ep_step.zero_()
        self.s = self._reset_values(self.episode)
        return self.s.clone()

    def step(self, a):
        a = a.to(self.dev, torch.float32).reshape(self.N, self.A)
        sn = self.s * 0.9 + (a[:, self.idx] * 0.05) * self.scale
        reward = a[:, 0] * 0.5 - sn[:, 0] * 0.001
        cost = (sn[:, 1 % self.O] > 0).to(torch.float32)
        term = ((self.gid * 7 + self.gstep * 13) % 11) == 0
        trunc = (self.ep_step + 1) >= self.tmax
        fin = term | trunc
        self.gstep += 1
        self.episode = torch.where(fin, self.episode + 1, self.episode)
        self.s = torch.where(fin[:, None], self._reset_values(self.episode), sn)
        self.ep_step = torch.where(fin, torch.zeros_like(self.ep_step), self.ep_step + 1)
        return self.s.clone(), reward, cost, term, trunc, sn, fin


def wide_box_cmdp(CMDP, Box):
    class WideBox(CMDP):
        _support_envs = [WIDE_BOX_ID]  # noqa: RUF012
        need_auto_reset_wrapper = False
        need_time_limit_wrapper = False
        need_evaluation = False

        def __init__(self, env_id, num_envs=1, device='cpu', obs_dim=45, act_dim=3, max_episode_steps=7, **_):
            super().__init__(env_id)
            self._num_envs = num_envs
            self._kw = (num_envs, obs_dim, act_dim, max_episode_steps)
            self._device = torch.device(device)
            self._observation_space = Box(-1e4, 1e4, (obs_dim,))
            lo, hi = wide_box_bounds(act_dim)
            self._action_space = Box(lo, hi, (act_dim,))
            self._core = None

        def set_seed(self, seed):
            self._core = WideBoxCore(*self._kw, seed=seed, device=self._device)

        def reset(self, seed=None, options=None):
            obs = self._core.reset()
            return (obs[0] if self._num_envs == 1 else obs), {}

        def step(self, action):
            nobs, rew, cost, term, trunc, final, fin = self._core.step(torch.as_tensor(action))
            info = {'final_observation': final, '_final_observation': fin} if bool(fin.any()) else {}
            return _unbatch((nobs, rew, cost, term, trunc), info, self._num_envs)

        def render(self):
            return None

        def close(self):
            pass

    return WideBox


class WideBoxOracle:
    """WideBoxCore on the CPU with the numpy interface of oracle/synthetic_env.py (for oracle/rollout.py)."""

    def __init__(self, num_envs, obs_dim, act_dim, max_episode_steps, seed):
        self.N, self.O, self.A = num_envs, obs_dim, act_dim
        self._core = WideBoxCore(num_envs, obs_dim, act_dim, max_episode_steps, seed, 'cpu')

    def reset(self):
        return self._core.reset().numpy()

    def step(self, action):
        out = self._core.step(torch.as_tensor(np.asarray(action, np.float32)))
        return tuple(x.numpy() for x in out)


def register(CMDP, Box, env_register, registered_ids):
    """Register both test envs once with the given registry (`registered_ids` = its current env ids)."""
    for factory, env_id in ((oracle_synthetic_cmdp, ORACLE_BOX_ID), (wide_box_cmdp, WIDE_BOX_ID)):
        if env_id not in registered_ids:
            env_register(factory(CMDP, Box))
