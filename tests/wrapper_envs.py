"""Test CMDPs that declare the TimeLimit / AutoReset wrappers (envs/core.py): they never reset themselves and report no
final observation, as upstream's custom envs (omnisafe/envs/custom_env.py).  Built by factory functions from a given
`CMDP` base class and `Box` type, so the same env runs here and, for tests/golden/make_golden_external_wrappers.py, in
the unmodified reference.

`WrappedBoxCore` keeps the arithmetic of tests/external_envs.py::WideBoxCore (CPU and CUDA give the same bits) but
steps without resetting: terminated is an integer function of the env's step counter, and the env also raises its own
truncated now and then, which TimeLimit discards and AutoReset alone honours.  `reset_envs(mask)` starts fresh episodes
for the masked envs exactly as `reset()` does for all of them, so at N = 1 the two are the same call.

- `WrappedBox-v0`: both wrappers, no hook;
- `AutoResetBox-v0`: AutoReset only (the env's own truncation), no hook;
- `WrappedBoxReset-v0`: both wrappers and `reset_envs`;
- `GraphWrappedBoxReset-v0`: the same, graph-safe: state and reset output written in place, `info` always empty;
- `WrappedSyntheticBox-v0`: the synthetic env of oracle/synthetic_env.py with its auto-reset taken out (it returns the
  final observation and hands the reset row to `reset_envs`), both wrappers with TimeLimit = its own episode length;
- `TimeLimitOnlyBox-v0` / `NoLimitBox-v0`: what the adapter refuses.
The CMDPs are seeded with 0 at construction, as `Evaluator` builds its env without calling `set_seed`.
"""
from __future__ import annotations

import numpy as np
import torch

import external_envs as xe
from oracle.synthetic_env import SyntheticBoxEnv as OracleEnv

WRAPPED_ID = 'WrappedBox-v0'
AUTO_RESET_ID = 'AutoResetBox-v0'
WRAPPED_RESET_ID = 'WrappedBoxReset-v0'
GRAPH_WRAPPED_ID = 'GraphWrappedBoxReset-v0'
WRAPPED_SYNTH_ID = 'WrappedSyntheticBox-v0'
TIME_LIMIT_ONLY_ID = 'TimeLimitOnlyBox-v0'
NO_LIMIT_ID = 'NoLimitBox-v0'


class WrappedBoxCore(xe.WideBoxCore):
    def step(self, a):
        a = a.to(self.dev, torch.float32).reshape(self.N, self.A)
        sn = self.s * 0.9 + (a[:, self.idx] * 0.05) * self.scale
        reward = a[:, 0] * 0.5 - sn[:, 0] * 0.001
        cost = (sn[:, 1 % self.O] > 0).to(torch.float32)
        term = (((self.gid * 7 + self.gstep * 13) % 11) == 0) | (((self.gid * 3 + self.gstep * 5) % 9) == 4)
        trunc = ((self.gid * 5 + self.gstep * 3) % 13) == 4
        self.gstep += 1
        self.s.copy_(sn)
        return sn.clone(), reward, cost, term, trunc

    def reset(self):
        self.episode += 1
        self.s.copy_(self._reset_values(self.episode))
        return self.s.clone()

    def reset_envs(self, mask):
        mask = torch.as_tensor(mask, device=self.dev).reshape(self.N)
        self.episode.copy_(torch.where(mask, self.episode + 1, self.episode))
        self.s.copy_(torch.where(mask[:, None], self._reset_values(self.episode), self.s))
        return self.s.clone()


class GraphWrappedBoxCore(WrappedBoxCore):
    """Every output in a fixed buffer: step and reset_envs return the same storage on every call."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.rst = torch.zeros_like(self.s)
        self.resets = 0                         # reset() calls (host counter: not advanced by a graph replay)

    def reset(self):
        self.resets += 1
        self.episode += 1
        self.s.copy_(self._reset_values(self.episode))
        return self.s

    def reset_envs(self, mask):
        self.episode.copy_(torch.where(mask, self.episode + 1, self.episode))
        self.rst.copy_(torch.where(mask[:, None], self._reset_values(self.episode), self.s))
        self.s.copy_(self.rst)
        return self.rst


def wrapper_cmdps(CMDP, Box):
    class WrappedBox(CMDP):
        _support_envs = [WRAPPED_ID]  # noqa: RUF012
        need_auto_reset_wrapper = True
        need_time_limit_wrapper = True
        need_evaluation = False
        _core_cls = WrappedBoxCore

        def __init__(self, env_id, num_envs=1, device='cpu', obs_dim=45, act_dim=3, max_episode_steps=4, **_):
            super().__init__(env_id)
            self._num_envs = num_envs
            self._kw = (num_envs, obs_dim, act_dim, max_episode_steps)
            self._max_episode_steps = max_episode_steps
            self._device = torch.device(device)
            self._observation_space = Box(-1e4, 1e4, (obs_dim,))
            lo, hi = xe.wide_box_bounds(act_dim)
            self._action_space = Box(lo, hi, (act_dim,))
            self.set_seed(0)

        @property
        def max_episode_steps(self):
            return self._max_episode_steps

        def set_seed(self, seed):
            self._core = self._core_cls(*self._kw, seed=seed, device=self._device)

        def _out(self, x):
            return x[0] if self._num_envs == 1 else x

        def reset(self, seed=None, options=None):
            return self._out(self._core.reset()), {}

        def step(self, action):
            out = self._core.step(torch.as_tensor(action))
            return (*(self._out(x) for x in out), {})

        def render(self):
            return None

        def close(self):
            pass

    class AutoResetBox(WrappedBox):
        _support_envs = [AUTO_RESET_ID]  # noqa: RUF012
        need_time_limit_wrapper = False

    class WrappedBoxReset(WrappedBox):
        _support_envs = [WRAPPED_RESET_ID]  # noqa: RUF012

        def reset_envs(self, mask):
            return self._out(self._core.reset_envs(mask))

    class GraphWrappedBoxReset(WrappedBox):
        _support_envs = [GRAPH_WRAPPED_ID]  # noqa: RUF012
        graph_safe = True
        _core_cls = GraphWrappedBoxCore

        def reset_envs(self, mask):
            return self._core.reset_envs(mask)

    class TimeLimitOnlyBox(WrappedBox):
        _support_envs = [TIME_LIMIT_ONLY_ID]  # noqa: RUF012
        need_auto_reset_wrapper = False

    class NoLimitBox(WrappedBoxReset):
        _support_envs = [NO_LIMIT_ID]  # noqa: RUF012

        @property
        def max_episode_steps(self):
            return None

    return WrappedBox, AutoResetBox, WrappedBoxReset, GraphWrappedBoxReset, TimeLimitOnlyBox, NoLimitBox


def wrapped_synthetic_cmdp(CMDP, Box):
    class WrappedSyntheticBox(xe.oracle_synthetic_cmdp(CMDP, Box)):
        """The oracle synthetic env without its auto-reset: step returns the final row of a finished env and keeps its
        reset row for reset_envs; TimeLimit at max_episode_steps replaces its own truncation, which it equals."""
        _support_envs = [WRAPPED_SYNTH_ID]  # noqa: RUF012
        need_auto_reset_wrapper = True
        need_time_limit_wrapper = True

        @property
        def max_episode_steps(self):
            return self._kw['max_episode_steps']

        def set_seed(self, seed):
            self._env = OracleEnv(self._num_envs, seed=seed, **self._kw)
            self._fin = np.zeros(self._num_envs, bool)

        def reset(self, seed=None, options=None):
            obs = torch.as_tensor(self._env.reset()).to(self._device)
            return (obs[0] if self._num_envs == 1 else obs), {}

        def step(self, action):
            a = torch.as_tensor(action).reshape(self._num_envs, -1).cpu().numpy()
            nobs, rew, cost, term, _, final, fin = self._env.step(a)
            self._fin = fin
            obs = np.where(fin[:, None], final, nobs)
            out = tuple(torch.as_tensor(x).to(self._device) for x in (obs, rew, cost, term, np.zeros_like(term)))
            return (*(x[0] if self._num_envs == 1 else x for x in out), {})

        def reset_envs(self, mask):
            mask = torch.as_tensor(mask).reshape(-1).cpu().numpy()
            assert np.array_equal(mask, self._fin), 'reset_envs must reset exactly the envs that finished'
            return torch.as_tensor(self._env.s).to(self._device)

    return WrappedSyntheticBox


def register(CMDP, Box, env_register, registered_ids):
    if WRAPPED_ID not in registered_ids:
        for cls in (*wrapper_cmdps(CMDP, Box), wrapped_synthetic_cmdp(CMDP, Box)):
            env_register(cls)


class WrappedBoxOracle:
    """WrappedBoxCore on the CPU with the numpy interface of oracle/wrapped_external.py."""

    def __init__(self, num_envs, obs_dim, act_dim, seed):
        self.N, self.O, self.A = num_envs, obs_dim, act_dim
        self._core = WrappedBoxCore(num_envs, obs_dim, act_dim, 1, seed, 'cpu')

    def reset(self):
        return self._core.reset().numpy()

    def step(self, action):
        return tuple(x.numpy() for x in self._core.step(torch.as_tensor(np.asarray(action, np.float32))))

    def reset_envs(self, mask):
        return self._core.reset_envs(torch.as_tensor(np.asarray(mask))).numpy()
