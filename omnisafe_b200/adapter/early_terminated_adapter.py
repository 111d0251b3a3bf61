"""EarlyTerminated adapter (omnisafe/adapter/early_terminated_adapter.py:L28-98): the episode ends as soon as the accumulated
cost exceeds `algo_cfgs.cost_limit` -- reward 0, terminated = 1, env reset, accumulator cleared.  Upstream supports a single
env only (`assert num_envs == 1`, L42); here every env carries its own accumulator in the rollout kernels
(csrc/rollout.cu: EarlySpec), which reduces to the reference's behaviour for one env (tests/test_saute_gpu.py checks it
against an unmodified PPOEarlyTerminated rollout).  As upstream, the accumulator is NOT cleared by ordinary episode ends.

`EarlyTerminatedAdapter` runs the rule inside the fused synthetic rollout; `ExternalEarlyTerminatedAdapter` runs it on a
user-registered env, in the observe kernel of the external-env path, and resets the envs the rule cut:
- an env with the optional `reset_envs(mask)` hook (envs/core.py), any number of envs: `reset_envs` is called after every
  observe with the device mask the kernel wrote, without a host synchronisation, so a graph-safe env keeps its epoch in
  the CUDA graph;
- an env without it and a single env (upstream's case): one 4-byte read-back per step, and `env.reset()` only when the
  rule fired; such an epoch runs eagerly even for a graph-safe env.
Either way the reset observations are pushed into ObsNormalize after the step's own pushes, as the reference's
`self._env.reset()` after `env.step` does."""
from __future__ import annotations

import torch

from omnisafe_b200._lib import lib, ptr
from omnisafe_b200.adapter.external_adapter import ExternalEnvAdapter
from omnisafe_b200.adapter.onpolicy_adapter import OnPolicyAdapter
from omnisafe_b200.utils.train_state import restore, snapshot


class _CostLimit:
    """The per-env cost accumulator of the rule and its place in the training state (both adapters)."""

    def __init__(self, env_id: str, num_envs: int, seed: int, cfgs, device='cuda', env_id_offset: int = 0) -> None:
        super().__init__(env_id, num_envs, seed, cfgs, device=device, env_id_offset=env_id_offset)
        self._cost_limit = float(cfgs.algo_cfgs.cost_limit)
        self._cost_logger = torch.zeros(self.num_envs, dtype=torch.float32, device=self._device)

    def train_state(self) -> dict:
        return {**super().train_state(), 'cost_logger': snapshot(self._cost_logger)[0]}

    def load_train_state(self, state: dict) -> None:
        super().load_train_state(state)
        restore(self._cost_logger, state['cost_logger'], 'early-termination cost accumulator')


class EarlyTerminatedAdapter(_CostLimit, OnPolicyAdapter):
    def rollout(self, steps_per_epoch: int, agent, buffer, logger=None, eps=None) -> None:
        lib().osb_rollout_set_early_termination(ptr(self._cost_logger), self._cost_limit)
        try:
            super().rollout(steps_per_epoch, agent, buffer, logger, eps=eps)
        finally:
            lib().osb_rollout_set_early_termination(0, 0.0)


class ExternalEarlyTerminatedAdapter(_CostLimit, ExternalEnvAdapter):
    def __init__(self, env_id: str, num_envs: int, seed: int, cfgs, device='cuda', env_id_offset: int = 0) -> None:
        if getattr(cfgs.algo_cfgs, 'reward_normalize', False):
            raise NotImplementedError(
                f'EarlyTerminated with reward_normalize=True is not supported on the registered env {env_id}: the '
                "reference's reward statistics take the env's reward where the rule stores 0, which the post-rollout "
                'normalisation of the reward slab cannot reproduce')
        super().__init__(env_id, num_envs, seed, cfgs, device=device, env_id_offset=env_id_offset)
        self._hook = callable(getattr(self._env, 'reset_envs', None))
        N = self._num_envs
        if not self._hook and N > 1:
            name = type(self._env).__name__
            self._env.close()
            raise NotImplementedError(
                f'EarlyTerminated on {name} with {N} envs needs the optional reset_envs(mask) hook (envs/core.py) to '
                'reset the envs the cost limit cuts; without it only a single env is supported, as upstream '
                '(early_terminated_adapter.py: num_envs == 1)')
        self._trig = torch.zeros(N, dtype=torch.bool, device=self._device)   # envs the rule cut in the last step
        self._rst_ptr = 0                               # storage of the last reset_envs() output (part of the graph key)
        self._why_eager = None
        if not self._hook:
            self._trig_total = torch.zeros(1, dtype=torch.int32, device=self._device)
            self._trig_host = torch.zeros(1, dtype=torch.int32).pin_memory()
            if self._use_graph:
                self._use_graph = False
                self._why_eager = (f'{type(self._env).__name__} is graph_safe but has no reset_envs(mask): the cost '
                                   'limit reads a trigger word back after every step and calls env.reset(), so every '
                                   'epoch runs eagerly')

    def rollout(self, steps_per_epoch: int, agent, buffer, logger=None, eps=None) -> None:
        if logger is not None and self._why_eager and not self._mode_logged:
            logger.log(self._why_eager)
        super().rollout(steps_per_epoch, agent, buffer, logger, eps=eps)

    def _observe(self, T: int, t: int, d, step_ptrs: tuple, s: int, env_dev) -> None:
        L, N, O = lib(), self._num_envs, self._obs_dim
        total = 0 if self._hook else ptr(self._trig_total)
        L.osb_ext_observe_early(*self._observe_args(T, t, d, step_ptrs), ptr(self._cost_logger), self._cost_limit,
                                ptr(self._trig), total, s)
        if self._hook:
            obs = self._env.reset_envs(self._trig.to(env_dev))
        else:
            self._trig_host.copy_(self._trig_total, non_blocking=True)
            torch.cuda.current_stream().synchronize()
            if not int(self._trig_host[0]):
                return
            obs, _ = self._env.reset()
        obs = self._rows(obs, O)
        self._rst_ptr = obs.untyped_storage().data_ptr()
        nz = self._obs_normalizer
        L.osb_ext_reset_rows(O, N, t, int(self._obs_normalize), ptr(self._trig), ptr(obs), ptr(self.s_raw), ptr(nz.mean),
                             ptr(nz.sumsq), ptr(nz.std), ptr(nz.count), ptr(nz.ticket), ptr(self._ws),
                             ptr(self.nonfinite), s)

    def _graph_key(self, T: int, agent, d, eps, reset_obs) -> tuple:
        return (*super()._graph_key(T, agent, d, eps, reset_obs), ptr(self._trig), self._rst_ptr)
