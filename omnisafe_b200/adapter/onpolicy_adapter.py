"""On-policy adapter: owns the env + ObsNormalize state and drives the fused rollout.

Mirrors omnisafe/adapter/onpolicy_adapter.py:L30-175 / online_adapter.py:L38-246: same
constructor `(env_id, num_envs, seed, cfgs)`, same `rollout(steps_per_epoch, agent, buffer,
logger)` entry; the body is one call into `osb_rollout_epoch` (reset, T fused step launches,
epoch-end bootstrap launch, episode window).
"""
from __future__ import annotations

import torch

from omnisafe_b200._lib import current_stream, lib, ptr
from omnisafe_b200.common.normalizer import Normalizer, ScalarNormalizer
from omnisafe_b200.envs.synthetic import SyntheticBoxEnv
from omnisafe_b200.utils.train_state import restore, snapshot


class OnPolicyAdapter:
    def __init__(self, env_id: str, num_envs: int, seed: int, cfgs, device='cuda',
                 env_id_offset: int = 0) -> None:
        self._cfgs = cfgs
        self._device = torch.device(device)
        env_cfgs = getattr(cfgs, 'env_cfgs', None) or {}
        env_cfgs = dict(env_cfgs.todict() if hasattr(env_cfgs, 'todict') else env_cfgs)
        env_cfgs.pop('env_id_offset', None)
        self._env = SyntheticBoxEnv(env_id, num_envs=num_envs, device=self._device,
                                    env_id_offset=env_id_offset, **env_cfgs)
        self._env.set_seed(seed)
        algo = cfgs.algo_cfgs
        # RewardNormalize / CostNormalize wrappers (online_adapter.py:L98-101, wrapper.py:L280-423)
        self._reward_normalizer = ScalarNormalizer(5.0, self._device) if getattr(algo, 'reward_normalize', False) else None
        self._cost_normalizer = ScalarNormalizer(5.0, self._device) if getattr(algo, 'cost_normalize', False) else None
        self._obs_normalize = bool(getattr(algo, 'obs_normalize', True))
        self._obs_normalizer = Normalizer((self._env.obs_dim,), clip=5.0, device=self._device)
        W = int(getattr(cfgs.logger_cfgs, 'window_lens', 100))
        self.window_lens = W
        self.ep_ring = torch.zeros(3, W, dtype=torch.float32, device=self._device)
        self.ep_meta = torch.zeros(2, dtype=torch.int32, device=self._device)
        self.window_sums = torch.zeros(4, dtype=torch.float64, device=self._device)
        self._epoch_index = 0
        prec = str(getattr(cfgs.train_cfgs, 'matmul_precision', 'bf16x3') if hasattr(cfgs, 'train_cfgs') else 'fp32')
        self.precision = {'fp32': 0, 'tf32': 1, 'bf16x3': 2}[prec]
        self.noise_seed = (int(seed) * 2654435761 + 12345) & 0xFFFFFFFF

    @property
    def env(self) -> SyntheticBoxEnv:
        return self._env

    @property
    def obs_dim(self) -> int:
        return self._env.obs_dim

    @property
    def act_dim(self) -> int:
        return self._env.act_dim

    @property
    def num_envs(self) -> int:
        return self._env.num_envs

    def save(self) -> dict:
        """What OnlineAdapter.save() exposes for checkpoints (online_adapter.py:L222-231)."""
        saved = {'obs_normalizer': self._obs_normalizer} if self._obs_normalize else {}
        if self._reward_normalizer is not None:
            saved['reward_normalizer'] = self._reward_normalizer
        if self._cost_normalizer is not None:
            saved['cost_normalizer'] = self._cost_normalizer
        return saved

    def rollout(self, steps_per_epoch: int, agent, buffer, logger=None, eps=None) -> None:
        """Roll the envs for `steps_per_epoch` steps each and fill `buffer`.

        `agent` is the flat-parameter ConstraintActorCritic; `eps` (optional, [T, N, A]) supplies
        the standard-normal stream (parity mode); by default the kernel draws Philox noise."""
        env, T = self._env, int(steps_per_epoch)
        assert T == buffer.T and env.num_envs == buffer.N
        if eps is not None:
            assert eps.shape == (T, env.num_envs, env.act_dim) and eps.dtype == torch.float32
        args = (env.spec_args(self._obs_normalize) + [env.num_envs, T] + env.state_ptrs()
                + self._obs_normalizer.ptrs() + buffer.slab_ptrs()
                + [ptr(agent.theta), ptr(eps), self.noise_seed, self._epoch_index & 0xFFFFFFFF,
                   self.window_lens, ptr(self.ep_ring), ptr(self.ep_meta), ptr(self.window_sums),
                   int(self.precision), current_stream()])
        agent.apply_net_spec()
        lib().osb_rollout_epoch(*args)
        # the policy never sees rewards inside a rollout: the per-step reward / cost normalisation of the
        # reference commutes with the rollout and runs on the finished slab (episode statistics stay raw,
        # info['original_reward'] in the reference)
        if self._reward_normalizer is not None:
            self._reward_normalizer.normalize_rows_(buffer.data['reward'])
        if self._cost_normalizer is not None:
            self._cost_normalizer.normalize_rows_(buffer.data['cost'])
        self._epoch_index += 1

    def train_state(self) -> dict:
        return {**episode_state(self), 'env': self._env.train_state()}

    def load_train_state(self, state: dict) -> None:
        load_episode_state(self, state)
        self._env.load_train_state(state['env'])

    def close(self) -> None:
        self._env.close()


def episode_state(ad) -> dict:
    """The state an adapter (OnPolicyAdapter, ExternalEnvAdapter) carries from one epoch to the next besides its env's:
    the Philox epoch counter, the episode window and every normaliser."""
    ring, meta, sums = snapshot(ad.ep_ring, ad.ep_meta, ad.window_sums)
    state = {'epoch_index': ad._epoch_index, 'ep_ring': ring, 'ep_meta': meta, 'window_sums': sums,
             'obs_normalizer': ad._obs_normalizer.train_state()}
    for key in ('reward_normalizer', 'cost_normalizer'):
        nz = getattr(ad, f'_{key}')
        if nz is not None:
            state[key] = nz.train_state()
    return state


def load_episode_state(ad, state: dict) -> None:
    ad._epoch_index = int(state['epoch_index'])
    restore(ad.ep_ring, state['ep_ring'], 'episode ring')
    restore(ad.ep_meta, state['ep_meta'], 'episode ring counters')
    restore(ad.window_sums, state['window_sums'], 'episode window sums')
    ad._obs_normalizer.load_train_state(state['obs_normalizer'])
    for key in ('reward_normalizer', 'cost_normalizer'):
        nz = getattr(ad, f'_{key}')
        if (nz is not None) != (key in state):
            raise RuntimeError(f'training state: {key} is {"absent" if nz is None else "present"} in this run, '
                               f'{"present" if key in state else "absent"} in the saved one')
        if nz is not None:
            nz.load_train_state(state[key])
