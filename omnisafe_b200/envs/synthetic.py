"""Device-resident synthetic Box CMDP (the env the fused rollout kernel steps in-kernel).

Mirrors the reference's vector-env contract (omnisafe/envs/core.py:L37-182): class attributes
`need_auto_reset_wrapper = need_time_limit_wrapper = False` (mandatory for num_envs > 1,
envs/wrapper.py:L51,L130), `need_evaluation = False`, constructor `(env_id, num_envs, device,
**env_cfgs)` (adapter/online_adapter.py:L71).  The transition itself is not a Python method: it is
fused into `osb_rollout_step` (csrc/rollout.cu); this object only owns the state tensors.
The specification of the dynamics lives in oracle/synthetic_env.py (test infrastructure).
"""
from __future__ import annotations

import numpy as np
import torch

from omnisafe_b200.utils.train_state import restore

_SUPPORT = ['SyntheticBox-v0']


def support_envs() -> list[str]:
    return list(_SUPPORT)


def env_bias(obs_dim: int) -> np.ndarray:
    j = np.arange(obs_dim)
    return (np.float32(0.02) * ((7 * j + 3) % 5 - 2).astype(np.float32)).astype(np.float32)


def term_threshold(term_prob: float) -> int:
    if term_prob >= 1.0:
        return 0xFFFFFFFF
    return int(max(term_prob, 0.0) * 4294967296.0) & 0xFFFFFFFF


class SyntheticBoxEnv:
    """N synthetic Box envs with state in HBM: obs in R^O, action in [-1, 1]^A."""

    need_auto_reset_wrapper = False
    need_time_limit_wrapper = False
    need_evaluation = False
    _support_envs = _SUPPORT

    def __init__(self, env_id: str, num_envs: int = 1, device='cuda', *, obs_dim: int = 60,
                 act_dim: int = 8, max_episode_steps: int = 64, term_prob: float = 0.0,
                 cost_threshold: float = 0.0, env_id_offset: int = 0) -> None:
        assert env_id in _SUPPORT, f'{env_id} is not supported by SyntheticBoxEnv'
        assert 0 < act_dim <= 16, 'act_dim must be in (0, 16]'
        assert num_envs * 10.0 * 10.0 * 2.0**36 < 2.0**62, 'too many envs for the fixed-point sums'
        self.env_id = env_id
        self._num_envs = int(num_envs)
        self.device = torch.device(device)
        self.obs_dim, self.act_dim = int(obs_dim), int(act_dim)
        self.max_episode_steps = int(max_episode_steps)
        self.term_threshold = term_threshold(term_prob)
        self.cost_threshold = float(cost_threshold)
        self.env_id_offset = int(env_id_offset)
        self.seed = 0
        N, O, dev = self._num_envs, self.obs_dim, self.device
        self.s_raw = torch.zeros(2, N, O, dtype=torch.float32, device=dev)
        self.final_raw = torch.zeros(2, N, O, dtype=torch.float32, device=dev)
        self.ep_step = torch.zeros(N, dtype=torch.int32, device=dev)
        self.episode = torch.zeros(N, dtype=torch.int32, device=dev)   # uint32 bits
        self.gstep = torch.zeros(N, dtype=torch.int32, device=dev)     # uint32 bits
        self.ep_ret = torch.zeros(N, dtype=torch.float32, device=dev)
        self.ep_cost = torch.zeros(N, dtype=torch.float32, device=dev)
        self.ep_len = torch.zeros(N, dtype=torch.int32, device=dev)
        self.bias = torch.from_numpy(env_bias(O)).to(dev)

    @property
    def num_envs(self) -> int:
        return self._num_envs

    def set_seed(self, seed: int) -> None:
        self.seed = int(seed) & 0xFFFFFFFF

    def spec_args(self, obs_normalize: bool) -> list:
        """Leading scalar arguments of the osb_env_reset / osb_rollout_* entry points."""
        return [self.obs_dim, self.act_dim, self.max_episode_steps, self.seed, self.term_threshold,
                self.env_id_offset & 0xFFFFFFFF, self.cost_threshold, int(obs_normalize)]

    def state_ptrs(self) -> list:
        return [t.data_ptr() for t in (self.s_raw, self.final_raw, self.ep_step, self.episode,
                                       self.gstep, self.ep_ret, self.ep_cost, self.ep_len, self.bias)]

    _STATE = ('s_raw', 'final_raw', 'ep_step', 'episode', 'gstep', 'ep_ret', 'ep_cost', 'ep_len')

    def train_state(self) -> dict:
        """The per-env state the rollout kernel carries across epochs (`bias` is a function of obs_dim)."""
        return {k: getattr(self, k).detach().cpu().clone() for k in self._STATE}

    def load_train_state(self, state: dict) -> None:
        for k in self._STATE:
            restore(getattr(self, k), state[k], f'synthetic env {k}')

    def close(self) -> None:
        pass
