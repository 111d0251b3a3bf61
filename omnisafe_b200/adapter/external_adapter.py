"""On-policy adapter for user-registered CMDPs: the env steps in PyTorch, everything else stays on the kernels.

Same constructor, `rollout(steps_per_epoch, agent, buffer, logger, eps=None)`, `save()` and `obs_dim / act_dim /
num_envs` as `OnPolicyAdapter` (omnisafe/adapter/onpolicy_adapter.py:L30-175).  One epoch:

    env.reset() -> osb_ext_reset_ingest
    for t in 0 .. T-1:  osb_ext_act(t) -> env.step(action) -> osb_ext_observe(t)
    osb_ext_act(T) (epoch-end bootstrap) -> osb_episode_window -> Reward / CostNormalize slab post-pass

osb_ext_act runs ObsNormalize, the three MLP forwards, sampling / log-prob and ActionScale, appends the obs / act /
logp / value slabs and writes the bootstrap values; osb_ext_observe appends reward / cost / flags, keeps the episode
statistics and feeds the observation normaliser.  Nothing in the loop synchronises the host except the env's own code
(and, for an env on the CPU, the copy of the action to it).  A non-finite observation raises `OsbError` at the end of
the epoch.

For an env that declares `graph_safe` (envs/core.py) the loop from osb_ext_act(0) to osb_ext_act(T) is captured into
one CUDA graph in the second epoch and replayed from then on (the first epoch the adapter runs -- also the first one
after `load_train_state` in a resumed process -- is eager and warms everything up); the
captured act launches read the Philox epoch from a device counter that the graph's last kernel advances.  The reset and
everything after the epoch-end act run outside the graph, with the same code as the eager loop.  OSB_NO_GRAPH=1 keeps
every epoch eager.
"""
from __future__ import annotations

import os

import torch

from omnisafe_b200._lib import OsbError, current_stream, lib, ptr
from omnisafe_b200.adapter.onpolicy_adapter import episode_state, load_episode_state
from omnisafe_b200.common.normalizer import Normalizer, ScalarNormalizer
from omnisafe_b200.envs.core import check_env, make
from omnisafe_b200.utils.train_state import restore, snapshot


class ExternalEnvAdapter:
    def __init__(self, env_id: str, num_envs: int, seed: int, cfgs, device='cuda',
                 env_id_offset: int = 0) -> None:
        self._cfgs = cfgs
        self._device = torch.device(device)
        env_cfgs = getattr(cfgs, 'env_cfgs', None) or {}
        env_cfgs = dict(env_cfgs.todict() if hasattr(env_cfgs, 'todict') else env_cfgs)
        env_cfgs.pop('env_id_offset', None)
        self._env = make(env_id, num_envs=num_envs, device=self._device, **env_cfgs)
        self._obs_dim, self._act_dim, lo, hi = check_env(self._env)
        self._num_envs = int(num_envs)
        self._env.set_seed(seed)                      # per-rank seed, as OnlineAdapter does (online_adapter.py:L81)
        self._env_id_offset = int(env_id_offset)
        algo = cfgs.algo_cfgs
        self._reward_normalizer = ScalarNormalizer(5.0, self._device) if getattr(algo, 'reward_normalize', False) else None
        self._cost_normalizer = ScalarNormalizer(5.0, self._device) if getattr(algo, 'cost_normalize', False) else None
        self._obs_normalize = bool(getattr(algo, 'obs_normalize', True))
        self._obs_normalizer = Normalizer((self._obs_dim,), clip=5.0, device=self._device)
        W = int(getattr(cfgs.logger_cfgs, 'window_lens', 100))
        self.window_lens = W
        self.ep_ring = torch.zeros(3, W, dtype=torch.float32, device=self._device)
        self.ep_meta = torch.zeros(2, dtype=torch.int32, device=self._device)
        self.window_sums = torch.zeros(4, dtype=torch.float64, device=self._device)
        self._epoch_index = 0
        prec = str(getattr(cfgs.train_cfgs, 'matmul_precision', 'bf16x3') if hasattr(cfgs, 'train_cfgs') else 'fp32')
        self.precision = {'fp32': 0, 'tf32': 1, 'bf16x3': 2}[prec]
        self.noise_seed = (int(seed) * 2654435761 + 12345) & 0xFFFFFFFF
        N, O, A, dev = self._num_envs, self._obs_dim, self._act_dim, self._device
        f32 = dict(dtype=torch.float32, device=dev)
        self.s_raw = torch.zeros(2, N, O, **f32)
        self.final_raw = torch.zeros(2, N, O, **f32)
        self.ep_ret = torch.zeros(N, **f32)
        self.ep_cost = torch.zeros(N, **f32)
        self.ep_len = torch.zeros(N, dtype=torch.int32, device=dev)
        self.act_lo = torch.as_tensor(lo).to(dev)
        self.act_hi = torch.as_tensor(hi).to(dev)
        self.act_env = torch.zeros(N, A, **f32)
        self._ws = torch.zeros(lib().osb_ext_workspace_doubles(O, N), dtype=torch.float64, device=dev)
        self.nonfinite = torch.zeros(1, dtype=torch.int32, device=dev)
        # CUDA-graph replay of the epoch for envs that declare graph_safe (envs/core.py); OSB_NO_GRAPH=1 turns it off
        self._use_graph = bool(getattr(self._env, 'graph_safe', False)) and not os.getenv('OSB_NO_GRAPH')
        self._mode_logged = False
        self._warm = False                              # an epoch ran in this process: the next one may replay
        self._graph = None
        self._graph_key_baked = None
        self.captures = 0                               # graphs captured so far (a recapture follows a pointer change)
        self._epoch_dev = torch.zeros(1, dtype=torch.int32, device=dev)    # u32 Philox epoch counter of the replays
        self._obs0 = torch.zeros(N, O, **f32)           # static copy of env.reset()'s observation (graph mode)
        self._eps_buf = None                            # static [T, N, A] copy of the parity-mode noise (graph mode)

    @property
    def env(self):
        return self._env

    @property
    def obs_dim(self) -> int:
        return self._obs_dim

    @property
    def act_dim(self) -> int:
        return self._act_dim

    @property
    def num_envs(self) -> int:
        return self._num_envs

    def save(self) -> dict:
        """What OnlineAdapter.save() exposes for checkpoints (online_adapter.py:L222-231)."""
        saved = {'obs_normalizer': self._obs_normalizer} if self._obs_normalize else {}
        if self._reward_normalizer is not None:
            saved['reward_normalizer'] = self._reward_normalizer
        if self._cost_normalizer is not None:
            saved['cost_normalizer'] = self._cost_normalizer
        return saved

    # ---- env output -> contiguous device tensors ---------------------------------------------------
    def _rows(self, x, width: int | None = None, dtype=torch.float32) -> torch.Tensor:
        x = torch.as_tensor(x)
        shape = (self._num_envs,) if width is None else (self._num_envs, width)
        return x.to(device=self._device, dtype=dtype).reshape(shape).contiguous()

    def _norm_ptrs(self) -> list:
        n = self._obs_normalizer
        return [ptr(n.mean), ptr(n.sumsq), ptr(n.std), ptr(n.mean1), ptr(n.std1), ptr(n.count), ptr(n.had_fin),
                ptr(n.ticket)]

    @property
    def graph_mode(self) -> str:
        """'graph' when the epoch's steps are replayed from a CUDA graph (from the second epoch on), else 'eager'."""
        return 'graph' if self._use_graph else 'eager'

    def _act(self, agent, d, T: int, t: int, eps_t, s: int, epoch_dev=None) -> None:
        """One act launch: eager with the host Philox counter, or (epoch_dev) the capturable form reading it on the GPU."""
        nz, O, A, N = self._obs_normalizer, self._obs_dim, self._act_dim, self._num_envs
        head = (O, A, int(self._obs_normalize), N, T, t, self._env_id_offset & 0xFFFFFFFF, ptr(self.s_raw),
                ptr(self.final_raw), ptr(nz.mean), ptr(nz.std), ptr(nz.mean1), ptr(nz.std1), ptr(nz.count),
                ptr(d['obs']), ptr(d['act']), ptr(d['logp']), ptr(d['value_r']), ptr(d['value_c']), ptr(d['boot_r']),
                ptr(d['boot_c']), ptr(d['flags']), ptr(agent.theta), ptr(eps_t), self.noise_seed)
        tail = (ptr(self.act_lo), ptr(self.act_hi), ptr(self.act_env), int(self.precision), s)
        if epoch_dev is None:
            lib().osb_ext_act(*head, (self._epoch_index * T + t) & 0xFFFFFFFF, *tail)
        else:
            lib().osb_ext_act_graph(*head, ptr(epoch_dev), *tail)

    def _steps(self, T: int, agent, d, eps, s: int, env_dev, epoch_dev=None, capture: bool = False) -> None:
        """Steps 0 .. T-1 (act, env.step, observe) and the epoch-end act, eagerly or into the graph being captured."""
        N, O = self._num_envs, self._obs_dim
        for t in range(T):
            self._act(agent, d, T, t, None if eps is None else eps[t], s, epoch_dev)
            # a fresh tensor every step, as the reference hands the env: the buffer is rewritten by the next act step
            action = self.act_env.to(env_dev, copy=True)
            if N == 1:
                action = action[0]                  # a single env takes an unbatched action (reference Unsqueeze)
            nobs, rew, cost, term, trunc, info = self._env.step(action)
            nobs = self._rows(nobs, O)
            rew, cost = self._rows(rew), self._rows(cost)
            term, trunc = self._rows(term, dtype=torch.uint8), self._rows(trunc, dtype=torch.uint8)
            final = mask = None
            if capture and ('final_observation' not in info or '_final_observation' not in info):
                raise OsbError(f'{type(self._env).__name__} is graph_safe but its step info lacks final_observation / '
                               '_final_observation: a captured step must report them on every step')
            if 'final_observation' in info:
                final = self._rows(info['final_observation'], O)
                mask = info.get('_final_observation')
                mask = (term | trunc) if mask is None else self._rows(mask, dtype=torch.uint8)
            self._observe(T, t, d, (ptr(nobs), ptr(rew), ptr(cost), ptr(term), ptr(trunc), ptr(final), ptr(mask)), s,
                          env_dev)
        self._act(agent, d, T, T, None, s, epoch_dev)

    def _observe(self, T: int, t: int, d, step_ptrs: tuple, s: int, env_dev) -> None:
        """The observe launch of step t; step_ptrs = (next obs, reward, cost, terminated, truncated, final obs, final
        mask) as device pointers."""
        lib().osb_ext_observe(*self._observe_args(T, t, d, step_ptrs), s)

    def _observe_args(self, T: int, t: int, d, step_ptrs: tuple) -> tuple:
        return (self._obs_dim, self._num_envs, T, t, int(self._obs_normalize), *step_ptrs, ptr(self.s_raw),
                ptr(self.final_raw), ptr(self.ep_ret), ptr(self.ep_cost), ptr(self.ep_len), *self._norm_ptrs(),
                ptr(d['reward']), ptr(d['cost']), ptr(d['flags']), ptr(d['epfin']), ptr(self._ws), ptr(self.nonfinite))

    def _graph_key(self, T: int, agent, d, eps, reset_obs) -> tuple:
        """The device pointers (and shape) a captured epoch bakes in; a change of any of them forces a recapture."""
        return (T, ptr(agent.theta), tuple(ptr(v) for v in d.values() if v is not None), ptr(eps),
                tuple(self._norm_ptrs()), torch.as_tensor(reset_obs).untyped_storage().data_ptr())

    def _capture(self, T: int, agent, d, eps, env_dev) -> None:
        """Capture the T steps, the epoch-end act and the Philox epoch advance into one CUDA graph."""
        N, O, A = self._num_envs, self._obs_dim, self._act_dim
        self._graph = None                          # release the old graph (and its pool) before capturing anew
        lib().osb_ext_prepare(O, A, N, int(self.precision))
        e = self._epoch_index & 0xFFFFFFFF
        self._epoch_dev.fill_(e - (1 << 32) if e >= (1 << 31) else e)     # the u32 counter, stored as int32 bits
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, pool=torch.cuda.graph_pool_handle()):
            s = current_stream()
            self._steps(T, agent, d, eps, s, env_dev, self._epoch_dev, capture=True)
            lib().osb_ext_epoch_advance(ptr(self._epoch_dev), s)
        self._graph = graph
        self.captures += 1

    def rollout(self, steps_per_epoch: int, agent, buffer, logger=None, eps=None) -> None:
        """Roll the envs for `steps_per_epoch` steps each and fill `buffer` (see the module docstring).

        `eps` (optional, [T, N, A]) supplies the standard-normal stream (parity mode); by default the kernel draws
        Philox noise."""
        T, N, O, A = int(steps_per_epoch), self._num_envs, self._obs_dim, self._act_dim
        assert T == buffer.T and N == buffer.N
        if eps is not None:
            assert eps.shape == (T, N, A) and eps.dtype == torch.float32
        if logger is not None and not self._mode_logged:
            logger.log(f'{type(self._env).__name__}: external-env rollout in {self.graph_mode} mode')
            self._mode_logged = True
        L, d, s = lib(), buffer.data, current_stream()
        obs, _ = self._env.reset()
        env_dev = torch.as_tensor(obs).device
        if self._use_graph and env_dev.type != 'cuda':
            raise ValueError(f'{type(self._env).__name__} declares graph_safe but reset() returned observations on {env_dev}')
        replay = self._use_graph and self._warm
        reset_obs = obs
        if replay:
            obs = self._obs0.copy_(torch.as_tensor(reset_obs).reshape(N, O))
        else:
            obs = self._rows(obs, O)
        L.osb_ext_reset_ingest(O, N, int(self._obs_normalize), ptr(obs), ptr(self.s_raw), ptr(self.ep_ret),
                               ptr(self.ep_cost), ptr(self.ep_len), *self._norm_ptrs(), ptr(self._ws),
                               ptr(self.nonfinite), s)
        if replay:
            if eps is not None:
                if self._eps_buf is None or self._eps_buf.shape != (T, N, A):
                    self._eps_buf = torch.empty(T, N, A, dtype=torch.float32, device=self._device)
                self._eps_buf.copy_(eps)
            eps_g = None if eps is None else self._eps_buf
            key = self._graph_key(T, agent, d, eps_g, reset_obs)
            if self._graph is None or key != self._graph_key_baked:
                self._capture(T, agent, d, eps_g, env_dev)
                self._graph_key_baked = key
            self._graph.replay()
        else:
            self._steps(T, agent, d, eps, s, env_dev)
        self._end_epoch(T, d, s)

    def _end_epoch(self, T: int, d, s: int) -> None:
        """Episode window, Reward / CostNormalize post-pass and the non-finite check (eager and graph epochs alike)."""
        N = self._num_envs
        lib().osb_episode_window(ptr(d['flags']), ptr(d['epfin']), T, N, self.window_lens, ptr(self.ep_ring),
                                 ptr(self.ep_meta), ptr(self.window_sums), s)
        # the per-step reward / cost normalisation of the reference commutes with the rollout (OnPolicyAdapter.rollout)
        if self._reward_normalizer is not None:
            self._reward_normalizer.normalize_rows_(d['reward'])
        if self._cost_normalizer is not None:
            self._cost_normalizer.normalize_rows_(d['cost'])
        self._epoch_index += 1
        self._warm = True
        if int(self.nonfinite.item()):
            self.nonfinite.zero_()
            raise OsbError(f'{type(self._env).__name__} returned a non-finite observation during the last epoch')

    def train_state(self) -> dict:
        """The adapter's own per-env state, the episode window, the normalisers and -- when the env has the optional
        `state_dict()` / `load_state_dict(sd)` hooks (envs/core.py) -- the env's state."""
        s_raw, final_raw, ep_ret, ep_cost, ep_len = snapshot(self.s_raw, self.final_raw, self.ep_ret, self.ep_cost,
                                                             self.ep_len)
        state = {**episode_state(self), 's_raw': s_raw, 'final_raw': final_raw, 'ep_ret': ep_ret, 'ep_cost': ep_cost,
                 'ep_len': ep_len}
        hook = getattr(self._env, 'state_dict', None)
        if callable(hook):
            state['env'] = hook()
        return state

    def load_train_state(self, state: dict) -> None:
        """Restores in place; the first epoch after it runs eagerly (graph-safe envs capture in the one after)."""
        load_episode_state(self, state)
        for k in ('s_raw', 'final_raw', 'ep_ret', 'ep_cost', 'ep_len'):
            restore(getattr(self, k), state[k], f'external-env adapter {k}')
        hook = getattr(self._env, 'load_state_dict', None)
        if 'env' in state and callable(hook):
            hook(state['env'])

    def close(self) -> None:
        self._env.close()
