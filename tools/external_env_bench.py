"""Throughput of the external-env path: the bench.py headline workload (PPOLag, 4096 envs x T = 128, obs 60 / act 8,
batch 16384, update_iters 8) on a PyTorch-on-GPU port of the synthetic dynamics registered as a user CMDP.

    python tools/external_env_bench.py [--steps K] [--warmup W] [--precision bf16x3|tf32|fp32] [--graph] [--algo NAME]

Every env step is one act launch, the env's own PyTorch kernels and one observe launch.  Prints ONE JSON line:
env-steps/s over full epochs (rollout + GAE + update, CUDA events), and one rollout split into the device time spent
inside env.step (CUDA events at its entry and exit) and the rest (act / observe kernels, episode window, launch gaps).
--graph runs the graph-safe TorchBox (same arithmetic, state written in place, no events inside step), whose epoch the
adapter replays from a CUDA graph; it reports env-steps/s and the rollout time per epoch only.  With OSB_NO_GRAPH=1 the
same env runs eagerly.  --algo picks the algorithm (default PPOLag); TorchBox has the optional reset_envs(mask) hook, so
PPOEarlyTerminated runs the cost-limit rule on all 4096 envs (graph-safe TorchBox: inside the replayed graph).  Logs go to
a temporary directory; nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

ENV_ID = 'TorchBox-v0'
GRAPH_ENV_ID = 'TorchBoxGraph-v0'
N, T, O, A, TMAX = 4096, 128, 60, 8, 64


def register_torch_box() -> None:
    """The synthetic dynamics (oracle/synthetic_env.py: hash resets, clipped linear step, reward 1 - mean s'^2, cost on
    s'_0, time-limit truncation; no hash terminations) in PyTorch.  step() records CUDA events around itself when
    `timing` is a list."""
    from omnisafe_b200.envs import CMDP, Box, env_register, is_registered

    if is_registered(ENV_ID):
        return
    M = 0xFFFFFFFF

    def mix(x):
        x = x ^ (x >> 16)
        x = (x * 0x7FEB352D) & M
        x = x ^ (x >> 15)
        x = (x * 0x846CA68B) & M
        return x ^ (x >> 16)

    class TorchBox(CMDP):
        _support_envs = [ENV_ID]  # noqa: RUF012
        need_auto_reset_wrapper = need_time_limit_wrapper = need_evaluation = False

        def __init__(self, env_id, num_envs=1, device='cuda', obs_dim=60, act_dim=8, max_episode_steps=64, **_):
            super().__init__(env_id)
            self._num_envs, dev = num_envs, torch.device(device)
            self._observation_space, self._action_space = Box(-10.0, 10.0, (obs_dim,)), Box(-1.0, 1.0, (act_dim,))
            self.tmax, self.seed, self.timing = max_episode_steps, 0, None
            self.j = torch.arange(obs_dim, device=dev)
            self.idx = self.j % act_dim
            self.bias = 0.02 * (((7 * self.j + 3) % 5) - 2).to(torch.float32)
            self.gid = torch.arange(num_envs, device=dev)
            self.episode = torch.zeros(num_envs, dtype=torch.int64, device=dev)
            self.ep_step = torch.zeros(num_envs, dtype=torch.int64, device=dev)
            self.s = torch.zeros(num_envs, obs_dim, device=dev)

        def _reset_values(self, episode):
            h = mix(self.seed ^ ((self.gid[:, None] * 0x9E3779B1) & M))
            h = mix(h ^ ((episode[:, None] * 0x85EBCA77) & M))
            h = mix(h ^ ((self.j[None, :] * 0xC2B2AE3D) & M))
            return (h >> 8).to(torch.float32) * (1.0 / 8388608.0) - 1.0

        def set_seed(self, seed):
            self.seed = int(seed) & M

        def reset(self, seed=None, options=None):
            self.episode += 1
            self.ep_step.zero_()
            self.s = self._reset_values(self.episode)
            return self.s, {}

        def step(self, action):
            ev = None
            if self.timing is not None:
                ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                ev[0].record()
            a = action.clamp(-1.0, 1.0)
            sn = (0.95 * self.s + 0.1 * a[:, self.idx] + self.bias).clamp(-10.0, 10.0)
            reward = 1.0 - (sn * sn).mean(1)
            cost = (sn[:, 0] > 0.0).to(torch.float32)
            trunc = (self.ep_step + 1) >= self.tmax
            term = torch.zeros_like(trunc)
            self.episode = torch.where(trunc, self.episode + 1, self.episode)
            self.s = torch.where(trunc[:, None], self._reset_values(self.episode), sn)
            self.ep_step = torch.where(trunc, torch.zeros_like(self.ep_step), self.ep_step + 1)
            info = {'final_observation': sn, '_final_observation': trunc}    # no host sync on "any env finished?"
            if ev is not None:
                ev[1].record()
                self.timing.append(ev)
            return self.s, reward, cost, term, trunc, info

        def reset_envs(self, mask):
            self.episode = torch.where(mask, self.episode + 1, self.episode)
            self.ep_step = torch.where(mask, torch.zeros_like(self.ep_step), self.ep_step)
            self.s = torch.where(mask[:, None], self._reset_values(self.episode), self.s)
            return self.s

        def close(self):
            pass

    class TorchBoxGraph(TorchBox):
        """TorchBox for CUDA-graph capture: the same arithmetic with the state updated in place."""
        _support_envs = [GRAPH_ENV_ID]  # noqa: RUF012
        graph_safe = True

        def __init__(self, env_id, num_envs=1, device='cuda', **kw):
            super().__init__(env_id, num_envs=num_envs, device=device, **kw)
            self._device = torch.device(device)

        def reset(self, seed=None, options=None):
            self.episode += 1
            self.ep_step.zero_()
            self.s.copy_(self._reset_values(self.episode))
            return self.s, {}

        def step(self, action):
            a = action.clamp(-1.0, 1.0)
            sn = (0.95 * self.s + 0.1 * a[:, self.idx] + self.bias).clamp(-10.0, 10.0)
            reward = 1.0 - (sn * sn).mean(1)
            cost = (sn[:, 0] > 0.0).to(torch.float32)
            trunc = (self.ep_step + 1) >= self.tmax
            term = torch.zeros_like(trunc)
            self.episode.copy_(torch.where(trunc, self.episode + 1, self.episode))
            self.s.copy_(torch.where(trunc[:, None], self._reset_values(self.episode), sn))
            self.ep_step.copy_(torch.where(trunc, torch.zeros_like(self.ep_step), self.ep_step + 1))
            return self.s, reward, cost, term, trunc, {'final_observation': sn, '_final_observation': trunc}

        def reset_envs(self, mask):
            self.episode.copy_(torch.where(mask, self.episode + 1, self.episode))
            self.ep_step.copy_(torch.where(mask, torch.zeros_like(self.ep_step), self.ep_step))
            self.s.copy_(torch.where(mask[:, None], self._reset_values(self.episode), self.s))
            return self.s

    env_register(TorchBox)
    env_register(TorchBoxGraph)


def timed(fn, k: int) -> float:
    """Device time of k calls of fn in ms (CUDA events, synchronised on both sides)."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(k):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def gpu_info() -> dict:
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i',
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=10).stdout
        name, power = (c.strip() for c in out.strip().split(','))
        return {'gpu': name, 'power_limit': power}
    except Exception:  # noqa: BLE001
        return {'gpu': torch.cuda.get_device_name(), 'power_limit': None}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--precision', default='bf16x3', choices=['bf16x3', 'tf32', 'fp32'])
    ap.add_argument('--graph', action='store_true', help='graph-safe TorchBox: the epoch is replayed from a CUDA graph')
    ap.add_argument('--algo', default='PPOLag', help='algorithm, e.g. PPOLag or PPOEarlyTerminated')
    args = ap.parse_args()
    import omnisafe_b200

    register_torch_box()
    env_id = GRAPH_ENV_ID if args.graph else ENV_ID
    spe = N * T
    cfg = {'seed': 0,
           'train_cfgs': {'device': 'cuda', 'vector_env_nums': N, 'parallel': 1,
                          'total_steps': spe * (args.steps + args.warmup + 8), 'matmul_precision': args.precision},
           'algo_cfgs': {'steps_per_epoch': spe, 'batch_size': 16384, 'update_iters': 8},
           'logger_cfgs': {'log_dir': tempfile.mkdtemp(prefix='osb_extbench_'), 'use_tensorboard': False,
                           'save_model_freq': 10 ** 9},
           'env_cfgs': {'obs_dim': O, 'act_dim': A, 'max_episode_steps': TMAX}}
    algo = omnisafe_b200.Agent(args.algo, env_id, custom_cfgs=cfg).agent
    for _ in range(max(args.warmup, 1)):
        algo.train_epoch()
    ms = timed(algo.train_epoch, args.steps) / args.steps
    env, k = algo._env.env, 3
    if not args.graph:
        env.timing = []
    ms_roll = timed(lambda: algo._env.rollout(algo._steps_per_epoch, algo._actor_critic, algo._buf, algo._logger), k) / k
    split = {}
    if not args.graph:
        ms_env = sum(a.elapsed_time(b) for a, b in env.timing) / k
        split = {'env_step_ms': ms_env, 'kernel_ms': ms_roll - ms_env}
    print(json.dumps({
        'metric': f'env-steps/sec (rollout+GAE+update) {args.algo}, {env_id} through the external-env path',
        'value': spe / (ms * 1e-3), 'unit': 'env-steps/s', 'ms_per_step': ms, 'steps': args.steps,
        'rollout_ms': ms_roll, **split, 'graph_mode': algo._env.graph_mode,
        'config': {'envs': N, 'steps_per_env': T, 'obs_dim': O, 'act_dim': A, 'batch_size': 16384, 'update_iters': 8,
                   'matmul_precision': args.precision, 'noise': 'in-kernel Philox'},
        **gpu_info()}), flush=True)


if __name__ == '__main__':
    main()
