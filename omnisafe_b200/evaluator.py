"""`Evaluator` -- score a saved policy: `load_saved(save_dir, model_name)` + `evaluate(num_episodes, cost_criteria)`.

Follows omnisafe/evaluator.py (load L134-303, on-policy branch; evaluate L399-490).  `load_saved` reads the run's
config.json and `torch_save/<model_name>`: the actor from 'pi' and, with `algo_cfgs.obs_normalize`, the observation
statistics from 'obs_normalizer'.  `evaluate` runs the episodes with the semantics of the reference loop, on the GPU in
the evaluation mode of the rollout step kernels (csrc/rollout.cu): the synthetic env entirely inside them
(osb_eval_synthetic), a registered env stepped in PyTorch between an act and an observe launch (osb_eval_ext_act /
osb_eval_ext_observe, one read of a 3-int counter per step):

- the env is built with the config's env_cfgs and its default seed (the evaluator does not call set_seed);
- every observation the env returns goes through ObsNormalize, which still pushes it into the loaded statistics, so they
  drift during the evaluation;
- the action is the mean (`predict(obs, deterministic=True)`), then ActionScale onto the env's box;
- return and cost are fp64 sums: ep_ret += reward, ep_cost += cost_criteria ** length * cost;
- Saute / Simmer runs: the network input ends with z, 1 at every episode start, z <- (z - cost / b) / saute_gamma with
  b the per-step budget of algo_cfgs.safety_budget; the reward is not replaced;
- EarlyTerminated runs: an episode also ends once ep_cost >= cost_limit.

One extension: `evaluate(num_envs=E)` runs E envs at once, env e playing episodes e, e + E, ...; results still come
back in episode order.  E changes the order in which rows reach the normaliser, and so the results: E = 1 (the default)
is the reference.  With E > 1 the envs reset themselves at their episode ends (an episode cut by the cost rule resets
its env on the synthetic env; on a registered env, which has no per-env reset, the cost rule needs E = 1), each step
pushes the rows of the envs still running, in env order.

The evaluator builds its own env state, normaliser and parameters; a live run's are never touched.
"""
from __future__ import annotations

import json
import os

import numpy as np
import torch

from omnisafe_b200._lib import OsbError, current_stream, lib, ptr
from omnisafe_b200.adapter.saute_adapter import per_step_budget
from omnisafe_b200.common.normalizer import Normalizer
from omnisafe_b200.envs.core import check_env, is_registered, make
from omnisafe_b200.envs.synthetic import SyntheticBoxEnv, support_envs
from omnisafe_b200.models.actor_critic import param_layout
from omnisafe_b200.utils.config import Config

PRECISIONS = {'fp32': 0, 'tf32': 1, 'bf16x3': 2}


class Evaluator:
    def __init__(self, device='cuda') -> None:
        self._device = torch.device(device)
        self._cfgs = None
        self._dividing_line = '\n' + '#' * 50 + '\n'
        self._per_step = False     # synthetic env: True forces one launch per step (tests compare the launch shapes)

    def load_saved(self, save_dir: str, model_name: str, render_mode: str = 'rgb_array', camera_name=None,
                   camera_id=None, width: int = 256, height: int = 256) -> None:
        """Load config.json and torch_save/<model_name> of a run directory.  The render arguments are accepted for
        signature parity and unused (rendering is not supported)."""
        with open(os.path.join(save_dir, 'config.json'), encoding='utf-8') as fh:
            cfgs = Config.dict2config(json.load(fh))
        self._synthetic = cfgs.env_id in support_envs()
        if not self._synthetic and not is_registered(cfgs.env_id):
            raise ValueError(f'{cfgs.env_id} is neither {support_envs()} nor a registered env (env_register)')
        try:
            params = torch.load(os.path.join(save_dir, 'torch_save', model_name), weights_only=False)
        except FileNotFoundError as error:
            raise FileNotFoundError('The model is not found in the save directory.') from error
        env_cfgs = getattr(cfgs, 'env_cfgs', None) or {}
        self._env_cfgs = dict(env_cfgs.todict() if hasattr(env_cfgs, 'todict') else env_cfgs)
        self._env_cfgs.pop('env_id_offset', None)
        self._cfgs = cfgs
        algo, a = str(cfgs.algo), cfgs.algo_cfgs
        self._saute = 'Saute' in algo or 'Simmer' in algo
        self._early = 'EarlyTerminated' in algo
        self._cost_limit = float(a.cost_limit) if self._early else 0.0
        self._budget = (per_step_budget(float(a.safety_budget), float(a.saute_gamma), float(a.max_ep_len))
                        if self._saute else 1.0)
        self._saute_gamma = float(a.saute_gamma) if self._saute else 1.0
        if self._synthetic:
            probe = SyntheticBoxEnv(cfgs.env_id, num_envs=1, device='cpu', **self._env_cfgs)
            self._obs_dim, self._act_dim = probe.obs_dim, probe.act_dim
        else:
            self._obs_dim, self._act_dim, _, _ = check_env(make(cfgs.env_id, num_envs=1, device=self._device,
                                                                **self._env_cfgs))
        On, A = self._obs_dim + int(self._saute), self._act_dim
        # the actor's flat parameters in the rollout's layout (the critics are not evaluated)
        layout = param_layout(On, A)
        theta = torch.zeros(layout['total'], dtype=torch.float32)
        for name, (off, shape) in layout['actor']['entries'].items():
            w = params['pi'][name]
            assert tuple(w.shape) == shape, f"'pi'.{name} has shape {tuple(w.shape)}, expected {shape}"
            theta[off:off + w.numel()] = w.reshape(-1).float()
        self._theta = theta.to(self._device)
        self._obs_normalize = bool(getattr(a, 'obs_normalize', True))
        self._norm_sd = params['obs_normalizer'] if self._obs_normalize else None
        prec = str(getattr(cfgs.train_cfgs, 'matmul_precision', 'bf16x3'))
        self._precision = PRECISIONS[prec]
        self.normalizer = None

    def evaluate(self, num_episodes: int = 10, cost_criteria: float = 1.0,
                 num_envs: int = 1) -> tuple[list[float], list[float]]:
        """Run `num_episodes` episodes; returns (episode_rewards, episode_costs).  `num_envs` envs run at once
        (at most num_episodes); the default 1 is the reference's loop.  The drifted normaliser is left in
        `self.normalizer`, the episode lengths in `self.episode_lengths`, each env's action in the last step it ran in
        `self.last_actions`."""
        if self._cfgs is None:
            raise ValueError('The environment and the policy must be provided or created before evaluating the agent.')
        num_episodes = int(num_episodes)
        assert num_episodes >= 1 and num_envs >= 1, 'num_episodes and num_envs must be positive'
        E, O, dev = min(int(num_envs), num_episodes), self._obs_dim, self._device
        if not self._synthetic and self._early and E > 1:
            raise NotImplementedError('the EarlyTerminated rule on a registered env needs num_envs=1: the env cannot be '
                                      'reset on its own when the cost rule cuts an episode')
        norm = Normalizer((O,), clip=5.0, device=dev)
        if self._norm_sd is not None:
            norm.load_state_dict(self._norm_sd)
        i32 = lambda n: torch.zeros(n, dtype=torch.int32, device=dev)      # noqa: E731
        f64 = lambda n: torch.zeros(n, dtype=torch.float64, device=dev)    # noqa: E731
        w = {'left': torch.tensor([(num_episodes - e + E - 1) // E for e in range(E)], dtype=torch.int32, device=dev),
             'done_eps': i32(E), 'len': i32(E), 'ret': f64(E), 'cost': f64(E),
             'ctr': torch.tensor([E, 0, 0], dtype=torch.int32, device=dev),
             'out_ret': f64(num_episodes), 'out_cost': f64(num_episodes), 'out_len': i32(num_episodes),
             'act_out': torch.zeros(E, self._act_dim, dtype=torch.float32, device=dev),
             'safety': torch.ones(2, E, dtype=torch.float32, device=dev) if self._saute else None}
        with torch.cuda.device(dev):
            if self._synthetic:
                self._run_synthetic(E, num_episodes, float(cost_criteria), norm, w)
            else:
                self._run_registered(E, float(cost_criteria), norm, w)
        out_ret, out_cost, out_len = w['out_ret'], w['out_cost'], w['out_len']
        self.last_actions = w['act_out']
        episode_rewards = [float(x) for x in out_ret.cpu().numpy()]
        episode_costs = [float(x) for x in out_cost.cpu().numpy()]
        episode_lengths = [float(x) for x in out_len.cpu().numpy()]
        self.normalizer, self.episode_lengths = norm, episode_lengths
        for k in range(num_episodes):
            print(f'Episode {k} results:')
            print(f'Episode reward: {episode_rewards[k]}')
            print(f'Episode cost: {episode_costs[k]}')
            print(f'Episode length: {episode_lengths[k]}')
        print(self._dividing_line)
        print('Evaluation results:')
        print(f'Average episode reward: {np.mean(a=episode_rewards)}')
        print(f'Average episode cost: {np.mean(a=episode_costs)}')
        print(f'Average episode length: {np.mean(a=episode_lengths)}')
        return episode_rewards, episode_costs

    def _run_synthetic(self, E, num_episodes, crit, norm, w) -> None:
        O, dev = self._obs_dim, self._device
        env = SyntheticBoxEnv(self._cfgs.env_id, num_envs=E, device=dev, **self._env_cfgs)
        acc_rst = torch.zeros(2, O, dtype=torch.int64, device=dev)
        lib().osb_eval_synthetic(
            O, self._act_dim, env.max_episode_steps, env.seed, env.term_threshold, env.cost_threshold,
            int(self._obs_normalize), E, num_episodes, *env.state_ptrs(), *norm.ptrs(),
            ptr(w['safety']), self._budget, self._saute_gamma, int(self._early), self._cost_limit, crit,
            ptr(w['left']), ptr(w['done_eps']), ptr(w['ret']), ptr(w['cost']), ptr(w['len']), ptr(acc_rst),
            ptr(w['ctr']), ptr(w['out_ret']), ptr(w['out_cost']), ptr(w['out_len']), ptr(w['act_out']),
            ptr(self._theta), self._precision, int(self._per_step), current_stream())

    def _run_registered(self, E, crit, norm, w) -> None:
        """env.reset() -> ingest; then per step: act launch -> env.step -> observe launch -> read the counters (done
        word, resets asked for); E = 1 resets the env after every episode that another one follows."""
        O, A, dev, L = self._obs_dim, self._act_dim, self._device, lib()
        env = make(self._cfgs.env_id, num_envs=E, device=dev, **self._env_cfgs)   # the env's default seed
        _, _, lo, hi = check_env(env)
        act_lo, act_hi = torch.as_tensor(lo).to(dev), torch.as_tensor(hi).to(dev)
        s_raw = torch.zeros(2, E, O, dtype=torch.float32, device=dev)
        act_env = torch.zeros(E, A, dtype=torch.float32, device=dev)
        ws = torch.zeros(L.osb_eval_ext_workspace_doubles(O, E), dtype=torch.float64, device=dev)
        nonfinite = torch.zeros(1, dtype=torch.int32, device=dev)
        rows = lambda x, width=None, dtype=torch.float32: torch.as_tensor(x).to(            # noqa: E731
            device=dev, dtype=dtype).reshape((E,) if width is None else (E, width)).contiguous()
        on, s = int(self._obs_normalize), current_stream()
        tail = (ptr(s_raw), ptr(norm.mean), ptr(norm.sumsq), ptr(norm.std), ptr(norm.count), ptr(norm.ticket),
                ptr(w['safety']), self._budget, self._saute_gamma, int(self._early), self._cost_limit, crit,
                ptr(w['left']), ptr(w['done_eps']), ptr(w['ret']), ptr(w['cost']), ptr(w['len']), ptr(w['ctr']),
                ptr(w['out_ret']), ptr(w['out_cost']), ptr(w['out_len']), ptr(ws), ptr(nonfinite), s)

        def ingest(t):
            obs = rows(env.reset()[0], O)
            L.osb_eval_ext_observe(O, E, t, on, 1, ptr(obs), 0, 0, 0, 0, 0, 0, *tail)

        ingest(-1)
        t = 0
        while True:
            L.osb_eval_ext_act(O, A, on, E, t, ptr(s_raw), ptr(norm.mean), ptr(norm.std), ptr(norm.count),
                               ptr(w['safety']), ptr(self._theta), ptr(act_lo), ptr(act_hi), ptr(act_env), ptr(w['left']),
                               ptr(w['ctr']), ptr(w['act_out']), self._precision, s)
            action = act_env.clone()
            nobs, rew, cost, term, trunc, info = env.step(action[0] if E == 1 else action)
            nobs, rew, cost = rows(nobs, O), rows(rew), rows(cost)
            term, trunc = rows(term, dtype=torch.uint8), rows(trunc, dtype=torch.uint8)
            final = mask = None
            if 'final_observation' in info:
                final = rows(info['final_observation'], O)
                mask = info.get('_final_observation')
                mask = (term | trunc) if mask is None else rows(mask, dtype=torch.uint8)
            L.osb_eval_ext_observe(O, E, t, on, 0, ptr(nobs), ptr(rew), ptr(cost), ptr(term), ptr(trunc), ptr(final),
                                   ptr(mask), *tail)
            running, _, resets = (int(x) for x in w['ctr'].cpu())
            if running == 0:
                break
            if resets:
                ingest(t)
            t += 1
        if int(nonfinite.item()):
            raise OsbError(f'{self._cfgs.env_id} returned a non-finite observation during the evaluation')

    def render(self, *_, **__):
        raise NotImplementedError('rendering is not supported')
