"""`Evaluator` -- score a saved policy: `load_saved(save_dir, model_name)` + `evaluate(num_episodes, cost_criteria)`.

Follows omnisafe/evaluator.py (load L134-303, on-policy branch; evaluate L399-490).  `load_saved` reads the run's
config.json and `torch_save/<model_name>`: the actor from 'pi' and, with `algo_cfgs.obs_normalize`, the observation
statistics from 'obs_normalizer'.  `evaluate` runs the episodes with the semantics of the reference loop, on the GPU in
the evaluation mode of the rollout step kernels (csrc/rollout.cu): the synthetic env entirely inside them
(osb_eval_synthetic), a registered env stepped in PyTorch between an act and an observe launch (osb_eval_ext_act /
osb_eval_ext_observe, one read of a 3-int counter per step; a graph-safe env at E > 1 replays blocks of 16 steps from
a CUDA graph and reads the 4-byte done word once per block, OSB_NO_GRAPH=1 keeps it eager):

- the env is built with the config's env_cfgs and its default seed (the evaluator does not call set_seed);
- every observation the env returns goes through ObsNormalize, which still pushes it into the loaded statistics, so they
  drift during the evaluation;
- the action is the mean (`predict(obs, deterministic=True)`), then ActionScale onto the env's box;
- return and cost are fp64 sums: ep_ret += reward, ep_cost += cost_criteria ** length * cost;
- Saute / Simmer runs: the network input ends with z, 1 at every episode start, z <- (z - cost / b) / saute_gamma with
  b the per-step budget of algo_cfgs.safety_budget; the reward is not replaced;
- EarlyTerminated runs: an episode also ends once ep_cost >= cost_limit;
- an env that declares need_time_limit_wrapper is truncated after 1000 steps, its own truncation discarded
  (TimeLimit(time_limit=1000), evaluator.py:L179-180); AutoReset is never applied, so such an env, like one that
  declares need_auto_reset_wrapper, does not reset itself and every episode end is reset by the evaluation.

One extension: `evaluate(num_envs=E)` runs E envs at once, env e playing episodes e, e + E, ...; results still come
back in episode order.  E changes the order in which rows reach the normaliser, and so the results: E = 1 (the default)
is the reference.  With E > 1 the envs reset themselves at their episode ends, and an episode cut by the cost rule
resets its env: on the synthetic env inside the kernels, on a registered env through its optional `reset_envs(mask)`
hook (envs/core.py; without it the cost rule needs E = 1).  Each step pushes the rows of the envs still running, in env
order, then the reset rows of the envs the rule cut that have episodes left.  An env that declares either wrapper
resets every finished env with episodes left through `reset_envs(mask)` (osb_eval_ext_observe_wrapped), so at E > 1 it
needs the hook.

The evaluator builds its own env state, normaliser and parameters; a live run's are never touched.
"""
from __future__ import annotations

import json
import os

import numpy as np
import torch

from omnisafe_b200._lib import OsbError, current_stream, lib, ptr
from omnisafe_b200.adapter.external_adapter import device_rows, step_rows
from omnisafe_b200.adapter.saute_adapter import per_step_budget
from omnisafe_b200.common.normalizer import Normalizer
from omnisafe_b200.envs.core import check_env, is_registered, make, needs_wrappers
from omnisafe_b200.envs.synthetic import SyntheticBoxEnv, support_envs
from omnisafe_b200.models.actor_critic import HID, ParamMap, activation_code, set_net_spec
from omnisafe_b200.utils.config import Config

PRECISIONS = {'fp32': 0, 'tf32': 1, 'bf16x3': 2}
TIME_LIMIT = 1000   # the TimeLimit the reference's evaluator applies (evaluator.py:L179-180)
GRAPH_BLOCK = 16    # steps per captured block of a graph-safe registered env (even: t enters only by its parity)


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
            probe = make(cfgs.env_id, num_envs=1, device=self._device, **self._env_cfgs)
            self._obs_dim, self._act_dim, _, _ = check_env(probe, wrappers=True)
            self._reset_envs = callable(getattr(probe, 'reset_envs', None))
            self._wrapped = needs_wrappers(probe)
            self._time_limit = TIME_LIMIT if getattr(probe, 'need_time_limit_wrapper', False) else 0
        On, A = self._obs_dim + int(self._saute), self._act_dim
        # the actor's flat parameters in the kernel layout, zero-padded to width 64 (the critics are not evaluated)
        actor_cfgs = getattr(getattr(cfgs, 'model_cfgs', None), 'actor', None)
        pmap = ParamMap(On, A, actor_hidden=getattr(actor_cfgs, 'hidden_sizes', [HID, HID]))
        # the actor's hidden activation, as upstream's evaluator builds its actor from config.json (evaluator.py:L292-299)
        self._actor_act = activation_code(getattr(actor_cfgs, 'activation', 'tanh'), 'actor')
        self._actor_hidden = pmap.actor_hidden
        theta = torch.zeros(pmap.kernel['total'], dtype=torch.float32)
        pmap.load_state_dict(theta, 'actor', params['pi'], what="'pi'")
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
        if not self._synthetic and self._early and E > 1 and not self._reset_envs:
            raise NotImplementedError(
                f'evaluating EarlyTerminated on {self._cfgs.env_id} with {E} envs needs the optional reset_envs(mask) '
                'hook (envs/core.py) to reset the envs the cost limit cuts; without it only num_envs=1 is supported')
        if not self._synthetic and self._wrapped and E > 1 and not self._reset_envs:
            raise NotImplementedError(
                f'evaluating {self._cfgs.env_id} with {E} envs needs the optional reset_envs(mask) hook (envs/core.py): '
                'the env declares need_time_limit_wrapper / need_auto_reset_wrapper, so it does not reset itself and '
                'the finished envs are reset through the hook; without it only num_envs=1 is supported')
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
        set_net_spec(self._actor_act, 0, self._actor_hidden, (HID, HID))
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
        """env.reset() -> ingest; then per step: act launch -> env.step -> observe launch.  Eagerly, the counters (done
        word, resets asked for) are read after every step, and E = 1 resets the env after every episode that another one
        follows.  With the cost rule at E > 1 the observe launch also writes the mask of the envs it cut, which
        env.reset_envs(mask) resets and osb_ext_reset_rows ingests, with no host synchronisation.  A graph-safe env at
        E > 1 runs one eager block of GRAPH_BLOCK steps, then replays the next block, captured into a CUDA graph, until
        the done word (read once per block) is 0: steps after the last episode ended change nothing but the env."""
        O, A, dev, L = self._obs_dim, self._act_dim, self._device, lib()
        env = make(self._cfgs.env_id, num_envs=E, device=dev, **self._env_cfgs)   # the env's default seed
        _, _, lo, hi = check_env(env, wrappers=True)
        act_lo, act_hi = torch.as_tensor(lo).to(dev), torch.as_tensor(hi).to(dev)
        s_raw = torch.zeros(2, E, O, dtype=torch.float32, device=dev)
        act_env = torch.zeros(E, A, dtype=torch.float32, device=dev)
        ws = torch.zeros(L.osb_eval_ext_workspace_doubles(O, E), dtype=torch.float64, device=dev)
        nonfinite = torch.zeros(1, dtype=torch.int32, device=dev)
        wrapped = self._wrapped
        # envs the cost rule cuts (and behind the wrappers every finished env) are reset through env.reset_envs(rst)
        cut = (self._early or wrapped) and E > 1
        rst = torch.zeros(E, dtype=torch.bool, device=dev) if cut or wrapped else None
        tl_steps = torch.zeros(E, dtype=torch.int32, device=dev) if wrapped else None   # TimeLimit's _time, per env
        graph = E > 1 and bool(getattr(env, 'graph_safe', False)) and not os.getenv('OSB_NO_GRAPH')
        on = int(self._obs_normalize)
        tail = (ptr(s_raw), ptr(norm.mean), ptr(norm.sumsq), ptr(norm.std), ptr(norm.count), ptr(norm.ticket),
                ptr(w['safety']), self._budget, self._saute_gamma, int(self._early), self._cost_limit, crit,
                ptr(w['left']), ptr(w['done_eps']), ptr(w['ret']), ptr(w['cost']), ptr(w['len']), ptr(w['ctr']),
                ptr(w['out_ret']), ptr(w['out_cost']), ptr(w['out_len']), ptr(ws), ptr(nonfinite))

        def ingest(t):
            obs = env.reset()[0]
            L.osb_eval_ext_observe(O, E, t, on, 1, ptr(device_rows(obs, E, dev, O)), 0, 0, 0, 0, 0, 0, *tail,
                                   current_stream())
            return torch.as_tensor(obs).device

        def step(t, capture=False):
            s = current_stream()
            L.osb_eval_ext_act(O, A, on, E, t, ptr(s_raw), ptr(norm.mean), ptr(norm.std), ptr(norm.count),
                               ptr(w['safety']), ptr(self._theta), ptr(act_lo), ptr(act_hi), ptr(act_env), ptr(w['left']),
                               ptr(w['ctr']), ptr(w['act_out']), self._precision, s)
            action = act_env.clone()
            rows = step_rows(env, action[0] if E == 1 else action, E, O, dev, capture, finals=not wrapped)
            step_ptrs = tuple(ptr(r) for r in rows)
            if wrapped:
                L.osb_eval_ext_observe_wrapped(O, E, t, on, *step_ptrs[:5], *tail, ptr(rst), ptr(tl_steps),
                                               self._time_limit, s)
            elif cut:
                L.osb_eval_ext_observe_rst(O, E, t, on, *step_ptrs, *tail, ptr(rst), s)
            else:
                L.osb_eval_ext_observe(O, E, t, on, 0, *step_ptrs, *tail, s)
            if not cut:
                return
            obs = device_rows(env.reset_envs(rst.to(env_dev)), E, dev, O)
            L.osb_ext_reset_rows(O, E, t, on, ptr(rst), ptr(obs), ptr(s_raw), ptr(norm.mean), ptr(norm.sumsq),
                                 ptr(norm.std), ptr(norm.count), ptr(norm.ticket), ptr(ws), ptr(nonfinite), s)

        env_dev = ingest(-1)
        if graph:
            if env_dev.type != 'cuda':
                raise ValueError(f'{type(env).__name__} declares graph_safe but reset() returned observations on '
                                 f'{env_dev}')
            done_host = torch.zeros(1, dtype=torch.int32).pin_memory()

            def finished():
                done_host.copy_(w['ctr'][:1], non_blocking=True)
                torch.cuda.current_stream().synchronize()
                return int(done_host[0]) == 0

            # t reaches the kernels only through its parity: a block captured at an even t replays at every even t
            for t in range(GRAPH_BLOCK):
                step(t)
            if not finished():
                L.osb_eval_ext_prepare(O + int(self._saute), A, E, self._precision)
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    for t in range(GRAPH_BLOCK, 2 * GRAPH_BLOCK):
                        step(t, capture=True)
                while True:
                    g.replay()
                    if finished():
                        break
        else:
            t = 0
            while True:
                step(t)
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
