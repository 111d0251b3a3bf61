"""Oracle of `omnisafe_b200.Evaluator.evaluate` on the synthetic env (numpy / torch-CPU restatement).

The reference Evaluator (omnisafe/evaluator.py:L399-490) with the synthetic env of oracle/synthetic_env.py, extended
to E envs as omnisafe_b200/evaluator.py describes; E = 1 is the reference loop.  Per step, over the envs still running:
ObsNormalize pushes the final observations of envs whose env episode ended, then the next observations of all of them,
then the observations of envs reset after the step (E = 1: every env whose episode ended and that has episodes left;
E > 1: only those cut by the cost rule).  TEST INFRASTRUCTURE ONLY (see oracle/__init__.py); imported by tests/test_evaluate_cpu.py and tests/test_evaluate_gpu.py.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle.normalizer import Normalizer
from oracle.synthetic_env import SyntheticBoxEnv, u32_to_unit, hash4

F32 = np.float32
U32 = np.uint32


def actor_mean(pi: dict, x: np.ndarray) -> np.ndarray:
    """GaussianLearningActor.mean in torch fp32 on the CPU: Linear-Tanh-Linear-Tanh-Linear."""
    t = lambda k: torch.as_tensor(np.asarray(pi[k]), dtype=torch.float32)    # noqa: E731
    h = torch.as_tensor(x, dtype=torch.float32)
    h = torch.tanh(torch.nn.functional.linear(h, t('mean.0.weight'), t('mean.0.bias')))
    h = torch.tanh(torch.nn.functional.linear(h, t('mean.2.weight'), t('mean.2.bias')))
    return torch.nn.functional.linear(h, t('mean.4.weight'), t('mean.4.bias')).numpy()


def _normalized(norm: Normalizer, x: np.ndarray) -> np.ndarray:
    if norm is None or norm.count <= 1:
        return x.astype(F32)
    return np.clip(((x - norm.mean) / norm.std).astype(F32), -norm.clip, norm.clip).astype(F32)


def load_normalizer(sd: dict) -> Normalizer:
    n = Normalizer(np.asarray(sd['_mean']).shape)
    n.mean = np.asarray(sd['_mean'], F32).copy()
    n.sumsq = np.asarray(sd['_sumsq'], F32).copy()
    n.std = np.asarray(sd['_std'], F32).copy()
    n.count = int(sd['_count'])
    return n


def evaluate(pi: dict, norm_sd: dict | None, env_kw: dict, num_episodes: int, cost_criteria: float = 1.0,
             num_envs: int = 1, saute: tuple[float, float] | None = None, cost_limit: float | None = None,
             actor=actor_mean):
    """Returns (returns, costs, lengths, normalizer).  saute = (per-step budget, saute_gamma); cost_limit: the
    EarlyTerminated rule; actor(pi, rows) -> means."""
    E = min(int(num_envs), int(num_episodes))
    env = SyntheticBoxEnv(E, seed=0, **env_kw)
    norm = load_normalizer(norm_sd) if norm_sd is not None else None
    push = (lambda rows: norm.push(rows) if len(rows) else None) if norm is not None else (lambda rows: None)
    left = np.array([(num_episodes - e + E - 1) // E for e in range(E)])
    done_eps = np.zeros(E, np.int64)
    ret, cost, length = np.zeros(E), np.zeros(E), np.zeros(E, np.int64)
    z = np.ones(E, F32)
    out_ret, out_cost, out_len = np.zeros(num_episodes), np.zeros(num_episodes), np.zeros(num_episodes, np.int64)
    push(env.reset())
    while (left > 0).any():
        run = left > 0
        x = _normalized(norm, env.s)
        if saute is not None:
            x = np.concatenate([x, z[:, None]], 1)
        act = actor(pi, x).astype(F32)
        act = ((act + F32(1)).astype(F32) - F32(1)).astype(F32)      # ActionScale onto the env's [-1, 1] box
        nobs, rew, cst, term, trunc, final, fin = env.step(act)
        push(final[run & fin])
        push(nobs[run])
        reset_rows = []
        for e in np.flatnonzero(run):
            ret[e] += float(rew[e])
            cost[e] += (cost_criteria ** float(length[e])) * float(cst[e])
            length[e] += 1
            if saute is not None:
                z[e] = F32(F32(z[e] - F32(cst[e] / F32(saute[0]))) / F32(saute[1]))
            done = bool(fin[e]) or (cost_limit is not None and cost[e] >= cost_limit)
            if not done:
                continue
            k = e + done_eps[e] * E
            out_ret[k], out_cost[k], out_len[k] = ret[e], cost[e], length[e]
            done_eps[e] += 1
            left[e] -= 1
            ret[e] = cost[e] = 0.0
            length[e] = 0
            z[e] = F32(1)
            if left[e] > 0 and (E == 1 or not fin[e]):       # env.reset() of this env
                with np.errstate(over='ignore'):
                    env.episode[e] = U32(env.episode[e] + U32(1))
                env.ep_step[e] = 0
                j = np.arange(env.O, dtype=U32)
                env.s[e] = u32_to_unit(hash4(U32(env.seed), env.gid[e], env.episode[e], j))
                reset_rows.append(env.s[e].copy())
        if reset_rows:
            push(np.stack(reset_rows))
    return out_ret, out_cost, out_len, norm
