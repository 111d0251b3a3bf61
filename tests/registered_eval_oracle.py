"""Oracle of `Evaluator.evaluate` on a registered env (numpy / torch-CPU restatement), including the EarlyTerminated rule
at E > 1 through the env's `reset_envs(mask)` hook.

The loop of oracle/evaluator.py::evaluate with the env behind the numpy interface of oracle/synthetic_env.py
(`reset() -> obs`, `step(action) -> (obs, reward, cost, terminated, truncated, final_obs, finished)`) plus
`reset_envs(mask) -> obs` and the env's action box (`act_lo`, `act_hi`).  Per step, over the envs still running,
ObsNormalize pushes the final observations of envs whose env episode ended, then the next observations of all of them,
then the reset rows: E = 1 calls env.reset() after every episode that another one follows (the reference loop); E > 1
calls env.reset_envs(mask) for the envs the cost rule cut while the env was still running and that have episodes left,
and pushes exactly those rows as the step's third batch.
"""
from __future__ import annotations

import numpy as np

from oracle.evaluator import _normalized, actor_mean, load_normalizer
from oracle.rollout import action_scale

F32 = np.float32


def evaluate(env, pi: dict, norm_sd: dict | None, num_episodes: int, cost_criteria: float = 1.0,
             saute: tuple[float, float] | None = None, cost_limit: float | None = None, actor=actor_mean):
    """Returns (returns, costs, lengths, normalizer, cut) with `cut` the number of episodes the cost rule ended while
    the env was still running.  E = env.N envs, env e playing episodes e, e + E, ..."""
    E = int(env.N)
    norm = load_normalizer(norm_sd) if norm_sd is not None else None
    push = (lambda rows: norm.push(rows) if len(rows) else None) if norm is not None else (lambda rows: None)
    left = np.array([(num_episodes - e + E - 1) // E for e in range(E)])
    done_eps = np.zeros(E, np.int64)
    ret, cost, length = np.zeros(E), np.zeros(E), np.zeros(E, np.int64)
    z = np.ones(E, F32)
    out_ret, out_cost, out_len = np.zeros(num_episodes), np.zeros(num_episodes), np.zeros(num_episodes, np.int64)
    lo, hi = getattr(env, 'act_lo', -1.0), getattr(env, 'act_hi', 1.0)
    n_cut = 0
    s = np.asarray(env.reset(), F32).reshape(E, -1)
    push(s)
    while (left > 0).any():
        run = left > 0
        x = _normalized(norm, s)
        if saute is not None:
            x = np.concatenate([x, z[:, None]], 1)
        act = actor(pi, x).astype(F32)
        nobs, rew, cst, term, trunc, final, fin = env.step(action_scale(act, lo, hi))
        fin = np.asarray(fin, bool)
        push(final[run & fin])
        push(nobs[run])
        s = np.array(nobs, F32)
        r = np.flatnonzero(run)
        ret[r] += rew[r].astype(np.float64)
        cost[r] += np.array([cost_criteria ** float(n) for n in length[r]]) * cst[r].astype(np.float64)
        length[r] += 1
        if saute is not None:
            z[r] = ((z[r] - (cst[r] / F32(saute[0])).astype(F32)).astype(F32) / F32(saute[1])).astype(F32)
        done = np.zeros(E, bool)
        done[r] = fin[r] | ((cost[r] >= cost_limit) if cost_limit is not None else False)
        d = np.flatnonzero(done)
        k = d + done_eps[d] * E
        out_ret[k], out_cost[k], out_len[k] = ret[d], cost[d], length[d]
        n_cut += int((done & ~fin).sum())
        done_eps[d] += 1
        left[d] -= 1
        ret[d] = cost[d] = 0.0
        length[d] = 0
        z[d] = F32(1)
        reset = done & (left > 0) & ((E == 1) | ~fin)
        if reset.any():
            obs = np.asarray(env.reset() if E == 1 else env.reset_envs(reset), F32).reshape(E, -1)
            s[reset] = obs[reset]
            push(obs[reset])
    return out_ret, out_cost, out_len, norm, n_cut
