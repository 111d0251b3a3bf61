"""Oracle: one epoch of the on-policy rollout on a user env behind TimeLimit and AutoReset, for any number of envs
(numpy + torch-CPU).  TEST INFRASTRUCTURE ONLY.

OnPolicyAdapter.rollout (adapter/onpolicy_adapter.py:L58-136) over the reference's wrapper chain (online_adapter.py:
L120-131): env -> TimeLimit -> AutoReset -> ObsNormalize, with one TimeLimit counter and one AutoReset per env.  After
env.step: steps += 1; with a time limit, truncated = steps >= time_limit (the env's own flag is discarded), else the
env's flag; done = terminated | truncated; steps = 0 where done (AutoReset's reset goes through TimeLimit.reset); the done
envs are reset (env.reset_envs(done)) and their step rows become the final observations.  ObsNormalize pushes B = the
final rows (normalised with the statistics after B), then A = every env's next row, the reset row for a done env.  The
epoch-start reset clears every counter.  With one env this is the reference's call sequence.
"""
from __future__ import annotations

import numpy as np

from oracle import actor_critic as ac
from oracle.gae import FLAG_TERMINATED, FLAG_TRUNCATED
from oracle.rollout import action_scale

F32 = np.float32


def rollout_epoch_wrapped(env, norm, theta, T, eps, time_limit, act_lo, act_hi, obs_normalize=True, window=None):
    """`env`: reset() -> [N, O], step(action) -> (obs, reward, cost, terminated, truncated) without any reset,
    reset_envs(mask) -> [N, O] (numpy).  time_limit: TimeLimit's limit, 0 for AutoReset alone.  Returns the time-major
    slabs of oracle/rollout.py, plus 'done' ([T, N] bool, the envs reset after each step)."""
    N, O, A = env.N, env.O, env.A
    sl = {
        'obs': np.zeros((T, N, O), F32), 'act': np.zeros((T, N, A), F32),
        'logp': np.zeros((T, N), F32), 'rew': np.zeros((T, N), F32), 'cost': np.zeros((T, N), F32),
        'val_r': np.zeros((T, N), F32), 'val_c': np.zeros((T, N), F32),
        'boot_r': np.zeros((T, N), F32), 'boot_c': np.zeros((T, N), F32),
        'flags': np.zeros((T, N), np.uint8), 'done': np.zeros((T, N), bool),
    }
    ep_ret = np.zeros(N, F32); ep_cost = np.zeros(N, F32); ep_len = np.zeros(N, F32)
    steps = np.zeros(N, np.int64)
    raw = env.reset()
    obs = norm.normalize(raw) if obs_normalize else raw
    for t in range(T):
        act, v_r, v_c, logp = ac.step(theta, obs, eps[t], O, A)
        sraw, rew, cost, term, trunc = env.step(action_scale(act, act_lo, act_hi))
        steps += 1
        if time_limit:
            trunc = steps >= time_limit
        done = term | trunc
        steps[done] = 0
        nraw = np.array(sraw, F32)
        final_norm = np.zeros((N, O), F32)
        if done.any():
            nraw[done] = env.reset_envs(done)[done]
            final_norm[done] = norm.normalize(sraw[done]) if obs_normalize else sraw[done]     # B
        nobs = norm.normalize(nraw) if obs_normalize else nraw                                   # A
        ep_ret = (ep_ret + rew).astype(F32); ep_cost = (ep_cost + cost).astype(F32); ep_len += 1
        sl['obs'][t] = obs; sl['act'][t] = act; sl['logp'][t] = logp
        sl['rew'][t] = rew; sl['cost'][t] = cost; sl['val_r'][t] = v_r; sl['val_c'][t] = v_c
        sl['flags'][t] = term.astype(np.uint8) * FLAG_TERMINATED + trunc.astype(np.uint8) * FLAG_TRUNCATED
        sl['done'][t] = done
        obs = nobs
        need_final = trunc & ~term
        need_next = (~term) & (~trunc) & (t == T - 1)
        if need_final.any():
            br, bc = ac.values(theta, final_norm, O, A)
            sl['boot_r'][t][need_final] = br[need_final]; sl['boot_c'][t][need_final] = bc[need_final]
        if need_next.any():
            br, bc = ac.values(theta, obs, O, A)
            sl['boot_r'][t][need_next] = br[need_next]; sl['boot_c'][t][need_next] = bc[need_next]
        for i in np.nonzero(done)[0]:
            if window is not None:
                window.append((float(ep_ret[i]), float(ep_cost[i]), float(ep_len[i])))
        ep_ret[done] = 0; ep_cost[done] = 0; ep_len[done] = 0
    return sl
