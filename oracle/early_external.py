"""Oracle: one epoch of the EarlyTerminated rollout on a user env stepped in PyTorch, for any number of envs (numpy +
torch-CPU).  TEST INFRASTRUCTURE ONLY.

EarlyTerminatedAdapter.step (adapter/early_terminated_adapter.py:L77-87) per env on top of OnPolicyAdapter.rollout
(adapter/onpolicy_adapter.py:L58-136), with ObsNormalize inside the env.  After env.step: acc += cost (fp32); where
acc > cost_limit the stored reward and the episode return take 0, terminated = 1, truncated stays as the env reported
it, the env is reset (env.reset_envs(mask)) and acc = 0.  Ordinary episode ends leave acc alone.  ObsNormalize pushes
B1 = the final observations of the envs that ended by themselves (they are normalised with the statistics after B1),
B2 = every env's next observation as env.step returned it, B3 = the reset observations of the cut envs.  The next step's
observations are normalised with the statistics after B3.  With one env this is the reference's call sequence.

The fused synthetic path (oracle/rollout.py, `early=`) orders the pushes differently when N > 1: it pushes the pre-reset
state of a cut env that did not end with the final rows, and never pushes the auto-reset row of an env that ended and
was cut in the same step.
"""
from __future__ import annotations

import numpy as np

from oracle import actor_critic as ac
from oracle.gae import FLAG_TERMINATED, FLAG_TRUNCATED
from oracle.rollout import action_scale

F32 = np.float32


def _apply(norm, x):
    """Normalizer.normalize without the push."""
    if norm.count <= 1:
        return np.asarray(x, F32)
    return np.clip(((x - norm.mean) / norm.std).astype(F32), -norm.clip, norm.clip).astype(F32)


def rollout_epoch_early(env, norm, theta, T, eps, early, act_lo, act_hi, obs_normalize=True, window=None):
    """`env`: reset() -> [N, O], step(action) -> (next obs, reward, cost, terminated, truncated, final obs, finished),
    reset_envs(mask) -> [N, O] (numpy).  `early` = {'cost_limit': c, 'acc': float32 [N]} is updated in place; it also
    receives 'trig' ([T, N] bool, the steps the rule cut).  Returns the time-major slabs of oracle/rollout.py."""
    N, O, A = env.N, env.O, env.A
    sl = {
        'obs': np.zeros((T, N, O), F32), 'act': np.zeros((T, N, A), F32),
        'logp': np.zeros((T, N), F32), 'rew': np.zeros((T, N), F32), 'cost': np.zeros((T, N), F32),
        'val_r': np.zeros((T, N), F32), 'val_c': np.zeros((T, N), F32),
        'boot_r': np.zeros((T, N), F32), 'boot_c': np.zeros((T, N), F32),
        'flags': np.zeros((T, N), np.uint8),
    }
    early['trig'] = np.zeros((T, N), bool)
    ep_ret = np.zeros(N, F32); ep_cost = np.zeros(N, F32); ep_len = np.zeros(N, F32)
    raw = env.reset()
    obs = norm.normalize(raw) if obs_normalize else raw
    for t in range(T):
        act, v_r, v_c, logp = ac.step(theta, obs, eps[t], O, A)
        nraw, rew, cost, term, trunc, final_raw, fin = env.step(action_scale(act, act_lo, act_hi))
        early['acc'] = (early['acc'] + cost).astype(F32)
        hit = early['acc'] > F32(early['cost_limit'])
        early['acc'] = np.where(hit, F32(0), early['acc']).astype(F32)
        early['trig'][t] = hit
        rew = np.where(hit, F32(0), rew).astype(F32)
        term = term | hit
        final_norm = np.zeros((N, O), F32)
        if fin.any():                                                   # B1
            final_norm[fin] = norm.normalize(final_raw[fin]) if obs_normalize else final_raw[fin]
        if obs_normalize:
            norm.push(nraw)                                             # B2
        nraw = np.array(nraw, F32)
        if hit.any():
            rst = env.reset_envs(hit)
            nraw[hit] = rst[hit]
            if obs_normalize:
                norm.push(rst[hit])                                     # B3
        nobs = _apply(norm, nraw) if obs_normalize else nraw
        ep_ret = (ep_ret + rew).astype(F32); ep_cost = (ep_cost + cost).astype(F32); ep_len += 1
        sl['obs'][t] = obs; sl['act'][t] = act; sl['logp'][t] = logp
        sl['rew'][t] = rew; sl['cost'][t] = cost; sl['val_r'][t] = v_r; sl['val_c'][t] = v_c
        sl['flags'][t] = term.astype(np.uint8) * FLAG_TERMINATED + trunc.astype(np.uint8) * FLAG_TRUNCATED
        obs = nobs
        need_final = trunc & ~term
        need_next = (~term) & (~trunc) & (t == T - 1)
        if need_final.any():
            br, bc = ac.values(theta, final_norm, O, A)
            sl['boot_r'][t][need_final] = br[need_final]; sl['boot_c'][t][need_final] = bc[need_final]
        if need_next.any():
            br, bc = ac.values(theta, obs, O, A)
            sl['boot_r'][t][need_next] = br[need_next]; sl['boot_c'][t][need_next] = bc[need_next]
        done = term | trunc
        for i in np.nonzero(done)[0]:
            if window is not None:
                window.append((float(ep_ret[i]), float(ep_cost[i]), float(ep_len[i])))
        ep_ret[done] = 0; ep_cost[done] = 0; ep_len[done] = 0
    return sl
