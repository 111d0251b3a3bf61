"""Oracle: float64 reference of the natural-gradient pieces (torch-CPU).  TEST INFRASTRUCTURE ONLY.

The policy mean, the Fisher-vector product, the full-batch surrogate gradients, the line-search evaluation and
the conjugate-gradient solve of the NaturalPG family, in float64 on per-tensor leaves of the actor, with the
reference's definitions:
  NaturalPG._fvp (Hessian of mean KL by double backward)   base/natural_pg.py:L74-119
  surrogates of the actor step / line searches             base/natural_pg.py:L146-166, second_order/cpo.py:L182-212
  advantage standardisation                                vector_onpolicy_buffer.py:L131-136
  conjugate_gradients                                      utils/math.py:L86-132
`theta` is the flat actor block (log_std first, as oracle.actor_critic.layout orders it) of a float32 parameter
vector; the act dim follows from its length and the obs dim.  `moments` is the 4-vector the buffer hands the
kernels: mean_r, std_r + 1e-8, mean_c, 1.  Work over the rows is done in chunks, so the 524 288-row batch of the
bench fits in memory.
"""
from __future__ import annotations

import numpy as np
import torch
from torch.distributions import Normal, kl_divergence

from oracle import actor_critic as ac

CHUNK = 65536
F64 = torch.float64


def _act_dim(n_actor: int, O: int) -> int:
    # actor size = A (log_std) + 64 O + 64 + 64 * 64 + 64 + 64 A + A
    A, rem = divmod(n_actor - ac.HID * O - 2 * ac.HID - ac.HID * ac.HID, ac.HID + 2)
    assert rem == 0 and A > 0, 'theta is not the actor block of a 64-64 MLP policy for this obs dim'
    return A


def _leaves(theta, O: int, grad: bool = False):
    t = torch.as_tensor(np.asarray(theta, np.float32).astype(np.float64)).reshape(-1)
    A = _act_dim(t.numel(), O)
    ents = ac.layout(O, A)['actor']['entries']
    return {name: t[o:o + int(np.prod(shape))].view(*shape).clone().requires_grad_(grad)
            for name, (o, shape) in ents.items()}


def _t64(x):
    return torch.as_tensor(np.asarray(x, np.float32).astype(np.float64))


def _chunks(n: int, chunk: int):
    for s in range(0, n, chunk):
        yield slice(s, min(n, s + chunk))


def _std_adv(data, moments, lam):
    """(adv_r - mean_r) / std_r, adv_c - mean_c (the cost advantage is centred only) and the Lagrangian mix
    (adv_r - lam adv_c) / (1 + lam) (PPOLag._compute_adv_surrogate)."""
    m = np.asarray(moments, np.float64)
    adv_r = (_t64(data['adv_r']) - m[0]) / m[1]
    adv_c = _t64(data['adv_c']) - m[2]
    return adv_r, adv_c, (adv_r - lam * adv_c) / (1.0 + lam)


def mean64(theta, obs, chunk: int = CHUNK) -> np.ndarray:
    """Policy mean at `theta` for every row of `obs` [B, O]."""
    obs = _t64(obs)
    p = _leaves(theta, obs.shape[1])
    with torch.no_grad():
        return torch.cat([ac.mlp(p, obs[sl]) for sl in _chunks(obs.shape[0], chunk)]).numpy()


def logp64(theta, obs, act, chunk: int = CHUNK) -> np.ndarray:
    """log pi(act | obs) at `theta`, summed over the action dims."""
    obs, act = _t64(obs), _t64(act)
    p = _leaves(theta, obs.shape[1])
    with torch.no_grad():
        return torch.cat([ac.actor_dist(p, obs[sl]).log_prob(act[sl]).sum(-1)
                          for sl in _chunks(obs.shape[0], chunk)]).numpy()


def fvp64(theta, vec, obs, damping: float, chunk: int = CHUNK) -> np.ndarray:
    """Hessian of mean_{rows, action dims} KL(p_old || p) at p == p_old, applied to `vec`, plus damping * vec.
    Each chunk's mean is weighted by n_chunk / B, so the result does not depend on the chunk size."""
    obs = _t64(obs)
    B = obs.shape[0]
    p = _leaves(theta, obs.shape[1], grad=True)
    params = list(p.values())
    v = torch.as_tensor(np.asarray(vec, np.float64))
    out = torch.zeros_like(v)
    for sl in _chunks(B, chunk):
        q = ac.actor_dist(p, obs[sl])
        p_old = Normal(q.loc.detach().clone(), q.scale.detach().clone())
        kl = kl_divergence(p_old, q).mean()
        grads = torch.autograd.grad(kl, params, create_graph=True)
        kl_v = (torch.cat([g.reshape(-1) for g in grads]) * v).sum()
        hv = torch.autograd.grad(kl_v, params)
        out += torch.cat([g.reshape(-1) for g in hv]) * ((sl.stop - sl.start) / B)
    return (out + damping * v).numpy()


def surrogate_grad64(theta, data, moments, lam: float, kind: str, chunk: int = CHUNK):
    """Gradient w.r.t. the actor and value of the full-batch surrogate:
      kind 'ratio': -mean(ratio * (adv_r - lam adv_c) / (1 + lam))    (NaturalPG / TRPO / CPO reward surrogate)
      kind 'cost':   mean(ratio * adv_c)                               (CPO._loss_pi_cost)
    with ratio = exp(log pi(act | obs) - logp) and the advantages standardised with `moments`."""
    assert kind in ('ratio', 'cost')
    obs, act, logp = _t64(data['obs']), _t64(data['act']), _t64(data['logp'])
    B = obs.shape[0]
    p = _leaves(theta, obs.shape[1], grad=True)
    _, adv_c, adv = _std_adv(data, moments, lam)
    w = adv_c if kind == 'cost' else -adv
    loss = 0.0
    for sl in _chunks(B, chunk):
        ratio = torch.exp(ac.actor_dist(p, obs[sl]).log_prob(act[sl]).sum(-1) - logp[sl])
        part = (ratio * w[sl]).sum() / B
        part.backward()
        loss += float(part.detach())
    return torch.cat([t.grad.reshape(-1) for t in p.values()]).numpy(), loss


def eval64(theta, theta_old, data, moments, lam: float, chunk: int = CHUNK) -> dict:
    """What UpdateEngine.evaluate returns for the trial actor `theta` against the old policy `theta_old`:
    kl (mean over samples AND action dims of KL(old || new)), loss (-mean ratio adv), loss_r (-mean ratio adv_r),
    loss_c (mean ratio adv_c), ratio (mean)."""
    obs, act, logp = _t64(data['obs']), _t64(data['act']), _t64(data['logp'])
    B, O = obs.shape
    p, p_old = _leaves(theta, O), _leaves(theta_old, O)
    adv_r, adv_c, adv = _std_adv(data, moments, lam)
    s = dict.fromkeys(('kl', 'loss', 'loss_r', 'loss_c', 'ratio'), 0.0)
    with torch.no_grad():
        for sl in _chunks(B, chunk):
            new, old = ac.actor_dist(p, obs[sl]), ac.actor_dist(p_old, obs[sl])
            ratio = torch.exp(new.log_prob(act[sl]).sum(-1) - logp[sl])
            s['kl'] += float(kl_divergence(old, new).sum())
            s['loss'] -= float((ratio * adv[sl]).sum())
            s['loss_r'] -= float((ratio * adv_r[sl]).sum())
            s['loss_c'] += float((ratio * adv_c[sl]).sum())
            s['ratio'] += float(ratio.sum())
    A = act.shape[1]
    return {k: v / (B * A if k == 'kl' else B) for k, v in s.items()}


def cg64(fvp, b, iters: int, residual_tol: float = 1e-10, eps: float = 1e-6):
    """conjugate_gradients (utils/math.py:L86-132) in float64.  `fvp` maps a float64 numpy vector to F v.
    Returns (x, steps run, residual norm after each step)."""
    b = np.asarray(b, np.float64)
    x = np.zeros_like(b)
    r = b - fvp(x)
    p = r.copy()
    rdotr = float(r @ r)
    norms = []
    for _ in range(iters):
        z = np.asarray(fvp(p), np.float64)
        alpha = rdotr / (float(p @ z) + eps)
        x = x + alpha * p
        r = r - alpha * z
        new_rdotr = float(r @ r)
        norms.append(np.sqrt(new_rdotr))
        if norms[-1] < residual_tol:
            break
        p = r + new_rdotr / (rdotr + eps) * p
        rdotr = new_rdotr
    return x, len(norms), norms
