"""Oracle: float64 reference of the optimiser step that ends every minibatch (torch-CPU).  TEST INFRASTRUCTURE ONLY.

Per network, in the order of policy_gradient.py:L407-524:
  critic L2 term coef * sum(theta^2) added to the critic losses   base/policy_gradient.py:L429-433 (Learner.critic_step)
  clip_grad_norm_(params_of_the_network, max_grad_norm)            base/policy_gradient.py:L436-443
  torch.optim.Adam(lr of the network).step()                       (dependency, called directly)
on float64 per-tensor leaves in oracle.actor_critic.layout order, one float64 torch.optim.Adam per network.  The
kernels read max_grad_norm <= 0 as "no clipping"; so does this reference (clip_grad_norm_ would zero the gradient).

`state` is a dict of float64 numpy vectors over the flat parameter vector [actor | reward_critic | cost_critic]:
theta, m (exp_avg), v (exp_avg_sq), and step (int64 [3], Adam steps taken per network).  step64 takes supplied
gradients; ppo_epoch64 takes minibatch gradients from float64 autograd at the current theta on advantages
standardised with the buffer's moments (oracle.fisher64), so the same theta / m / v / step can be compared with
the device after every minibatch step, every pass, and across ppo_epoch calls.
"""
from __future__ import annotations

import numpy as np
import torch
from torch.distributions import Normal, kl_divergence
from torch.nn.utils.clip_grad import clip_grad_norm_

from oracle import actor_critic as ac
from oracle import fisher64 as f64

NETS = ('actor', 'reward_critic', 'cost_critic')
F64 = torch.float64


def _dims(P: int, O: int):
    """Act dim of the flat [actor | 2 critics] vector of a 64-64 MLP for obs dim O."""
    nc = ac.HID * O + ac.HID + ac.HID * ac.HID + ac.HID + ac.HID + 1
    A = f64._act_dim(P - 2 * nc, O)
    return ac.layout(O, A)


def init_state(theta) -> dict:
    theta = np.asarray(theta, np.float32).astype(np.float64)
    return {'theta': theta.copy(), 'm': np.zeros_like(theta), 'v': np.zeros_like(theta), 'step': np.zeros(3, np.int64)}


def _copy(state) -> dict:
    return {k: np.array(v, copy=True) for k, v in state.items()}


def _leaves(vec, lay, net, grad=False):
    t = torch.as_tensor(vec)
    return {name: t[o:o + int(np.prod(shape))].view(*shape).clone().requires_grad_(grad)
            for name, (o, shape) in lay[net]['entries'].items()}


def _flat(tensors) -> np.ndarray:
    return torch.cat([t.detach().reshape(-1) for t in tensors]).numpy()


def _net_step(state, lay, net, loss_fn, *, max_grad_norm, lr, critic_norm_coef):
    """One optimiser step of one network: loss_fn(params) is the data loss; the critic L2 term is added exactly as
    Learner.critic_step adds it.  Updates `state` in place; returns (pre-clip norm, clip coefficient, clipped
    gradient, logged loss)."""
    s, n = lay[net]['start'], lay[net]['size']
    sl = slice(s, s + n)
    p = _leaves(state['theta'], lay, net, grad=True)
    params = list(p.values())
    loss = loss_fn(p)
    if net != 'actor' and critic_norm_coef:
        for t in params:
            loss = loss + t.pow(2).sum() * critic_norm_coef
    loss.backward()
    opt = torch.optim.Adam(params, lr=lr)
    t = int(state['step'][NETS.index(net)])
    if t:
        m, v = _leaves(state['m'], lay, net), _leaves(state['v'], lay, net)
        for name, q in p.items():
            opt.state[q] = {'step': torch.tensor(float(t), dtype=F64), 'exp_avg': m[name].detach().clone(),
                            'exp_avg_sq': v[name].detach().clone()}
    if max_grad_norm > 0:
        norm = float(clip_grad_norm_(params, max_grad_norm))
        coef = min(max_grad_norm / (norm + 1e-6), 1.0)
    else:
        norm, coef = float(torch.cat([q.grad.reshape(-1) for q in params]).norm()), 1.0
    grad = _flat([q.grad for q in params])
    opt.step()
    state['theta'][sl] = _flat(params)
    state['m'][sl] = _flat([opt.state[q]['exp_avg'] for q in params])
    state['v'][sl] = _flat([opt.state[q]['exp_avg_sq'] for q in params])
    state['step'][NETS.index(net)] = t + 1
    return norm, coef, grad, float(loss.detach())


def step64(state, grads, *, max_grad_norm, lrs, critic_norm_coef, O, net_mask: int = 7):
    """One optimiser step on supplied data gradients `grads` (flat, all networks; the critic L2 term is added here).
    Returns (new state, record) with record = {norm [3] (pre-clip), coef [3] (clip coefficient, 1 when not
    clipped), grad (the clipped gradient, flat; zero for networks outside net_mask), l2 [3] (coef * sum theta^2 of
    the critics before the step: what the logged critic loss adds)}."""
    state = _copy(state)
    grads = np.asarray(grads, np.float64)
    lay = _dims(state['theta'].size, O)
    rec = {'norm': np.zeros(3), 'coef': np.ones(3), 'grad': np.zeros_like(grads), 'l2': np.zeros(3)}
    for k, net in enumerate(NETS):
        if not (net_mask >> k) & 1:
            continue
        s, n = lay[net]['start'], lay[net]['size']
        g = torch.as_tensor(grads[s:s + n])
        if net != 'actor':
            rec['l2'][k] = critic_norm_coef * float((torch.as_tensor(state['theta'][s:s + n]) ** 2).sum())
        norm, coef, clipped, _ = _net_step(
            state, lay, net, lambda p, g=g: (torch.cat([q.reshape(-1) for q in p.values()]) * g).sum(),
            max_grad_norm=max_grad_norm, lr=lrs[k], critic_norm_coef=critic_norm_coef)
        rec['norm'][k], rec['coef'][k] = norm, coef
        rec['grad'][s:s + n] = clipped
    return state, rec


def ppo_epoch64(theta, data, moments, perms, lam, *, net_mask, loss_kind, batch_size, update_iters, clip=0.2,
                entropy_coef=0.0, critic_norm_coef=0.001, max_grad_norm=40.0, lrs=(3e-4, 3e-4, 3e-4),
                target_kl=0.02, kl_early_stop=False, state=None):
    """PolicyGradient._update (policy_gradient.py:L345-405) in float64 for the loss kinds of the fused kernels:
    0 PPO clip (+ entropy bonus), 1 plain ratio surrogate, 3 cost surrogate (CPO / PCPO cost pass).  `data` is
    env-major with RAW advantages; `perms[i]` is the env-major sample order of pass i.  The minibatch gradients of
    all networks are taken at the same theta (the networks do not share parameters, so the order of the three
    steps does not matter).  A pass that trains the actor ends with the full-batch KL against the policy the epoch
    started from and the early stop; without the actor every pass runs.

    Returns (state, record, passes): record is one dict per minibatch step with norm [3], coef [3], grad (clipped,
    flat), loss [3] (logged values: critic mse + coef * sum theta^2; actor surrogate without the entropy bonus),
    ratio (mean ratio of the actor), plus 'kl' [passes]."""
    assert loss_kind in (0, 1, 3)
    state = init_state(theta) if state is None else _copy(state)
    P = state['theta'].size
    O = np.asarray(data['obs']).shape[1]
    lay = _dims(P, O)
    obs, act, logp = f64._t64(data['obs']), f64._t64(data['act']), f64._t64(data['logp'])
    tgt = {'reward_critic': f64._t64(data['target_value_r']), 'cost_critic': f64._t64(data['target_value_c'])}
    _, adv_c, adv = f64._std_adv(data, moments, lam)
    train_actor = bool(net_mask & 1)
    if train_actor:
        with torch.no_grad():
            old = ac.actor_dist(_leaves(state['theta'], lay, 'actor'), obs)
            old = Normal(old.loc.clone(), old.scale.clone())
    record, kls, passes = [], [], 0
    for it in range(update_iters):
        perm = torch.as_tensor(np.asarray(perms[it], np.int64))
        for s0 in range(0, len(perm), batch_size):
            idx = perm[s0:s0 + batch_size]
            o = obs[idx]
            rec = {'norm': np.zeros(3), 'coef': np.ones(3), 'grad': np.zeros(P), 'loss': np.zeros(3), 'ratio': 0.0}
            for k, net in enumerate(NETS):
                if not (net_mask >> k) & 1:
                    continue
                if net == 'actor':
                    surr = {}

                    def loss_fn(p, surr=surr):
                        d = ac.actor_dist(p, o)
                        ratio = torch.exp(d.log_prob(act[idx]).sum(-1) - logp[idx])
                        if loss_kind == 0:
                            a = adv[idx]
                            loss = -torch.min(ratio * a, torch.clamp(ratio, 1 - clip, 1 + clip) * a).mean()
                        elif loss_kind == 1:
                            loss = -(ratio * adv[idx]).mean()
                        else:
                            loss = (ratio * adv_c[idx]).mean()
                        surr['loss'], surr['ratio'] = float(loss.detach()), float(ratio.detach().mean())
                        if loss_kind == 0 and entropy_coef:
                            loss = loss - entropy_coef * d.entropy().mean()
                        return loss
                else:
                    def loss_fn(p, net=net):
                        return torch.nn.functional.mse_loss(ac.critic_value(p, o), tgt[net][idx])
                norm, coef, grad, logged = _net_step(state, lay, net, loss_fn, max_grad_norm=max_grad_norm, lr=lrs[k],
                                                     critic_norm_coef=critic_norm_coef)
                sl = slice(lay[net]['start'], lay[net]['start'] + lay[net]['size'])
                rec['norm'][k], rec['coef'][k], rec['grad'][sl] = norm, coef, grad
                rec['loss'][k] = surr['loss'] if net == 'actor' else logged
                if net == 'actor':
                    rec['ratio'] = surr['ratio']
            record.append(rec)
        passes += 1
        if train_actor:
            with torch.no_grad():
                new = ac.actor_dist(_leaves(state['theta'], lay, 'actor'), obs)
                kls.append(float(kl_divergence(old, new).sum(-1).mean()))
            if kl_early_stop and kls[-1] > target_kl:
                break
    return state, {'steps': record, 'kl': kls}, passes
