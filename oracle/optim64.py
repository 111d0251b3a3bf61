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


def actor_loss64(d, old, act, logp, adv, adv_r, adv_c, *, loss_kind, clip=0.2, entropy_coef=0.0, focops_lam=1.0,
                 focops_eta=0.0):
    """Actor loss of one minibatch for every loss kind of the update kernels, in float64.  d: the policy being
    trained on the minibatch rows; old: the old policy on the same rows (FOCOPS only); adv: the Lagrangian mix;
    adv_r / adv_c: the standardised advantages.  The kernels' parameter names: FOCOPS temperature focops_lam and
    trust region focops_eta; P3O kappa = focops_lam and Jc - cost_limit = focops_eta.
      0 PPO clip on adv (+ entropy bonus)                                    base/ppo.py:L35-87
      1 -mean(ratio adv), 3 mean(ratio adv_c)                                policy_gradient.py:L551-588, cpo.py:L182-212
      2 FOCOPS: mean_i(m_i kl_i) - mean_i(m_i) mean_j(ratio_j adv_j) / lam (+ entropy bonus), kl_i = KL(new || old)
        summed over the action dims, m_i = 1{kl_i <= eta} on detached values.  This is the mean of the reference's
        [b, b] broadcast (first_order/focops.py:L85-89, Learner.loss_pi_focops) without forming it.
      5 P3O: PPO clip on adv_r (+ entropy bonus) + kappa relu(mean(ratio adv_c) + Jc - limit)   p3o.py:L48-91
    Returns (loss to differentiate, info): info['stats'] = [slot 0, slot 1, slot 2, slot 4] of the kernels' logged
    actor statistics (slot 0: the loss without the entropy bonus and without the P3O penalty; slot 1: mean ratio;
    slot 2: FOCOPS mean KL, P3O penalty term; slot 4: FOCOPS mask mean); info['pass1']: what the forward-only pass
    reduces (FOCOPS mask mean, P3O mean(ratio adv_c)); info['gate']: P3O kappa or 0; info['margin']: distance of
    the pass-1 decisions from their boundary (FOCOPS min_i |kl_i - eta|, P3O |mean + Jc - limit|); info['entropy']: the
    mean entropy over rows and action dims (what the bonus multiplies)."""
    ratio = torch.exp(d.log_prob(act).sum(-1) - logp)
    slot2 = slot4 = 0.0
    info = {'pass1': None, 'gate': None, 'margin': None}
    if loss_kind in (0, 5):
        a = adv_r if loss_kind == 5 else adv
        loss = -torch.min(ratio * a, torch.clamp(ratio, 1 - clip, 1 + clip) * a).mean()
    elif loss_kind == 1:
        loss = -(ratio * adv).mean()
    elif loss_kind == 3:
        loss = (ratio * adv_c).mean()
    else:
        assert loss_kind == 2
        kl = kl_divergence(d, old).sum(-1)
        m = (kl.detach() <= focops_eta).to(F64)
        loss = (m * kl).mean() - m.mean() * (ratio * adv).mean() / focops_lam
        slot2, slot4 = float(kl.detach().mean()), float(m.mean())
        info['pass1'] = slot4
        info['margin'] = float((kl.detach() - focops_eta).abs().min())
    slot0 = float(loss.detach())
    if loss_kind == 5:
        z = (ratio * adv_c).mean() + focops_eta
        penalty = focops_lam * torch.relu(z)
        loss = loss + penalty
        slot2 = float(penalty.detach())
        info['pass1'] = float(z.detach()) - focops_eta
        info['gate'] = focops_lam if float(z.detach()) > 0 else 0.0
        info['margin'] = abs(float(z.detach()))
    if loss_kind in (0, 2, 5) and entropy_coef:
        loss = loss - entropy_coef * d.entropy().mean()
    info['stats'] = [slot0, float(ratio.detach().mean()), slot2, slot4]
    info['entropy'] = float(d.entropy().detach().mean())
    return loss, info


def minibatch64(theta, data, moments, idx, lam, *, loss_kind, old_mu=None, old_logstd=None, critic_norm_coef=0.0,
                net_mask=7, **loss_kw):
    """The data gradient of every network on the minibatch rows `idx` (env-major) at `theta`, as one launch of a
    minibatch gradient kernel + osb_grad_reduce leaves it: critics mse + critic_norm_coef sum theta^2, the actor
    loss of actor_loss64 with the old policy Normal(old_mu[idx], exp(old_logstd)).  Returns (flat gradient, actor
    info of actor_loss64)."""
    theta = np.asarray(theta, np.float32).astype(np.float64)
    O = np.asarray(data['obs']).shape[1]
    lay = _dims(theta.size, O)
    idx = torch.as_tensor(np.asarray(idx, np.int64))
    o = f64._t64(data['obs'])[idx]
    adv_r, adv_c, adv = (x[idx] for x in f64._std_adv(data, moments, lam))
    grad, info = np.zeros_like(theta), None
    for k, net in enumerate(NETS):
        if not (net_mask >> k) & 1:
            continue
        p = _leaves(theta, lay, net, grad=True)
        if net == 'actor':
            old = None
            if old_mu is not None:
                old = Normal(f64._t64(old_mu)[idx], torch.exp(f64._t64(old_logstd)).expand(len(idx), -1))
            loss, info = actor_loss64(ac.actor_dist(p, o), old, f64._t64(data['act'])[idx], f64._t64(data['logp'])[idx],
                                      adv, adv_r, adv_c, loss_kind=loss_kind, **loss_kw)
        else:
            tgt = f64._t64(data['target_value_r' if net == 'reward_critic' else 'target_value_c'])[idx]
            loss = torch.nn.functional.mse_loss(ac.critic_value(p, o), tgt)
            for t in p.values():
                loss = loss + t.pow(2).sum() * critic_norm_coef
        loss.backward()
        s = lay[net]['start']
        grad[s:s + lay[net]['size']] = _flat([t.grad for t in p.values()])
    return grad, info


def ppo_epoch64(theta, data, moments, perms, lam, *, net_mask, loss_kind, batch_size, update_iters, clip=0.2,
                entropy_coef=0.0, focops_lam=1.0, focops_eta=0.0, critic_norm_coef=0.001, max_grad_norm=40.0,
                lrs=(3e-4, 3e-4, 3e-4), target_kl=0.02, kl_early_stop=False, state=None):
    """PolicyGradient._update (policy_gradient.py:L345-405) / FOCOPS._update in float64 for every loss kind of the
    update kernels (actor_loss64): 0 PPO clip (+ entropy bonus), 1 plain ratio surrogate, 2 FOCOPS, 3 cost surrogate
    (CPO / PCPO cost pass), 5 P3O (no Lagrangian mix: P3O trains on adv_r).  `data` is env-major with RAW
    advantages; `perms[i]` is the env-major sample order of pass i.  The minibatch gradients of all networks are
    taken at the same theta (the networks do not share parameters, so the order of the three steps does not
    matter).  FOCOPS's old policy is the one the epoch started from.  A pass that trains the actor ends with the
    full-batch KL against that policy and the early stop; without the actor every pass runs.

    Returns (state, record, passes): record is one dict per minibatch step with norm [3], coef [3], grad (clipped,
    flat), loss [3] (logged values: critic mse + coef * sum theta^2; actor: slot 0 of actor_loss64), ratio (mean
    ratio of the actor), and for the actor 'stats' / 'pass1' / 'gate' / 'margin' / 'entropy' of actor_loss64; plus 'kl'
    [passes]."""
    assert loss_kind in (0, 1, 2, 3, 5)
    state = init_state(theta) if state is None else _copy(state)
    P = state['theta'].size
    O = np.asarray(data['obs']).shape[1]
    lay = _dims(P, O)
    obs, act, logp = f64._t64(data['obs']), f64._t64(data['act']), f64._t64(data['logp'])
    tgt = {'reward_critic': f64._t64(data['target_value_r']), 'cost_critic': f64._t64(data['target_value_c'])}
    adv_r, adv_c, adv = f64._std_adv(data, moments, lam)
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
                        loss, info = actor_loss64(
                            ac.actor_dist(p, o), Normal(old.loc[idx], old.scale[idx]), act[idx], logp[idx], adv[idx],
                            adv_r[idx], adv_c[idx], loss_kind=loss_kind, clip=clip, entropy_coef=entropy_coef,
                            focops_lam=focops_lam, focops_eta=focops_eta)
                        surr.update(info)
                        return loss
                else:
                    def loss_fn(p, net=net):
                        return torch.nn.functional.mse_loss(ac.critic_value(p, o), tgt[net][idx])
                norm, coef, grad, logged = _net_step(state, lay, net, loss_fn, max_grad_norm=max_grad_norm, lr=lrs[k],
                                                     critic_norm_coef=critic_norm_coef)
                sl = slice(lay[net]['start'], lay[net]['start'] + lay[net]['size'])
                rec['norm'][k], rec['coef'][k], rec['grad'][sl] = norm, coef, grad
                rec['loss'][k] = surr['stats'][0] if net == 'actor' else logged
                if net == 'actor':
                    rec['ratio'] = surr['stats'][1]
                    rec.update({key: surr[key] for key in ('stats', 'pass1', 'gate', 'margin', 'entropy')})
            record.append(rec)
        passes += 1
        if train_actor:
            with torch.no_grad():
                new = ac.actor_dist(_leaves(state['theta'], lay, 'actor'), obs)
                kls.append(float(kl_divergence(old, new).sum(-1).mean()))
            if kl_early_stop and kls[-1] > target_kl:
                break
    return state, {'steps': record, 'kl': kls}, passes
