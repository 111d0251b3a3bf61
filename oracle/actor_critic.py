"""Oracle: actor / critic MLPs and the Gaussian policy head (torch-CPU).  TEST INFRASTRUCTURE ONLY.

Follows omnisafe/utils/model.py:L73-111 (Linear-Tanh-Linear-Tanh-Linear), models/actor/
gaussian_learning_actor.py:L64-139 (Normal(mean, exp(log_std)), rsample, log_prob summed over the
action dim), models/critic/v_critic.py:L75-92, models/actor_critic/constraint_actor_critic.py:L84-109
and the flat parameter order of utils/tools.py:L35-129 (named_parameters order, log_std first).
"""
from __future__ import annotations

import contextlib
import math

import numpy as np
import torch
import torch.nn.functional as F
from torch.distributions import Normal

HID = 64
# model_cfgs.*.activation (utils/model.py:L62-70); softplus with nn.Softplus's defaults (beta 1, threshold 20)
ACT = {'tanh': torch.tanh, 'identity': lambda z: z, 'relu': torch.relu, 'sigmoid': torch.sigmoid, 'softplus': F.softplus}
_DEFAULT = {'actor': ('tanh', (HID, HID)), 'critic': ('tanh', (HID, HID))}
_spec = dict(_DEFAULT)


@contextlib.contextmanager
def nets(actor: str = 'tanh', critic: str = 'tanh', actor_hidden=(HID, HID), critic_hidden=(HID, HID)):
    """Inside the block, `mlp` is the network of these activations and real hidden widths: the actor's when its
    parameters hold 'log_std', both critics' otherwise.  Parameters keep the 64-wide layout; each layer computes its real
    units only (the leading rows / columns of the padded tensors), so a sigmoid or softplus network is the narrow one and
    not one whose pad units output sigmoid(0) or log 2, and autograd leaves exact zeros at the pads.  Leaving the block
    restores the enclosing spec (tanh, 64 wide outside every block)."""
    global _spec
    for which, act, hs in (('actor', actor, actor_hidden), ('critic', critic, critic_hidden)):
        assert act in ACT, (which, act)
        assert len(hs) == 2 and all(1 <= int(h) <= HID for h in hs), (which, hs)
    saved = _spec
    _spec = {'actor': (actor, tuple(int(h) for h in actor_hidden)),
             'critic': (critic, tuple(int(h) for h in critic_hidden))}
    try:
        yield
    finally:
        _spec = saved


def net_spec(which: str):
    """(activation function, (width 1, width 2)) of 'actor' or 'critic' under the current `nets` block."""
    act, widths = _spec[which]
    return ACT[act], widths


def layout(O: int, A: int, hid: int = HID):
    """Sizes/offsets of the flat vector theta = [actor | reward_critic | cost_critic]."""
    actor = [('log_std', (A,)), ('w1', (hid, O)), ('b1', (hid,)), ('w2', (hid, hid)), ('b2', (hid,)),
             ('w3', (A, hid)), ('b3', (A,))]
    critic = [('w1', (hid, O)), ('b1', (hid,)), ('w2', (hid, hid)), ('b2', (hid,)),
              ('w3', (1, hid)), ('b3', (1,))]
    out, off = {}, 0
    for net, spec in (('actor', actor), ('reward_critic', critic), ('cost_critic', critic)):
        start = off
        entries = {}
        for name, shape in spec:
            n = int(np.prod(shape))
            entries[name] = (off, shape)
            off += n
        out[net] = {'start': start, 'size': off - start, 'entries': entries}
    out['total'] = off
    return out


def unflatten(theta, O: int, A: int):
    """dict net -> dict name -> torch view (shares memory with theta if theta is a torch tensor)."""
    theta = torch.as_tensor(theta)
    lay = layout(O, A)
    return {net: {name: theta[o:o + int(np.prod(shape))].view(*shape)
                  for name, (o, shape) in lay[net]['entries'].items()}
            for net in ('actor', 'reward_critic', 'cost_critic')}


def init_theta(O: int, A: int, seed: int = 0, log_std=None, actor_hidden=(HID, HID),
               critic_hidden=(HID, HID)) -> np.ndarray:
    """Random init with the reference's scheme: kaiming_uniform_(a=sqrt(5)) weights and torch's
    default Linear bias init (utils/model.py:L25-44), log_std = 0 (the reference's initial value) or the
    given [A] values (a policy whose std has been trained, e.g. trained_log_std(A)).  Hidden widths below 64: only the
    real block of each layer is drawn, with its real fan-in, and every pad stays +0."""
    g = torch.Generator().manual_seed(seed)
    lay = layout(O, A)
    theta = torch.zeros(lay['total'])
    views = unflatten(theta, O, A)
    for net, (h1, h2) in (('actor', actor_hidden), ('reward_critic', critic_hidden), ('cost_critic', critic_hidden)):
        for w, b, rows, cols in (('w1', 'b1', h1, O), ('w2', 'b2', h2, h1), ('w3', 'b3', None, h2)):
            W, B = views[net][w][:rows, :cols], views[net][b][:rows]
            fan_in = W.shape[1]
            bound_w = math.sqrt(6.0 / ((1 + 5.0) * fan_in))
            W.copy_(torch.empty(W.shape).uniform_(-bound_w, bound_w, generator=g))
            bound_b = 1.0 / math.sqrt(fan_in)
            B.copy_(torch.empty(B.shape).uniform_(-bound_b, bound_b, generator=g))
    if log_std is not None:
        views['actor']['log_std'].copy_(torch.as_tensor(np.asarray(log_std, np.float32)).reshape(A))
    return theta.numpy().copy()


def trained_log_std(A: int, seed: int = 0) -> np.ndarray:
    """log_std of a policy after training: distinct per action, spread evenly over [-1.6, 0.4] (sigma 0.20 to 1.49)
    in a seeded order that is neither increasing nor decreasing; A = 1: -0.7.  At log_std = 0 sigma, sigma^2 and
    1 / sigma^2 are all 1 and log sigma is 0, so a loss or Fisher product that confuses them looks right there."""
    if A == 1:
        return np.array([-0.7], np.float32)
    vals = np.linspace(-1.6, 0.4, A)
    rng = np.random.default_rng(seed)
    while True:
        order = rng.permutation(A)
        steps = np.diff(order)
        if A < 3 or ((steps > 0).any() and (steps < 0).any()):
            return vals[order].astype(np.float32)


def log_std_shift(A: int, seed: int = 0) -> np.ndarray:
    """Per-action change of log_std between an old policy and the current one: magnitudes in [0.05, 0.3], seeded
    signs, so the KL terms see sigma_old != sigma in every action."""
    rng = np.random.default_rng(seed + 1)
    return (rng.uniform(0.05, 0.3, A) * rng.choice([-1.0, 1.0], A)).astype(np.float32)


def mlp(p, x):
    """Linear-Act-Linear-Act-Linear of the actor ('log_std' in p) or a critic, with the activation and the real widths
    of the current `nets` block (tanh, 64 wide outside one)."""
    f, (a1, a2) = net_spec('actor' if 'log_std' in p else 'critic')
    h = f(F.linear(x, p['w1'][:a1], p['b1'][:a1]))
    h = f(F.linear(h, p['w2'][:a2, :a1], p['b2'][:a2]))
    return F.linear(h, p['w3'][:, :a2], p['b3'])


def actor_dist(p, obs) -> Normal:
    return Normal(mlp(p, obs), torch.exp(p['log_std']))


def critic_value(p, obs):
    return torch.squeeze(mlp(p, obs), -1)


def step(theta, obs, eps, O: int, A: int):
    """ConstraintActorCritic.step with the standard-normal draw `eps` supplied by the caller
    (Normal.rsample == loc + eps * scale).  Returns float32 numpy (act, v_r, v_c, logp)."""
    nets = unflatten(torch.as_tensor(np.asarray(theta, np.float32)), O, A)
    obs = torch.as_tensor(np.asarray(obs, np.float32))
    eps = torch.as_tensor(np.asarray(eps, np.float32))
    with torch.no_grad():
        v_r = critic_value(nets['reward_critic'], obs)
        v_c = critic_value(nets['cost_critic'], obs)
        dist = actor_dist(nets['actor'], obs)
        act = dist.loc + eps * dist.scale
        logp = dist.log_prob(act).sum(-1)
    return act.numpy(), v_r.numpy(), v_c.numpy(), logp.numpy()


def values(theta, obs, O: int, A: int):
    nets = unflatten(torch.as_tensor(np.asarray(theta, np.float32)), O, A)
    obs = torch.as_tensor(np.asarray(obs, np.float32))
    with torch.no_grad():
        return (critic_value(nets['reward_critic'], obs).numpy(),
                critic_value(nets['cost_critic'], obs).numpy())
