"""Flat-parameter ConstraintActorCritic (actor + reward critic + cost critic).

Mirrors omnisafe/models/actor_critic/constraint_actor_critic.py:L31-109 and
actor_critic.py:L60-113: three independent Linear-Act-Linear-Act-Linear trunks
(utils/model.py:L73-111; Act = model_cfgs.actor.activation for the actor, model_cfgs.critic.activation for both
critics: identity, relu, sigmoid, softplus or tanh), GaussianLearningActor with a state-independent `log_std`
(models/actor/gaussian_learning_actor.py:L29-62), one Adam optimiser per network and a LinearLR
decay of the actor learning rate.  All parameters live in ONE flat fp32 device vector
`theta = [actor | reward_critic | cost_critic]` in the reference's named_parameters() order
(utils/tools.py:L35-129), so the CG vector layout, the flat gradient all-reduce and the fused
kernels share it.  `actor_state_dict()` re-exports the actor under the reference's key names so
`{'pi': ..., 'obs_normalizer': ...}` checkpoints stay loadable by the reference Evaluator
(omnisafe/evaluator.py:L153-178, algorithms/on_policy/base/policy_gradient.py:L183-189).

`model_cfgs.actor.hidden_sizes` and `model_cfgs.critic.hidden_sizes` may be any two widths from 1 to 64.  `theta`, the
gradient and the Adam moments keep the 64-wide kernel layout; a narrower network sits in it zero-padded (ParamMap), which
owns the one mapping between the reference's shapes and that layout: `named_views`, `actor_state_dict()`, the
initialisation, the critic hooks, the evaluator and the golden fixtures all go through it.

The kernels read the activations and the real widths from one process-wide spec (osb_set_net_spec).  Every launch for
this model -- `step`, the actor and critic calls, the rollout, the update, the Fisher products and the critic hooks --
is preceded by `apply_net_spec()`, so models with different specs can alternate in one process.

The reference's model API on a trained policy -- `step` / `forward`, `actor.predict / forward / log_prob / std` and
`reward_critic(obs)` / `cost_critic(obs)` -- runs on one batched launch of the policy-step kernel (csrc/policy.cu,
osb_policy_step) in the model's `precision` (0 fp32, 1 tf32, 2 bf16x3; the algorithms set it from
train_cfgs.matmul_precision).  Observations are the normalised ones the networks see, `[O]` or `[..., O]`.  These calls
read `theta` and nothing else: the rollout's Philox counters, slabs and normalisers and the optimiser state are not
touched.  A stochastic action draws its noise from torch's global generator exactly as Normal.rsample does.
"""
from __future__ import annotations

import math

import numpy as np
import torch
from torch.distributions import Normal
from torch.distributions.utils import _standard_normal

from omnisafe_b200._lib import lib, ptr
from omnisafe_b200.utils.train_state import restore, snapshot

HID = 64     # the hidden width every kernel computes
# model_cfgs.*.activation (omnisafe/utils/model.py:L62-70); the index is the kernels' code (OSB_ACT_*)
ACTIVATIONS = ('tanh', 'identity', 'relu', 'sigmoid', 'softplus')
NET_ACTOR, NET_REWARD, NET_COST = 1, 2, 4   # net_mask bits of osb_policy_step
NETS = ('actor', 'reward_critic', 'cost_critic')
# model_cfgs.weight_initialization_mode -> the weight draw of utils/model.py:L25-44 (kaiming_uniform is drawn directly)
INIT_MODES = {
    'kaiming_uniform': None,
    'xavier_normal': torch.nn.init.xavier_normal_,
    'glorot': torch.nn.init.xavier_uniform_,
    'xavier_uniform': torch.nn.init.xavier_uniform_,
    'orthogonal': lambda w, generator: torch.nn.init.orthogonal_(w, gain=np.sqrt(2), generator=generator),
}


def param_layout(obs_dim: int, act_dim: int, hid: int = HID, *, actor_hidden=None, critic_hidden=None) -> dict:
    """Offsets and shapes of the flat vector [actor | reward_critic | cost_critic] in the reference's named_parameters()
    order, for two-hidden-layer networks: both layers `hid` wide, or of widths `actor_hidden` / `critic_hidden` where
    given.  The default is the kernel layout, the one `theta`, its gradient and the Adam moments always have; other
    widths give the reference layout of a narrower model."""
    O, A = obs_dim, act_dim
    a1, a2 = (hid, hid) if actor_hidden is None else actor_hidden
    c1, c2 = (hid, hid) if critic_hidden is None else critic_hidden
    actor = [('log_std', (A,)), ('mean.0.weight', (a1, O)), ('mean.0.bias', (a1,)),
             ('mean.2.weight', (a2, a1)), ('mean.2.bias', (a2,)), ('mean.4.weight', (A, a2)),
             ('mean.4.bias', (A,))]
    critic = [('critic_0.0.weight', (c1, O)), ('critic_0.0.bias', (c1,)),
              ('critic_0.2.weight', (c2, c1)), ('critic_0.2.bias', (c2,)),
              ('critic_0.4.weight', (1, c2)), ('critic_0.4.bias', (1,))]
    out, off = {}, 0
    for net, spec in (('actor', actor), ('reward_critic', critic), ('cost_critic', critic)):
        start, entries = off, {}
        for name, shape in spec:
            entries[name] = (off, shape)
            off += int(np.prod(shape))
        out[net] = {'start': start, 'size': off - start, 'entries': entries}
    out['total'] = off
    return out


class ParamMap:
    """Where the reference's parameters of networks with hidden widths `actor_hidden` [a1, a2] and `critic_hidden`
    [c1, c2] (both critics) live in the kernel layout.

    Every kernel computes 64-wide hidden layers.  A narrower network is the 64-wide one with its real weights in the
    leading rows / columns of each padded matrix and zeros everywhere else: a padded unit has z = 0 and outputs +0 (tanh,
    identity and relu map 0 to 0; for sigmoid and softplus the kernels output +0 past the layer's real width), every
    product touching a pad is +-0 in every precision, and every gradient at a pad is +-0, so Adam, clipping, the Fisher
    products and CG leave the pads at +0 and the padded network computes exactly the narrow one."""

    def __init__(self, obs_dim: int, act_dim: int, actor_hidden=(HID, HID), critic_hidden=(HID, HID)) -> None:
        for which, hs in (('actor', actor_hidden), ('critic', critic_hidden)):
            assert isinstance(hs, (list, tuple)) and len(hs) == 2 and all(
                isinstance(h, (int, np.integer)) and not isinstance(h, bool) and 1 <= h <= HID for h in hs), (
                f'model_cfgs.{which}.hidden_sizes must be exactly two hidden layers of widths 1..{HID}, got {hs!r}')
        self.actor_hidden = tuple(int(h) for h in actor_hidden)
        self.critic_hidden = tuple(int(h) for h in critic_hidden)
        self.kernel = param_layout(obs_dim, act_dim)
        self.ref = param_layout(obs_dim, act_dim, actor_hidden=self.actor_hidden, critic_hidden=self.critic_hidden)

    def views(self, theta: torch.Tensor, net: str) -> dict[str, torch.Tensor]:
        """The reference's parameters of `net` as views of a kernel-layout vector: each is the leading block of its
        padded tensor (the whole tensor at width 64, a strided view below)."""
        out = {}
        for name, (off, shape) in self.kernel[net]['entries'].items():
            block = tuple(slice(0, n) for n in self.ref[net]['entries'][name][1])
            out[name] = theta[off:off + int(np.prod(shape))].view(*shape)[block]
        return out

    def to_kernel(self, flat) -> torch.Tensor:
        """A reference-order flat vector (`ref` layout) as a kernel-layout vector with zero pads."""
        flat = torch.as_tensor(flat)
        assert flat.shape == (self.ref['total'],), f'expected a flat vector of {self.ref["total"]}, got {tuple(flat.shape)}'
        theta = torch.zeros(self.kernel['total'], dtype=flat.dtype, device=flat.device)
        for net in NETS:
            for name, view in self.views(theta, net).items():
                off, shape = self.ref[net]['entries'][name]
                view.copy_(flat[off:off + view.numel()].view(shape))
        return theta

    def to_ref(self, theta) -> torch.Tensor:
        """A kernel-layout vector as the reference-order flat vector (pads dropped)."""
        theta = torch.as_tensor(theta)
        return torch.cat([v.reshape(-1) for net in NETS for v in self.views(theta, net).values()])

    def state_dict(self, theta: torch.Tensor, net: str) -> dict[str, torch.Tensor]:
        """`net`'s parameters under the reference's names and shapes: contiguous CPU copies."""
        return {k: v.detach().cpu().contiguous().clone() for k, v in self.views(theta, net).items()}

    def load_state_dict(self, theta: torch.Tensor, net: str, state: dict, what: str = '') -> None:
        """Copy a reference-shaped state dict of `net` into its blocks of the kernel-layout `theta` (pads untouched)."""
        for name, view in self.views(theta, net).items():
            assert name in state, f'{what or net} has no {name!r}'
            w = torch.as_tensor(state[name])
            assert tuple(w.shape) == tuple(view.shape), (
                f'{what or net}.{name} has shape {tuple(w.shape)}, expected {tuple(view.shape)}')
            view.copy_(w)


def activation_code(name, which: str) -> int:
    """The kernel code of `model_cfgs.<which>.activation`; any other name fails as utils/model.py:L69 does."""
    assert name in ACTIVATIONS, f'model_cfgs.{which}.activation must be one of {ACTIVATIONS}, got {name!r}'
    return ACTIVATIONS.index(name)


def set_net_spec(actor_act: int, critic_act: int, actor_hidden, critic_hidden) -> None:
    """The activations and real hidden widths the following kernel launches compute with (osb_set_net_spec)."""
    lib().osb_set_net_spec(int(actor_act), int(critic_act), *(int(h) for h in actor_hidden),
                           *(int(h) for h in critic_hidden))


class ConstraintActorCritic:
    NETS = NETS

    def __init__(self, obs_dim: int, act_dim: int, model_cfgs, epochs: int, device='cuda',
                 generator: torch.Generator | None = None) -> None:
        self.param_map = ParamMap(obs_dim, act_dim, model_cfgs.actor.hidden_sizes, model_cfgs.critic.hidden_sizes)
        self.activation = (model_cfgs.actor.activation, model_cfgs.critic.activation)
        self.net_spec = (activation_code(model_cfgs.actor.activation, 'actor'),
                         activation_code(model_cfgs.critic.activation, 'critic'),
                         self.param_map.actor_hidden, self.param_map.critic_hidden)
        assert model_cfgs.actor_type == 'gaussian_learning'
        self.init_mode = model_cfgs.weight_initialization_mode
        if self.init_mode not in INIT_MODES:
            raise TypeError(f'Invalid initialization function: {self.init_mode}')   # utils/model.py:L44
        self.obs_dim, self.act_dim = int(obs_dim), int(act_dim)
        self.device = torch.device(device)
        self.layout = self.param_map.kernel
        P = self.layout['total']
        self.theta = torch.zeros(P, dtype=torch.float32, device=self.device)
        self.grad = torch.zeros(P, dtype=torch.float32, device=self.device)
        self.adam_m = torch.zeros(P, dtype=torch.float32, device=self.device)
        self.adam_v = torch.zeros(P, dtype=torch.float32, device=self.device)
        self.adam_step = torch.zeros(4, dtype=torch.int32, device=self.device)  # per-net step counts
        self.actor_lr0 = model_cfgs.actor.lr
        self.critic_lr = model_cfgs.critic.lr
        self.linear_lr_decay = bool(model_cfgs.linear_lr_decay)
        self.epochs = max(int(epochs), 1)
        self._sched_epoch = 0
        self._init_parameters(generator)
        self.precision = 2   # arithmetic of step / actor / critics: 0 fp32, 1 tf32, 2 bf16x3
        self.actor = GaussianLearningActor(self)
        self.reward_critic = VCritic(self, NET_REWARD)
        self.cost_critic = VCritic(self, NET_COST)

    # -- initialisation (utils/model.py:L25-44: initialize_layer on each weight; torch default bias) ----------------------
    def _init_parameters(self, generator) -> None:
        """Each layer's real block drawn with its real fans, weight then bias, layer by layer; the pads stay 0.
        kaiming_uniform_(a=sqrt(5)) is U(+-1/sqrt(fan_in)); the other modes are torch.nn.init's on the real block."""
        theta = torch.zeros(self.layout['total'], dtype=torch.float32)
        for net in self.NETS:
            views = self.param_map.views(theta, net)
            names = list(views)
            for wname, bname in zip(names[-6::2], names[-5::2]):
                w, b = views[wname], views[bname]
                fan_in = w.shape[1]
                if self.init_mode == 'kaiming_uniform':
                    bw = math.sqrt(6.0 / ((1.0 + 5.0) * fan_in))
                    w.copy_(torch.empty(w.shape).uniform_(-bw, bw, generator=generator))
                else:
                    w.copy_(INIT_MODES[self.init_mode](torch.empty(w.shape), generator=generator))
                bb = 1.0 / math.sqrt(fan_in)
                b.copy_(torch.empty(b.shape).uniform_(-bb, bb, generator=generator))
        self.theta.copy_(theta)

    def apply_net_spec(self) -> None:
        """Make this model's activations and widths the ones the next kernel launches use."""
        set_net_spec(*self.net_spec)

    # -- views ------------------------------------------------------------------------------
    def net_slice(self, net: str) -> slice:
        e = self.layout[net]
        return slice(e['start'], e['start'] + e['size'])

    def named_views(self, net: str) -> dict[str, torch.Tensor]:
        """`net`'s parameters under the reference's names and shapes, as views of `theta`."""
        return self.param_map.views(self.theta, net)

    def actor_state_dict(self) -> dict[str, torch.Tensor]:
        return self.param_map.state_dict(self.theta, 'actor')

    def load_flat(self, theta) -> None:
        """Load a kernel-layout vector (ParamMap.to_kernel makes one from the reference's flat order)."""
        self.theta.copy_(torch.as_tensor(theta, dtype=torch.float32))

    # -- learning-rate schedule (actor_critic.py:L99-113: LinearLR 1 -> 0 over `epochs`) ------
    @property
    def actor_lr(self) -> float:
        if self.actor_lr0 is None:
            return 0.0
        if not self.linear_lr_decay:
            return float(self.actor_lr0)
        frac = 1.0 - min(self._sched_epoch, self.epochs) / self.epochs
        return float(self.actor_lr0) * frac

    def actor_scheduler_step(self) -> None:
        self._sched_epoch += 1

    # -- training state (the reference-format actor_state_dict() stays what epoch-k.pt holds) -----
    def train_state(self) -> dict:
        """Parameters, Adam moments, per-network Adam step counts and the LinearLR epoch."""
        theta, m, v, step = snapshot(self.theta, self.adam_m, self.adam_v, self.adam_step)
        return {'theta': theta, 'adam_m': m, 'adam_v': v, 'adam_step': step, 'sched_epoch': self._sched_epoch}

    def load_train_state(self, state: dict) -> None:
        for k in ('theta', 'adam_m', 'adam_v', 'adam_step'):
            restore(getattr(self, k), state[k], f'model {k}')
        self._sched_epoch = int(state['sched_epoch'])

    # -- acting (constraint_actor_critic.py:L84-109) ----------------------------------------------
    def step(self, obs, deterministic: bool = False) -> tuple[torch.Tensor, ...]:
        """(action, value_r, value_c, log_prob) of `obs` in one launch: the action is the mean when `deterministic`,
        otherwise mean + std * eps with eps drawn as Normal.rsample draws it."""
        obs, lead = self._flat_obs(obs)
        eps = None if deterministic else self._draw_eps(lead)
        out = self._launch(obs, NET_ACTOR | NET_REWARD | NET_COST, eps=eps, act=True, logp=True)
        self.actor._after_inference = False   # predict + log_prob, as the reference's step leaves the actor
        return (out['act'].view(*lead, self.act_dim), out['value_r'].view(lead), out['value_c'].view(lead),
                out['logp'].view(lead))

    def forward(self, obs, deterministic: bool = False) -> tuple[torch.Tensor, ...]:
        return self.step(obs, deterministic=deterministic)

    __call__ = forward

    def _flat_obs(self, obs) -> tuple[torch.Tensor, torch.Size]:
        obs = torch.as_tensor(obs).to(device=self.device, dtype=torch.float32)
        assert obs.dim() >= 1 and obs.shape[-1] == self.obs_dim, (
            f'observations must be [{self.obs_dim}] or [..., {self.obs_dim}], got {tuple(obs.shape)}')
        return obs.reshape(-1, self.obs_dim).contiguous(), obs.shape[:-1]

    def _draw_eps(self, lead: torch.Size) -> torch.Tensor:
        # the draw Normal(mean, std).rsample() makes for a [..., A] batch (torch/distributions/normal.py)
        return _standard_normal((*lead, self.act_dim), dtype=torch.float32, device=self.device).reshape(-1, self.act_dim)

    def _launch(self, obs: torch.Tensor, net_mask: int, eps=None, act_in=None, mean=False, act=False,
                logp=False) -> dict[str, torch.Tensor]:
        """One osb_policy_step launch on rows obs[B][O]; returns the requested outputs, flat ([B][A] / [B])."""
        B, A = obs.shape[0], self.act_dim
        new = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=self.device)   # noqa: E731
        out = {}
        if net_mask & NET_ACTOR:
            if mean:
                out['mean'] = new(B, A)
            if act:
                out['act'] = new(B, A)
            if logp:
                out['logp'] = new(B)
        if net_mask & NET_REWARD:
            out['value_r'] = new(B)
        if net_mask & NET_COST:
            out['value_c'] = new(B)
        if B == 0:
            return out
        self.apply_net_spec()
        with torch.cuda.device(self.device):
            lib().osb_policy_step(
                ptr(self.theta), self.obs_dim, A, B, ptr(obs), ptr(eps), ptr(act_in), net_mask, int(self.precision),
                ptr(out.get('mean')), ptr(out.get('act')), ptr(out.get('logp')), ptr(out.get('value_r')),
                ptr(out.get('value_c')), torch.cuda.current_stream(self.device).cuda_stream)
        return out


class GaussianLearningActor:
    """models/actor/gaussian_learning_actor.py:L64-139 on the policy-step kernel: the mean network and the
    state-independent `log_std` are the actor's slice of the model's `theta`."""

    def __init__(self, model: ConstraintActorCritic) -> None:
        self._model = model
        self._after_inference = False
        self._current_obs: torch.Tensor | None = None
        self._current_lead: torch.Size | None = None

    def _log_std(self) -> torch.Tensor:
        m = self._model
        off, shape = m.layout['actor']['entries']['log_std']
        return m.theta[off:off + shape[0]]

    def _remember(self, obs: torch.Tensor, lead: torch.Size) -> None:
        self._current_obs, self._current_lead = obs, lead
        self._after_inference = True

    def predict(self, obs, deterministic: bool = False) -> torch.Tensor:
        """The mean if `deterministic`, else a sample of Normal(mean, std) (rsample's noise draw)."""
        m = self._model
        obs, lead = m._flat_obs(obs)
        eps = None if deterministic else m._draw_eps(lead)
        act = m._launch(obs, NET_ACTOR, eps=eps, act=True)['act']
        self._remember(obs, lead)
        return act.view(*lead, m.act_dim)

    def forward(self, obs) -> Normal:
        """Normal(mean(obs), exp(log_std))."""
        m = self._model
        obs, lead = m._flat_obs(obs)
        mean = m._launch(obs, NET_ACTOR, mean=True)['mean']
        self._remember(obs, lead)
        return Normal(mean.view(*lead, m.act_dim), torch.exp(self._log_std()))

    __call__ = forward

    def log_prob(self, act) -> torch.Tensor:
        """Summed log-probability of `act` under the distribution of the last predict / forward."""
        assert self._after_inference, 'log_prob() should be called after predict() or forward()'
        self._after_inference = False
        m = self._model
        act = torch.as_tensor(act).to(device=m.device, dtype=torch.float32)
        assert act.shape == (*self._current_lead, m.act_dim), (
            f'act must be {(*self._current_lead, m.act_dim)} like the last predict / forward, got {tuple(act.shape)}')
        act_in = act.reshape(-1, m.act_dim).contiguous()
        return m._launch(self._current_obs, NET_ACTOR, act_in=act_in, logp=True)['logp'].view(self._current_lead)

    @property
    def std(self) -> float:
        return torch.exp(self._log_std()).mean().item()

    @std.setter
    def std(self, std: float) -> None:
        self._log_std().fill_(torch.log(torch.tensor(std, device=self._model.device)))


class VCritic:
    """models/critic/v_critic.py:L75-92 (one critic): `critic(obs)` returns the list [value], value = [...]."""

    def __init__(self, model: ConstraintActorCritic, net_bit: int) -> None:
        self._model = model
        self._bit = net_bit

    def forward(self, obs) -> list[torch.Tensor]:
        m = self._model
        obs, lead = m._flat_obs(obs)
        out = m._launch(obs, self._bit)
        return [out['value_r' if self._bit == NET_REWARD else 'value_c'].view(lead)]

    __call__ = forward
