"""Flat-parameter ConstraintActorCritic (actor + reward critic + cost critic).

Mirrors omnisafe/models/actor_critic/constraint_actor_critic.py:L31-109 and
actor_critic.py:L60-113: three independent Linear-Tanh-Linear-Tanh-Linear trunks
(utils/model.py:L73-111), GaussianLearningActor with a state-independent `log_std`
(models/actor/gaussian_learning_actor.py:L29-62), one Adam optimiser per network and a LinearLR
decay of the actor learning rate.  All parameters live in ONE flat fp32 device vector
`theta = [actor | reward_critic | cost_critic]` in the reference's named_parameters() order
(utils/tools.py:L35-129), so the CG vector layout, the flat gradient all-reduce and the fused
kernels share it.  `actor_state_dict()` re-exports the actor under the reference's key names so
`{'pi': ..., 'obs_normalizer': ...}` checkpoints stay loadable by the reference Evaluator
(omnisafe/evaluator.py:L153-178, algorithms/on_policy/base/policy_gradient.py:L183-189).

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

HID = 64
NET_ACTOR, NET_REWARD, NET_COST = 1, 2, 4   # net_mask bits of osb_policy_step


def param_layout(obs_dim: int, act_dim: int, hid: int = HID) -> dict:
    O, A = obs_dim, act_dim
    actor = [('log_std', (A,)), ('mean.0.weight', (hid, O)), ('mean.0.bias', (hid,)),
             ('mean.2.weight', (hid, hid)), ('mean.2.bias', (hid,)), ('mean.4.weight', (A, hid)),
             ('mean.4.bias', (A,))]
    critic = [('critic_0.0.weight', (hid, O)), ('critic_0.0.bias', (hid,)),
              ('critic_0.2.weight', (hid, hid)), ('critic_0.2.bias', (hid,)),
              ('critic_0.4.weight', (1, hid)), ('critic_0.4.bias', (1,))]
    out, off = {}, 0
    for net, spec in (('actor', actor), ('reward_critic', critic), ('cost_critic', critic)):
        start, entries = off, {}
        for name, shape in spec:
            entries[name] = (off, shape)
            off += int(np.prod(shape))
        out[net] = {'start': start, 'size': off - start, 'entries': entries}
    out['total'] = off
    return out


class ConstraintActorCritic:
    NETS = ('actor', 'reward_critic', 'cost_critic')

    def __init__(self, obs_dim: int, act_dim: int, model_cfgs, epochs: int, device='cuda',
                 generator: torch.Generator | None = None) -> None:
        hs_a = list(model_cfgs.actor.hidden_sizes)
        hs_c = list(model_cfgs.critic.hidden_sizes)
        assert hs_a == [HID, HID] and hs_c == [HID, HID], (
            'the fused sm_90a kernels are specialised for hidden_sizes [64, 64]')
        assert model_cfgs.actor.activation == 'tanh' and model_cfgs.critic.activation == 'tanh', (
            'the fused kernels implement tanh activations')
        assert model_cfgs.actor_type == 'gaussian_learning'
        assert model_cfgs.weight_initialization_mode == 'kaiming_uniform'
        self.obs_dim, self.act_dim = int(obs_dim), int(act_dim)
        self.device = torch.device(device)
        self.layout = param_layout(obs_dim, act_dim)
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

    # -- initialisation (utils/model.py:L25-44: kaiming_uniform_(a=sqrt(5)); torch default bias)
    def _init_parameters(self, generator) -> None:
        theta = torch.zeros(self.layout['total'], dtype=torch.float32)
        for net in self.NETS:
            ent = self.layout[net]['entries']
            names = list(ent)
            for wname, bname in zip(names[-6::2], names[-5::2]):
                off, shape = ent[wname]
                fan_in = shape[1]
                bw = math.sqrt(6.0 / ((1.0 + 5.0) * fan_in))
                theta[off:off + shape[0] * shape[1]].uniform_(-bw, bw, generator=generator)
                boff, bshape = ent[bname]
                bb = 1.0 / math.sqrt(fan_in)
                theta[boff:boff + bshape[0]].uniform_(-bb, bb, generator=generator)
        self.theta.copy_(theta)

    # -- views ------------------------------------------------------------------------------
    def net_slice(self, net: str) -> slice:
        e = self.layout[net]
        return slice(e['start'], e['start'] + e['size'])

    def named_views(self, net: str) -> dict[str, torch.Tensor]:
        return {name: self.theta[off:off + int(np.prod(shape))].view(*shape)
                for name, (off, shape) in self.layout[net]['entries'].items()}

    def actor_state_dict(self) -> dict[str, torch.Tensor]:
        return {k: v.detach().cpu().clone() for k, v in self.named_views('actor').items()}

    def load_flat(self, theta) -> None:
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
