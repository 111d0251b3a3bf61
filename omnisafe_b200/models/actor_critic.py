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
"""
from __future__ import annotations

import math

import numpy as np
import torch

HID = 64


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
