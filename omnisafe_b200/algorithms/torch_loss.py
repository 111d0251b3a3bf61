"""Actor and critic objectives written in PyTorch on the kernel update path.

A subclass that overrides `_loss_pi`, `_compute_adv_surrogate` or `_loss_pi_cost` trains its actor through autograd on
that loss; the clipping, rank averaging, Adam, KL early stop, Fisher-vector products and CG stay on the kernels.  The
actor mean mu(obs) is a `torch.autograd.Function`: forward on the actor-evaluation kernel of the run's precision,
backward on the supplied-dmu kernel (osb_actor_dmu_backward, loss kind LOSS_DMU), so the objective sees exactly the
network the fused path trains.

A subclass that overrides `_update_reward_critic` or `_update_cost_critic` trains that critic with its own minibatch
step.  While it runs, the critic is a `TrainingCritic`: V(obs) forward and backward on the supplied-dV kernel
(osb_critic_dv_backward, the update kernels of the run's precision), leaf parameters that are views of the flat
`theta`, and an optimiser whose step() is the library's Adam on that network.  Networks without a hook keep their
kernel step.
"""
from __future__ import annotations

import contextlib

import torch
from torch.distributions import Normal

from omnisafe_b200._lib import current_stream, lib, ptr

ACTOR_HOOKS = ('_loss_pi', '_compute_adv_surrogate', '_loss_pi_cost')
CRITIC_HOOKS = ('_update_reward_critic', '_update_cost_critic')
HOOKS = ACTOR_HOOKS + CRITIC_HOOKS
_LIBRARY = 'omnisafe_b200'


def overridden_hooks(cls: type) -> list[tuple[str, str]]:
    """[(hook, defining class)] for every hook `cls` takes from a class defined outside the library."""
    found = []
    for name in HOOKS:
        for klass in cls.__mro__:
            if name in vars(klass):
                mod = klass.__module__ or ''
                if mod != _LIBRARY and not mod.startswith(_LIBRARY + '.'):
                    found.append((name, f'{mod}.{klass.__qualname__}'))
                break
    return found


class ActorMean(torch.autograd.Function):
    """mu [B, A] of rows obs [B, O] (contiguous, normalised) under the flat actor parameters theta_actor [P_actor].
    The gradient is J^T dmu on the MLP entries and zero on log_std (its gradient comes from the Normal built on top)."""

    @staticmethod
    def forward(ctx, obs: torch.Tensor, theta_actor: torch.Tensor, engine) -> torch.Tensor:
        B, A = obs.shape[0], engine.A
        mu = torch.empty(B, A, dtype=torch.float32, device=obs.device)
        if B > 0:
            engine.agent.apply_net_spec()
            engine._eval_fn()(ptr(theta_actor), engine.O, A, ptr(obs), 0, 0, 0, 0, 0, 0, 0, 0, B, 1, ptr(mu), 0, 0,
                              current_stream())
        ctx.save_for_backward(obs, theta_actor)
        ctx.engine = engine
        return mu

    @staticmethod
    def backward(ctx, dmu: torch.Tensor):
        obs, theta_actor = ctx.saved_tensors
        e = ctx.engine
        grad = torch.zeros(e.Pa, dtype=torch.float32, device=obs.device)
        B = obs.shape[0]
        if B > 0:
            dmu = dmu.to(torch.float32).contiguous()
            nb = lib().osb_actor_dmu_grid_blocks(B, e.O, e.precision)
            s = current_stream()
            e.agent.apply_net_spec()
            lib().osb_actor_dmu_backward(ptr(theta_actor), e.O, e.A, ptr(obs), ptr(dmu), B, e.precision,
                                         ptr(e.fvp_part), ptr(e.stats_part), s)
            lib().osb_reduce_partials(ptr(e.fvp_part), nb, e.Pa, e.Pa, 1.0, 0, 0.0, ptr(grad), s)
        return None, grad, None


class TrainingActor:
    """What `self._actor_critic.actor` is while a PyTorch actor loss runs: the reference's GaussianLearningActor API
    (`actor(obs)` -> Normal, `log_prob(act)`, `std`, `log_std`), differentiable in the flat actor parameters `theta`."""

    def __init__(self, engine, theta: torch.Tensor) -> None:
        self._engine, self.theta = engine, theta
        self._dist: Normal | None = None

    @property
    def log_std(self) -> torch.Tensor:
        return self.theta[: self._engine.A]

    def forward(self, obs: torch.Tensor) -> Normal:
        e = self._engine
        assert obs.dim() == 2 and obs.shape[1] == e.O, f'obs must be [B, {e.O}], got {tuple(obs.shape)}'
        mu = ActorMean.apply(obs.to(torch.float32).contiguous(), self.theta, e)
        self._dist = Normal(mu, torch.exp(self.log_std), validate_args=False)   # no host read per call
        return self._dist

    __call__ = forward

    def log_prob(self, act: torch.Tensor) -> torch.Tensor:
        assert self._dist is not None, 'log_prob() should be called after forward()'
        dist, self._dist = self._dist, None
        return dist.log_prob(act).sum(-1)

    @property
    def std(self) -> float:
        return torch.exp(self.log_std).mean().item()


@contextlib.contextmanager
def training_actor(model, engine, theta: torch.Tensor):
    """Swap `model.actor` for a TrainingActor on `theta` for the duration of one loss evaluation."""
    saved = model.actor
    model.actor = TrainingActor(engine, theta)
    try:
        yield model.actor
    finally:
        model.actor = saved


class CriticValue(torch.autograd.Function):
    """V [B] of rows obs [B, O] (contiguous, normalised) for a TrainingCritic; differentiable in its leaf parameters
    (`params`, views of the flat theta the kernels read).  Forward and backward are osb_critic_dv_backward, the update
    kernels of the run's precision on that critic: the forward with dV = 0 gives the values with the bits the stepwise
    update computes; the gradient is J_V^T dV of the critic MLP."""

    @staticmethod
    def forward(ctx, obs: torch.Tensor, critic, *params: torch.Tensor) -> torch.Tensor:
        B = obs.shape[0]
        value = torch.empty(B, dtype=torch.float32, device=obs.device)
        if B > 0:
            critic._launch(obs, torch.zeros(B, dtype=torch.float32, device=obs.device), value)
        ctx.save_for_backward(obs)
        ctx.critic = critic
        return value

    @staticmethod
    def backward(ctx, dv: torch.Tensor):
        (obs,) = ctx.saved_tensors
        c = ctx.critic
        e = c._engine
        grad = torch.zeros(e.P, dtype=torch.float32, device=obs.device)   # kernel layout, so the pads are in place
        B = obs.shape[0]
        if B > 0:
            nb = c._launch(obs, dv.to(torch.float32).contiguous(), None)
            lib().osb_reduce_partials(ptr(e.gpart[c.start:]), nb, e.P, c.size, 1.0, 0, 0.0, ptr(grad[c.start:]),
                                      current_stream())
        return (None, None, *c._pmap.views(grad, c.name).values())


class TrainingCritic:
    """What `self._actor_critic.reward_critic` / `.cost_critic` is while a critic hook runs: the reference's VCritic API
    (`critic(obs)` -> [value]) and nn.Module's `parameters()` / `named_parameters()`: leaf tensors with the reference's
    names, shapes and order that are views of the network's blocks of the flat `theta` (ParamMap.views; strided for
    hidden widths below 64), so they always hold what the kernels train."""

    def __init__(self, engine, net: int) -> None:
        self._engine, self.net = engine, net            # net: 1 reward critic, 2 cost critic
        self.name = 'reward_critic' if net == 1 else 'cost_critic'
        agent = engine.agent
        self._pmap = agent.param_map
        lay = agent.layout[self.name]
        self.start, self.size = lay['start'], lay['size']
        self._named = [(name, v.requires_grad_(True)) for name, v in self._pmap.views(agent.theta, self.name).items()]
        self._params = [p for _, p in self._named]

    def _launch(self, obs: torch.Tensor, dv: torch.Tensor, value: torch.Tensor | None) -> int:
        """osb_critic_dv_backward on rows obs [B, O] into the engine's partials; returns their row count."""
        e = self._engine
        B = obs.shape[0]
        e.agent.apply_net_spec()
        lib().osb_critic_dv_backward(ptr(e.agent.theta), e.O, e.A, self.net, ptr(obs), ptr(dv), ptr(value), B,
                                     e.precision, ptr(e.gpart), ptr(e.stats_part), current_stream())
        return lib().osb_critic_dv_grid_blocks(B, e.O, e.precision)

    def forward(self, obs: torch.Tensor) -> list[torch.Tensor]:
        e = self._engine
        assert obs.shape[-1] == e.O, f'obs must be [..., {e.O}], got {tuple(obs.shape)}'
        lead = obs.shape[:-1]
        flat = obs.to(torch.float32).reshape(-1, e.O).contiguous()
        return [CriticValue.apply(flat, self, *self._params).view(lead)]

    __call__ = forward

    def parameters(self):
        return iter(self._params)

    def named_parameters(self):
        return iter(self._named)

    def flat_grad(self) -> torch.Tensor:
        """The leaves' gradients as the network's slice of the kernel layout: zero where a leaf has none and at the
        pads."""
        grad = torch.zeros(self._engine.P, dtype=torch.float32, device=self._params[0].device)
        for g, p in zip(self._pmap.views(grad, self.name).values(), self._params):
            if p.grad is not None:
                g.copy_(p.grad)
        return grad[self.start:self.start + self.size]


class TrainingCriticOptimizer:
    """What `reward_critic_optimizer` / `cost_critic_optimizer` is while a critic hook runs: zero_grad() and step(),
    the library's Adam on the network's slice of theta with its own step count and the critic learning rate (the Adam
    state the fused path trains, saves and resumes).  No clipping and no L2 term are added: the hook's are the only
    ones."""

    def __init__(self, critic: TrainingCritic, lr: float) -> None:
        self._critic, self.lr = critic, float(lr)

    def zero_grad(self, set_to_none: bool = True) -> None:
        for p in self._critic.parameters():
            if set_to_none:
                p.grad = None
            elif p.grad is not None:
                p.grad.zero_()

    def step(self) -> None:
        c = self._critic
        c._engine.adam_step(c.net, c.flat_grad(), self.lr)


class HookLogger:
    """What `self._logger` is while a critic hook runs: `store` keeps the values on the device (DeviceStats) until the
    epoch is logged; everything else is the logger's."""

    def __init__(self, logger, stats: 'DeviceStats') -> None:
        self._logger, self._stats = logger, stats

    def store(self, data: dict | None = None, **kwargs) -> None:
        self._stats.store({**(data or {}), **kwargs})

    def __getattr__(self, name: str):
        return getattr(self._logger, name)


@contextlib.contextmanager
def training_critic(algo, net: int, lr: float):
    """Swap the model's critic `net` (1 reward, 2 cost) and its optimiser for a TrainingCritic and its optimiser, and
    `algo._logger` for a HookLogger, for the duration of one critic hook."""
    model, name = algo._actor_critic, 'reward_critic' if net == 1 else 'cost_critic'
    saved = getattr(model, name), getattr(model, f'{name}_optimizer', None), algo._logger
    critic = TrainingCritic(algo._engine, net)
    setattr(model, name, critic)
    setattr(model, f'{name}_optimizer', TrainingCriticOptimizer(critic, lr))
    algo._logger = HookLogger(saved[2], algo._loss_stats)
    try:
        yield critic
    finally:
        setattr(model, name, saved[0])
        if saved[1] is None:
            delattr(model, f'{name}_optimizer')
        else:
            setattr(model, f'{name}_optimizer', saved[1])
        algo._logger = saved[2]


class DeviceStats:
    """Logger values stored by PyTorch losses, kept on the device until the epoch is logged (one read per epoch).
    Python numbers are stored on `device`."""

    def __init__(self, device=None) -> None:
        self._vals: dict[str, list[torch.Tensor]] = {}
        self._device = device

    def store(self, data: dict) -> None:
        for key, val in data.items():
            t = torch.as_tensor(val, device=None if torch.is_tensor(val) else self._device)
            t = t.detach().to(torch.float32).mean().reshape(1)
            self._vals.setdefault(key, []).append(t)

    def clear(self) -> None:
        self._vals.clear()

    def means(self) -> dict[str, float]:
        if not self._vals:
            return {}
        keys = list(self._vals)
        means = torch.cat([torch.cat(self._vals[k]).mean().reshape(1) for k in keys]).tolist()
        return dict(zip(keys, means))


def _mix32(x: torch.Tensor) -> torch.Tensor:
    m = 0xFFFFFFFF
    x = x ^ (x >> 16)
    x = (x * 0x7FEB352D) & m
    x = x ^ (x >> 15)
    x = (x * 0x846CA68B) & m
    return x ^ (x >> 16)


def feistel_order(n: int, seed: int, device) -> torch.Tensor:
    """The sample order the update kernels draw without a supplied permutation (csrc/loss.cuh feistel_perm): a keyed
    4-round Feistel bijection on the enclosing power-of-four domain with cycle walking.  int64 [n]."""
    bits = 2
    while (1 << bits) < n:
        bits += 2
    half = bits >> 1
    mask = (1 << half) - 1
    keys = [(seed + 0x9E3779B9 * (r + 1)) & 0xFFFFFFFF for r in range(4)]
    out = torch.empty(n, dtype=torch.int64, device=device)
    pos = torch.arange(n, dtype=torch.int64, device=device)
    x = pos.clone()
    while pos.numel():
        left, right = (x >> half) & mask, x & mask
        for key in keys:
            left, right = right, left ^ (_mix32(right ^ key) & mask)
        x = (left << half) | right
        ok = x < n
        out[pos[ok]] = x[ok]
        pos, x = pos[~ok], x[~ok]
    return out
