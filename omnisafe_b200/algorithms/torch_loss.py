"""Actor objectives written in PyTorch on the kernel update path.

A subclass that overrides `_loss_pi`, `_compute_adv_surrogate` or `_loss_pi_cost` trains its actor through autograd on
that loss; everything else of the update (critics, clipping, rank averaging, Adam, KL early stop, Fisher-vector
products, CG) stays on the kernels.  The actor mean mu(obs) is a `torch.autograd.Function`: forward on the actor-
evaluation kernel of the run's precision, backward on the supplied-dmu kernel (osb_actor_dmu_backward, loss kind
LOSS_DMU), so the objective sees exactly the network the fused path trains.
"""
from __future__ import annotations

import contextlib

import torch
from torch.distributions import Normal

from omnisafe_b200._lib import current_stream, lib, ptr

HOOKS = ('_loss_pi', '_compute_adv_surrogate', '_loss_pi_cost')
_LIBRARY = 'omnisafe_b200'


def overridden_hooks(cls: type) -> list[tuple[str, str]]:
    """[(hook, defining class)] for every actor hook `cls` takes from a class defined outside the library."""
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


class DeviceStats:
    """Logger values stored by PyTorch losses, kept on the device until the epoch is logged (one read per epoch)."""

    def __init__(self) -> None:
        self._vals: dict[str, list[torch.Tensor]] = {}

    def store(self, data: dict) -> None:
        for key, val in data.items():
            t = torch.as_tensor(val).detach().to(torch.float32).mean().reshape(1)
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
