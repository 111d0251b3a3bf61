"""Running observation normaliser state (device resident).

Mirrors omnisafe/common/normalizer.py:L25-158: `_mean`, `_sumsq`, `_var`, `_std`, `_count`, `_clip`
are exposed through state_dict() with the reference's key names so checkpoints stay loadable by
the reference Evaluator (omnisafe/evaluator.py:L153-178).  The update itself (Normalizer._push) is
fused into the rollout kernels (csrc/rollout.cu: norm_fold on the synthetic env, the observe kernels on a registered
env; the fp32 update itself in csrc/normalizer.cuh).
"""
from __future__ import annotations

import torch

from omnisafe_b200.utils.train_state import restore, snapshot


class Normalizer:
    def __init__(self, shape: tuple[int, ...], clip: float = 5.0, device='cuda') -> None:
        assert len(shape) == 1, 'the fused path normalises flat Box observations'
        O, dev = shape[0], torch.device(device)
        self._shape = tuple(shape)
        self.clip = float(clip)
        self.mean = torch.zeros(O, dtype=torch.float32, device=dev)
        self.sumsq = torch.zeros(O, dtype=torch.float32, device=dev)
        self.std = torch.zeros(O, dtype=torch.float32, device=dev)
        self.mean1 = torch.zeros(O, dtype=torch.float32, device=dev)
        self.std1 = torch.zeros(O, dtype=torch.float32, device=dev)
        self.count = torch.zeros(2, dtype=torch.int64, device=dev)
        self.acc_all = torch.zeros(2, O, dtype=torch.int64, device=dev)
        self.acc_fin = torch.zeros(2, O, dtype=torch.int64, device=dev)
        self.fin_count = torch.zeros(1, dtype=torch.int32, device=dev)
        self.had_fin = torch.zeros(1, dtype=torch.int32, device=dev)
        self.ticket = torch.zeros(1, dtype=torch.int32, device=dev)

    @property
    def shape(self) -> tuple[int, ...]:
        return self._shape

    def ptrs(self) -> list:
        return [t.data_ptr() for t in (self.mean, self.sumsq, self.std, self.mean1, self.std1,
                                       self.count, self.acc_all, self.acc_fin, self.fin_count,
                                       self.had_fin, self.ticket)]

    def state_dict(self) -> dict[str, torch.Tensor]:
        count = self.count[0]
        var = self.sumsq / (count - 1).clamp(min=1).to(torch.float32)
        return {
            '_mean': self.mean.detach().cpu().clone(),
            '_sumsq': self.sumsq.detach().cpu().clone(),
            '_var': var.detach().cpu(),
            '_std': self.std.detach().cpu().clone(),
            '_count': count.detach().cpu().clone(),
            '_clip': self.clip * torch.ones(self._shape),
        }

    def load_state_dict(self, sd: dict[str, torch.Tensor]) -> None:
        self.mean.copy_(sd['_mean']); self.sumsq.copy_(sd['_sumsq']); self.std.copy_(sd['_std'])
        self.count[0] = int(sd['_count'])

    _STATE = ('mean', 'sumsq', 'std', 'mean1', 'std1', 'count', 'acc_all', 'acc_fin', 'fin_count', 'had_fin', 'ticket')

    def train_state(self) -> dict[str, torch.Tensor]:
        """Every tensor the rollout kernels carry from step to step (state_dict() keeps the reference's subset)."""
        return dict(zip(self._STATE, snapshot(*(getattr(self, k) for k in self._STATE))))

    def load_train_state(self, state: dict) -> None:
        for k in self._STATE:
            restore(getattr(self, k), state[k], f'obs normaliser {k}')


class ScalarNormalizer:
    """`Normalizer(shape=(), clip=5)` of RewardNormalize / CostNormalize (envs/wrapper.py:L280-423) with its
    state on the device; one call normalises a whole epoch's slab in the reference's per-step order
    (`osb_scalar_normalize_rows`, csrc/scalar_norm.cu).  state_dict() uses the reference's key names."""

    def __init__(self, clip: float = 5.0, device='cuda') -> None:
        dev = torch.device(device)
        self.clip = float(clip)
        self.state = torch.zeros(4, dtype=torch.float32, device=dev)      # mean, sumsq, std, -
        self.count = torch.zeros(1, dtype=torch.int64, device=dev)
        self._ws = None

    @property
    def mean(self) -> torch.Tensor:
        return self.state[0]

    @property
    def std(self) -> torch.Tensor:
        return self.state[2]

    def normalize_rows_(self, slab: torch.Tensor) -> None:
        """slab: [T, N] fp32, time-major, normalised in place."""
        from omnisafe_b200._lib import current_stream, lib, ptr
        assert slab.dim() == 2 and slab.dtype == torch.float32 and slab.is_contiguous()
        T, N = slab.shape
        if self._ws is None or self._ws.numel() < 4 * T:
            self._ws = torch.zeros(4 * T, dtype=torch.float32, device=slab.device)
        lib().osb_scalar_normalize_rows(ptr(slab), T, N, self.clip, ptr(self.state), ptr(self.count),
                                        ptr(self._ws), current_stream())

    def state_dict(self) -> dict[str, torch.Tensor]:
        count = self.count[0]
        var = self.state[1] / (count - 1).clamp(min=1).to(torch.float32)
        return {'_mean': self.state[0].detach().cpu().clone(), '_sumsq': self.state[1].detach().cpu().clone(),
                '_var': var.detach().cpu(), '_std': self.state[2].detach().cpu().clone(),
                '_count': count.detach().cpu().clone(), '_clip': self.clip * torch.ones(())}

    def load_state_dict(self, sd: dict[str, torch.Tensor]) -> None:
        self.state[0] = float(sd['_mean']); self.state[1] = float(sd['_sumsq']); self.state[2] = float(sd['_std'])
        self.count[0] = int(sd['_count'])

    def train_state(self) -> dict[str, torch.Tensor]:
        state, count = snapshot(self.state, self.count)
        return {'state': state, 'count': count}

    def load_train_state(self, state: dict) -> None:
        restore(self.state, state['state'], 'scalar normaliser state')
        restore(self.count, state['count'], 'scalar normaliser count')
