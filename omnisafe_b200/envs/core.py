"""User-registered CMDPs: `CMDP`, `env_register`, `make`, `support_envs` and a minimal `Box`.

Mirrors omnisafe/envs/core.py:L37-182 and L300-420 (names, class attributes, registry semantics), so a class written
against the reference `CMDP` also works here.  Such an env is stepped in PyTorch by `ExternalEnvAdapter`
(adapter/external_adapter.py); the policy step and everything after it stays on the CUDA kernels.

The env keeps the reference's multi-env contract (online_adapter.py:L52-140): `reset() -> (obs[N, O], info)`,
`step(action[N, A]) -> (obs, reward[N], cost[N], terminated[N], truncated[N], info)`, it auto-resets finished envs
itself and reports their last observation in `info['final_observation']` (rows selected by the boolean
`info['_final_observation']`; when that mask is absent every finished row is taken).  With `num_envs == 1` unbatched
tensors are accepted, as the reference's `Unsqueeze` wrapper does.  Tensors may live on the CPU or on any CUDA device.

An env may set `graph_safe = True` (an omnisafe_b200 extension, like the `need_*` flags).  The adapter then captures
the epoch's steps -- the act kernels, `env.step` and the observe kernels -- into one CUDA graph and replays it every
epoch, which removes the host's per-launch cost.  Such an env promises:
- it lives on the training CUDA device and says so in `device` (or `_device`), a CUDA `torch.device`;
- `step` and `reset` keep their state in the same storage from call to call, writing it in place (`copy_`, `out=`)
  instead of rebinding attributes: a replay reads the state the previous replay wrote.  `reset` returns the same
  storage every epoch (its state, or a fixed buffer); a new one makes the adapter capture the graph again;
- `step` does not synchronise with the host, has no data-dependent Python control flow and keeps no host-side state
  (RNG, counters) that must advance from step to step: it runs once per step at capture, never at replay;
- `info` holds `final_observation` and `_final_observation` on every step (the mask all false when nothing finished),
  so its structure is the same on every step;
- the tensors `step` returns may be fresh each call: the adapter copies them inside the graph.

An env may define `reset_envs(mask) -> obs` (optional, an omnisafe_b200 extension): a reset of some envs only.  `mask` is
an [N] bool tensor on the env's device; the masked envs start fresh episodes and the masked rows of the returned [N, O]
hold their first observations (the other rows are ignored).  An all-false mask leaves the env's state untouched; at
N = 1, `reset_envs(tensor([True]))` is equivalent to `reset()`.  For a `graph_safe` env the call must be capturable, as
`step` is: no host synchronisation, and the same output storage on every call.  The EarlyTerminated algorithms use it to
reset the envs the cost limit cuts: with it they run any number of envs (a graph-safe env keeps its epoch in the CUDA
graph); without it they run a single env only, as upstream does, resetting it through `reset()` and eagerly.

An env may also define `state_dict() -> dict` and `load_state_dict(sd)` (optional, an omnisafe_b200 extension).  When it
does, a saved training state (`AlgoWrapper.save_state`, `learn(save_state_freq=...)`) holds what `state_dict()` returns and
`Agent.resume` hands it back to `load_state_dict` right after `set_seed`, before the first epoch; a run that resumes then
continues to the same bits as one that never stopped.  `sd` holds CPU tensors (the file is loaded onto the CPU).  A
graph-safe env writes them into its existing state in place (`copy_`), since the storage is captured.  Without the hooks
the env starts the resumed run in its freshly seeded state, and only the library's own state is restored.
"""
from __future__ import annotations

import inspect
from abc import ABC, abstractmethod
from typing import Any, ClassVar

import numpy as np

from omnisafe_b200.envs.synthetic import support_envs as _synthetic_envs

MAX_ACT_DIM = 16    # OUTP of the rollout kernels: actions per env


class Box:
    """The part of `gymnasium.spaces.Box` the adapter reads: `shape`, `low`, `high` (float32 arrays of `shape`)."""

    def __init__(self, low, high, shape: tuple[int, ...] | None = None, dtype=np.float32) -> None:
        if shape is None:
            shape = np.broadcast(np.asarray(low), np.asarray(high)).shape
        self.shape = tuple(int(s) for s in shape)
        self.dtype = np.dtype(dtype)
        self.low = np.broadcast_to(np.asarray(low, np.float32), self.shape).copy()
        self.high = np.broadcast_to(np.asarray(high, np.float32), self.shape).copy()

    def __repr__(self) -> str:
        return f'Box({self.low.min()}, {self.high.max()}, {self.shape}, {self.dtype})'


class CMDP(ABC):
    """Base class of a user environment (omnisafe/envs/core.py:L37-182)."""

    _action_space: Any
    _observation_space: Any
    _metadata: dict[str, Any]

    _num_envs: int = 1
    _time_limit: int | None = None
    need_time_limit_wrapper: bool = False
    need_auto_reset_wrapper: bool = False
    need_evaluation: bool = True
    graph_safe: bool = False        # omnisafe_b200: the step may be captured into a CUDA graph (module docstring)

    _support_envs: ClassVar[list[str]]

    @classmethod
    def support_envs(cls) -> list[str]:
        return cls._support_envs

    @abstractmethod
    def __init__(self, env_id: str, **kwargs: Any) -> None:
        assert env_id in self.support_envs(), f'env_id {env_id} is not supported by {self.__class__.__name__}'

    @property
    def action_space(self):
        return self._action_space

    @property
    def observation_space(self):
        return self._observation_space

    @property
    def max_episode_steps(self) -> int | None:
        return None

    @property
    def metadata(self) -> dict[str, Any]:
        return getattr(self, '_metadata', {})

    @property
    def num_envs(self) -> int:
        return self._num_envs

    @property
    def time_limit(self) -> int | None:
        return self._time_limit

    @abstractmethod
    def step(self, action):
        """-> (obs, reward, cost, terminated, truncated, info)"""

    @abstractmethod
    def reset(self, seed: int | None = None, options: dict[str, Any] | None = None):
        """-> (obs, info)"""

    @abstractmethod
    def set_seed(self, seed: int) -> None: ...

    def render(self) -> Any:
        raise NotImplementedError

    def save(self) -> dict:
        return {}

    @abstractmethod
    def close(self) -> None: ...


class EnvRegister:
    """Class-name -> env ids registry (omnisafe/envs/core.py:L300-395)."""

    def __init__(self) -> None:
        self._class: dict[str, type] = {}
        self._support_envs: dict[str, list[str]] = {}

    def register(self, env_class: type) -> type:
        if not inspect.isclass(env_class):
            raise TypeError(f'{env_class} must be a class')
        name = env_class.__name__
        if not issubclass(env_class, CMDP):
            raise TypeError(f'{name} must be subclass of CMDP')
        if name in self._class:
            raise ValueError(f'{name} has been registered')
        ids = list(env_class.support_envs())
        taken = sorted(set(ids) & (set(self.support_envs()) | set(_synthetic_envs())))
        if taken:
            raise ValueError(f'{name}: env ids {taken} are already provided by another class')
        self._class[name] = env_class
        self._support_envs[name] = ids
        return env_class

    def unregister(self, env_class: type) -> type:
        self._class.pop(env_class.__name__, None)
        self._support_envs.pop(env_class.__name__, None)
        return env_class

    def get_class(self, env_id: str, class_name: str | None = None) -> type:
        if class_name is not None:
            assert class_name in self._class, f'{class_name} is not registered'
            assert env_id in self._support_envs[class_name], f'{env_id} is not supported by {class_name}'
            return self._class[class_name]
        for name, ids in self._support_envs.items():
            if env_id in ids:
                return self._class[name]
        raise ValueError(f'{env_id} is not supported by any environment class')

    def support_envs(self) -> list[str]:
        return sorted({i for ids in self._support_envs.values() for i in ids})


ENV_REGISTRY = EnvRegister()
env_register = ENV_REGISTRY.register
env_unregister = ENV_REGISTRY.unregister


def support_envs() -> list[str]:
    """The synthetic env stepped inside the rollout kernel, then every registered id."""
    return _synthetic_envs() + [i for i in ENV_REGISTRY.support_envs() if i not in _synthetic_envs()]


def is_registered(env_id: str) -> bool:
    return env_id in ENV_REGISTRY.support_envs()


def make(env_id: str, num_envs: int = 1, device='cpu', class_name: str | None = None, **env_cfgs: Any):
    """Instantiate a registered env: `cls(env_id, num_envs=num_envs, device=device, **env_cfgs)`."""
    cls = ENV_REGISTRY.get_class(env_id, class_name)
    return cls(env_id, num_envs=num_envs, device=device, **env_cfgs)


def check_env(env) -> tuple[int, int, np.ndarray, np.ndarray]:
    """Refuse what the external-env rollout cannot run; returns (obs_dim, act_dim, act_low, act_high)."""
    name = type(env).__name__
    if getattr(env, 'need_time_limit_wrapper', False) or getattr(env, 'need_auto_reset_wrapper', False):
        raise ValueError(f'{name} declares need_time_limit_wrapper / need_auto_reset_wrapper: the env must truncate and '
                         'auto-reset itself (reporting info["final_observation"]); the wrappers are not provided')
    spaces = {}
    for which, space in (('observation', env.observation_space), ('action', env.action_space)):
        if not all(hasattr(space, k) for k in ('shape', 'low', 'high')):
            raise ValueError(f'{name}: the {which} space must be a Box (shape / low / high), got {type(space).__name__}')
        shape = tuple(space.shape)
        if len(shape) != 1 or shape[0] < 1:
            raise ValueError(f'{name}: the {which} space must be 1-D, got shape {shape}')
        spaces[which] = (shape[0], space)
    O, _ = spaces['observation']
    A, act = spaces['action']
    if A > MAX_ACT_DIM:
        raise ValueError(f'{name}: act_dim {A} > {MAX_ACT_DIM} is not supported by the rollout kernels')
    lo = np.broadcast_to(np.asarray(act.low, np.float32), (A,)).copy()
    hi = np.broadcast_to(np.asarray(act.high, np.float32), (A,)).copy()
    if not (np.isfinite(lo).all() and np.isfinite(hi).all()):
        raise ValueError(f'{name}: the action bounds must be finite (ActionScale maps [-1, 1] onto them), got {lo} .. {hi}')
    if getattr(env, 'graph_safe', False):
        dev = getattr(env, 'device', None) or getattr(env, '_device', None)
        if dev is None or getattr(dev, 'type', str(dev).split(':')[0]) != 'cuda':
            raise ValueError(f'{name} declares graph_safe but its observations are not on a CUDA device (device = {dev}): '
                             'a graph-safe env lives on the training GPU and exposes it as `device`')
    return O, A, lo, hi
