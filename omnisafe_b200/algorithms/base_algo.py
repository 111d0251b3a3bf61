"""BaseAlgo: fixed construction order `_init_env -> _init_model -> _init -> _init_log`
(mirrors omnisafe/algorithms/base_algo.py:L28-83)."""
from __future__ import annotations

from abc import ABC, abstractmethod

import torch

from omnisafe_b200.utils import distributed
from omnisafe_b200.utils.config import Config


class BaseAlgo(ABC):
    _run_dir: str | None = None     # the directory of a run being resumed (`continuing`): the logger continues it

    @classmethod
    def continuing(cls, run_dir: str, env_id: str, cfgs: Config) -> BaseAlgo:
        """Construct the algorithm of an existing run directory (for `load_train_state`), keeping the upstream
        constructor signature `(env_id, cfgs)`."""
        obj = cls.__new__(cls)
        obj._run_dir = run_dir
        obj.__init__(env_id, cfgs)
        return obj

    def __init__(self, env_id: str, cfgs: Config) -> None:
        self._env_id = env_id
        self._cfgs = cfgs
        assert hasattr(cfgs, 'seed'), 'Please specify the seed in the config file.'
        self._seed = int(cfgs.seed) + distributed.get_rank() * 1000
        torch.manual_seed(self._seed)
        dev = str(cfgs.train_cfgs.device)
        if not dev.startswith('cuda'):
            raise RuntimeError(
                f"train_cfgs.device={dev!r}: omnisafe_b200 runs this path as sm_90a CUDA kernels only "
                "(no CPU fallback); use the upstream omnisafe classes for CPU training")
        if not torch.cuda.is_available():
            raise RuntimeError('omnisafe_b200 needs a CUDA device (no CPU fallback)')
        self._device = torch.device('cuda', torch.cuda.current_device())
        self._init_env()
        self._init_model()
        self._init()
        self._init_log()

    @property
    def logger(self):
        return self._logger

    @property
    def cost_limit(self):
        return getattr(self._cfgs.algo_cfgs, '_cost_limit', None)

    @abstractmethod
    def _init_env(self) -> None: ...

    @abstractmethod
    def _init_model(self) -> None: ...

    @abstractmethod
    def _init(self) -> None: ...

    @abstractmethod
    def _init_log(self) -> None: ...

    @abstractmethod
    def learn(self) -> tuple[float, float, float]: ...
