"""`omnisafe_b200.Agent` -- the `omnisafe.Agent(algo, env_id, train_terminal_cfgs, custom_cfgs)`
entry point (mirrors omnisafe/algorithms/algo_wrapper.py:L36-269: config merge, checks,
`distributed.fork`, `registry.get(algo)(env_id, cfgs)`, `learn()`, `evaluate()`), plus saving the training state and resuming a
stopped run from it (`save_state`, `learn(save_state_freq=...)`, `resume`; upstream has no resume)."""
from __future__ import annotations

import json
import os
import sys

from omnisafe_b200.algorithms import ALGORITHM2TYPE, registry
from omnisafe_b200.envs import support_envs
from omnisafe_b200.evaluator import Evaluator
from omnisafe_b200.utils import distributed, train_state
from omnisafe_b200.utils.config import (Config, check_all_configs, get_default_kwargs_yaml,
                                        recursive_check_config)


class AlgoWrapper:
    def __init__(self, algo: str, env_id: str, train_terminal_cfgs: dict | None = None,
                 custom_cfgs: dict | None = None) -> None:
        self.algo, self.env_id = algo, env_id
        self.train_terminal_cfgs, self.custom_cfgs = train_terminal_cfgs, custom_cfgs
        self._evaluator = None
        self.cfgs = self._init_config()
        self._init_checks()
        self._init_algo()

    def _init_config(self) -> Config:
        assert self.algo in ALGORITHM2TYPE, f'{self.algo} doesn\'t exist. Please choose from {list(ALGORITHM2TYPE)}.'
        self.algo_type = ALGORITHM2TYPE[self.algo]
        cfgs = get_default_kwargs_yaml(self.algo, self.env_id, self.algo_type)
        cfgs.recurisve_update({'exp_name': f'{self.algo}-{{{self.env_id}}}', 'env_id': self.env_id, 'algo': self.algo})
        if self.custom_cfgs:
            recursive_check_config(self.custom_cfgs, cfgs, exclude_keys=('algo', 'env_id'))
            cfgs.recurisve_update(self.custom_cfgs)
        if self.train_terminal_cfgs:
            recursive_check_config(self.train_terminal_cfgs, cfgs.train_cfgs)
            cfgs.train_cfgs.recurisve_update(self.train_terminal_cfgs)
        epochs = cfgs.train_cfgs.total_steps // cfgs.algo_cfgs.steps_per_epoch
        cfgs.train_cfgs.recurisve_update({'epochs': epochs})
        return cfgs

    def _init_checks(self) -> None:
        assert isinstance(self.algo, str), 'algo must be a string!'
        assert isinstance(self.cfgs.train_cfgs.parallel, int), 'parallel must be an integer!'
        assert self.cfgs.train_cfgs.parallel > 0, 'parallel must be greater than 0!'
        assert self.env_id in support_envs(), (
            f"{self.env_id} doesn't exist. omnisafe_b200 accelerates {support_envs()}; "
            'use upstream omnisafe for simulator-backed environments.')

    def _init_algo(self, run_dir: str | None = None) -> None:
        check_all_configs(self.cfgs)
        if distributed.fork(self.cfgs.train_cfgs.parallel, device=self.cfgs.train_cfgs.device):
            sys.exit()
        if run_dir is None:
            self.agent = registry.get(self.algo)(env_id=self.env_id, cfgs=self.cfgs)
        else:
            self.agent = registry.get(self.algo).continuing(run_dir, env_id=self.env_id, cfgs=self.cfgs)

    @classmethod
    def resume(cls, state_dir: str) -> AlgoWrapper:
        """Continue a run from a training state `save_state` / `learn(save_state_freq=...)` wrote.

        The run is rebuilt from its config.json (the configuration cannot change on resume) through the same checks and
        `distributed.fork` as a new run -- so a script calling `Agent.resume(d).learn()` under `parallel: 2` works --
        then every rank loads its state in place.  `learn()` trains the remaining epochs into the original run directory:
        progress.csv is appended to, torch_save/epoch-k.pt keeps its numbering, config.json stays as it is."""
        state_dir = os.path.abspath(state_dir)
        meta = train_state.read_meta(state_dir)
        run_dir = train_state.run_dir(state_dir)
        path = os.path.join(run_dir, 'config.json')
        if not os.path.exists(path):
            raise RuntimeError(f'{path} is missing: {state_dir} is not inside a run directory')
        with open(path, encoding='utf-8') as fh:
            cfgs = Config.dict2config(json.load(fh))
        self = cls.__new__(cls)
        self.algo, self.env_id = cfgs.algo, cfgs.env_id
        self.train_terminal_cfgs = self.custom_cfgs = None
        self._evaluator = None
        assert self.algo in ALGORITHM2TYPE, f'{self.algo} doesn\'t exist. Please choose from {list(ALGORITHM2TYPE)}.'
        self.algo_type = ALGORITHM2TYPE[self.algo]
        self.cfgs = cfgs
        self._init_checks()
        train_state.check_meta(meta, train_state.config_meta(cfgs, int(cfgs.train_cfgs.parallel)), state_dir)
        self._init_algo(run_dir=run_dir)
        self.agent.load_train_state(state_dir)
        return self

    def learn(self, save_state_freq: int = 0) -> tuple[float, float, float]:
        """Train (the remaining epochs, after `resume`).  `save_state_freq` > 0: also write the training state after every
        `save_state_freq`-th epoch and after the last one, to <log_dir>/train_state/epoch-{k}/."""
        return self.agent.learn(save_state_freq=save_state_freq)

    def save_state(self) -> str:
        """Write the training state now (between epochs; every rank calls it) and return its directory."""
        return self.agent.save_train_state()

    def evaluate(self, num_episodes: int = 10, cost_criteria: float = 1.0, num_envs: int = 1) -> None:
        """Evaluate every torch_save/*.pt of this run with `Evaluator` (algo_wrapper.py:L215-231), in sorted file order
        (upstream takes the directory's scandir order).  `num_envs`: see `Evaluator.evaluate`."""
        log_dir = self.agent.logger.log_dir
        save_dir = os.path.join(log_dir, 'torch_save')
        assert os.path.isdir(save_dir), 'Please run learn() first!'
        if self._evaluator is None:
            self._evaluator = Evaluator()
        for name in sorted(os.listdir(save_dir)):
            if os.path.isfile(os.path.join(save_dir, name)) and name.split('.')[-1] == 'pt':
                self._evaluator.load_saved(save_dir=log_dir, model_name=name)
                self._evaluator.evaluate(num_episodes=num_episodes, cost_criteria=cost_criteria, num_envs=num_envs)

    def render(self, *_, **__):
        raise NotImplementedError('rendering is not supported')
