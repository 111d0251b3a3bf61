"""Minimal Logger with the reference's on-disk artefacts.

Mirrors omnisafe/common/logger.py: `<log_dir>/<exp_name>/seed-xxx-<time>/{config.json,
progress.csv, torch_save/epoch-k.pt}` (L105-194), `register_key / store / get_stats /
dump_tabular` (L196-374).  Values arrive as python floats or device scalars that were produced by
the kernels; windowed episode metrics are NOT re-buffered here -- they live in the device ring
(`osb_episode_window`) and are stored as ready-made means.  TensorBoard / W&B sinks are out of
scope (SURVEY §2.1 row 8).
"""
from __future__ import annotations

import csv
import os
import time

import torch

from omnisafe_b200.utils import distributed


class Logger:
    def __init__(self, output_dir: str, exp_name: str, seed: int = 0, config=None, verbose: bool = False,
                 run_dir: str | None = None) -> None:
        """`run_dir`: continue an existing run's directory (a resumed run): config.json stays as it is and
        progress.csv is opened by `load_train_state`."""
        hms = time.strftime('%Y-%m-%d-%H-%M-%S')
        self._log_dir = run_dir or os.path.join(output_dir, exp_name, f'seed-{str(seed).zfill(3)}-{hms}')
        self._master = distributed.is_master()
        self._verbose = verbose
        self._epoch = 0
        self._keys: list[str] = []
        self._row: dict[str, float] = {}
        self._first = True
        self._what_to_save = None
        self._csv = None
        self._file = None
        if self._master and run_dir is None:
            os.makedirs(os.path.join(self._log_dir, 'torch_save'), exist_ok=True)
            self._file = open(os.path.join(self._log_dir, 'progress.csv'), 'w', encoding='utf-8', newline='')
            if config is not None:
                with open(os.path.join(self._log_dir, 'config.json'), 'w', encoding='utf-8') as fh:
                    fh.write(config.tojson())

    @property
    def log_dir(self) -> str:
        return self._log_dir

    @property
    def current_epoch(self) -> int:
        return self._epoch

    def log(self, msg: str) -> None:
        if self._master and self._verbose:
            print(msg, flush=True)

    def register_key(self, key: str, **_ignored) -> None:
        assert key not in self._keys, f'Key {key} has been registered'
        self._keys.append(key)
        self._row[key] = float('nan')

    def store(self, data: dict) -> None:
        for key, val in data.items():
            assert key in self._row, f'Key {key} has not been registered'
            self._row[key] = float(val)

    def get_stats(self, key: str) -> tuple[float]:
        return (self._row[key],)

    def setup_torch_saver(self, what_to_save: dict) -> None:
        self._what_to_save = what_to_save

    def torch_save(self) -> None:
        """{'pi': actor.state_dict(), 'obs_normalizer': Normalizer.state_dict()} (logger.py:L183-194)."""
        if not self._master:
            return
        assert self._what_to_save is not None, 'Please setup torch saver first'
        params = {k: (v.state_dict() if hasattr(v, 'state_dict') else v() if callable(v) else v)
                  for k, v in self._what_to_save.items()}
        torch.save(params, os.path.join(self._log_dir, 'torch_save', f'epoch-{self._epoch}.pt'))

    def dump_tabular(self) -> None:
        if self._master:
            if self._first:
                self._csv = csv.writer(self._file)
                self._csv.writerow(self._keys)
                self._first = False
            self._csv.writerow([self._row[k] for k in self._keys])
            self._file.flush()
            if self._verbose:
                print(' | '.join(f'{k}={self._row[k]:.4g}' for k in self._keys if 'Metrics' in k or 'FPS' in k), flush=True)
        self._epoch += 1

    def train_state(self) -> dict:
        return {'epoch': self._epoch}

    def load_train_state(self, state: dict) -> None:
        """Continue at epoch `state['epoch']`: progress.csv keeps its header and the rows of the epochs before it -- rows
        a stopped run wrote after its last saved state belong to epochs that run again -- and is appended to."""
        self._epoch = int(state['epoch'])
        if not self._master:
            return
        path = os.path.join(self._log_dir, 'progress.csv')
        lines = []
        if os.path.exists(path):
            with open(path, encoding='utf-8', newline='') as fh:
                lines = fh.read().splitlines(keepends=True)
        if self._epoch > 0:
            if len(lines) < 1 + self._epoch:
                raise RuntimeError(f'{path} has {max(len(lines) - 1, 0)} epoch rows, the training state is at epoch '
                                   f'{self._epoch}')
            header = next(csv.reader(lines[:1]))
            if header != self._keys:
                raise RuntimeError(f'{path}: the header differs from the keys this run logs')
        lines = lines[:1 + self._epoch] if self._epoch > 0 else []
        tmp = f'{path}.tmp-{os.getpid()}'
        with open(tmp, 'w', encoding='utf-8', newline='') as fh:
            fh.writelines(lines)
        os.replace(tmp, path)
        self._file = open(path, 'a', encoding='utf-8', newline='')
        if lines:
            self._csv = csv.writer(self._file)
            self._first = False

    def close(self) -> None:
        if self._master and self._file:
            self._file.close()
