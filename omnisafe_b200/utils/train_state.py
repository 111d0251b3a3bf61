"""On-disk layout of a saved training state (`AlgoWrapper.save_state`, `Agent.resume`).

    <log_dir>/train_state/epoch-{k}/rank-{r}.pt    one per rank: {'format_version', 'epoch', 'rank', 'state'}
    <log_dir>/train_state/epoch-{k}/meta.json      written by rank 0 after every rank file is in place

`state` is the nested dict the algorithm composes from the `train_state()` methods of the objects it owns; this module
only writes, finds and validates the files.  Every file goes to a temporary name first and is moved into place with
`os.replace`, so a reader sees a whole file or none.  A directory without `meta.json`, or with a rank file missing, is
an interrupted save and is refused.  The directory is not under `torch_save/`: the upstream `Evaluator` loads every
`*.pt` file there.
"""
from __future__ import annotations

import json
import os

import torch

FORMAT_VERSION = 1
# what a resumed run must agree on with the state it loads (meta.json keys besides format_version / epoch)
MATCH_KEYS = ('algo', 'env_id', 'obs_dim', 'act_dim', 'num_envs', 'steps', 'world_size', 'precision')


def config_meta(cfgs, world_size: int) -> dict:
    """The meta.json entries a run's configuration fixes (obs_dim / act_dim come from the env)."""
    t, a = cfgs.train_cfgs, cfgs.algo_cfgs
    n = int(t.vector_env_nums)
    return {'algo': cfgs.algo, 'env_id': cfgs.env_id, 'num_envs': n, 'steps': int(a.steps_per_epoch) // world_size // n,
            'world_size': int(world_size), 'precision': str(getattr(t, 'matmul_precision', 'bf16x3'))}


def state_dir(log_dir: str, epoch: int) -> str:
    return os.path.join(log_dir, 'train_state', f'epoch-{int(epoch)}')


def run_dir(sdir: str) -> str:
    """The run directory (`log_dir`) a state directory belongs to."""
    return os.path.dirname(os.path.dirname(os.path.abspath(sdir)))


def rank_path(sdir: str, rank: int) -> str:
    return os.path.join(sdir, f'rank-{int(rank)}.pt')


def _atomic(path: str, write) -> None:
    tmp = f'{path}.tmp-{os.getpid()}'
    try:
        write(tmp)
        os.replace(tmp, path)
    finally:
        if os.path.exists(tmp):
            os.remove(tmp)


def begin(sdir: str) -> None:
    """Rank 0, before any rank writes: mark the directory incomplete (a save over an earlier one at the same epoch)."""
    os.makedirs(sdir, exist_ok=True)
    meta = os.path.join(sdir, 'meta.json')
    if os.path.exists(meta):
        os.remove(meta)


def write_rank(sdir: str, rank: int, epoch: int, state: dict) -> None:
    os.makedirs(sdir, exist_ok=True)
    blob = {'format_version': FORMAT_VERSION, 'epoch': int(epoch), 'rank': int(rank), 'state': state}
    _atomic(rank_path(sdir, rank), lambda p: torch.save(blob, p))


def write_meta(sdir: str, meta: dict) -> None:
    meta = {'format_version': FORMAT_VERSION, **meta}

    def write(p):
        with open(p, 'w', encoding='utf-8') as fh:
            json.dump(meta, fh, indent=4)

    _atomic(os.path.join(sdir, 'meta.json'), write)


def read_meta(sdir: str) -> dict:
    """meta.json of a complete save; refuses an interrupted one (no meta.json, a rank file missing)."""
    path = os.path.join(sdir, 'meta.json')
    if not os.path.isdir(sdir):
        raise FileNotFoundError(f'{sdir}: no such training-state directory')
    if not os.path.exists(path):
        raise RuntimeError(f'{sdir} has no meta.json: the save was interrupted, resume from an earlier epoch')
    try:
        with open(path, encoding='utf-8') as fh:
            meta = json.load(fh)
    except (OSError, ValueError) as exc:
        raise RuntimeError(f'{path} is unreadable: {exc}') from exc
    if not isinstance(meta, dict) or meta.get('format_version') != FORMAT_VERSION:
        got = meta.get('format_version') if isinstance(meta, dict) else None
        raise RuntimeError(f'{path}: training-state format version {got}, this library reads version {FORMAT_VERSION}')
    missing = [k for k in (*MATCH_KEYS, 'epoch') if k not in meta]
    if missing:
        raise RuntimeError(f'{path} lacks {missing}')
    absent = [r for r in range(int(meta['world_size'])) if not os.path.exists(rank_path(sdir, r))]
    if absent:
        raise RuntimeError(f'{sdir}: rank file(s) {absent} missing of a {meta["world_size"]}-rank save: '
                           'the save was interrupted or the directory is incomplete')
    return meta


def check_meta(meta: dict, expected: dict, sdir: str = '') -> None:
    """Refuse a state whose run differs from the one being rebuilt in any of `expected`'s keys."""
    bad = [f'{k}: saved {meta.get(k)!r}, this run {v!r}' for k, v in expected.items() if meta.get(k) != v]
    if bad:
        raise RuntimeError(f'training state {sdir} does not belong to this run ({"; ".join(bad)}); '
                           'a run resumes with the configuration it was saved with')


def snapshot(*tensors: torch.Tensor) -> list[torch.Tensor]:
    """Host copies of device tensors, for a `train_state()` dict."""
    return [t.detach().cpu().clone() for t in tensors]


def restore(dst: torch.Tensor, src, what: str) -> None:
    """Copy a saved tensor into the tensor the constructor allocated, in place: its address stays the one the CUDA
    graphs and the NVLink exchange were set up with.  Shape and dtype must match exactly (copy_ would broadcast)."""
    src = torch.as_tensor(src)
    if src.shape != dst.shape or src.dtype != dst.dtype:
        raise RuntimeError(f'training state: {what} is {tuple(src.shape)} {src.dtype}, this run has '
                           f'{tuple(dst.shape)} {dst.dtype}')
    dst.copy_(src)


def load_rank(sdir: str, rank: int, epoch: int) -> dict:
    """This rank's state dict (CPU tensors), checked to be the file of this rank and epoch."""
    path = rank_path(sdir, rank)
    if not os.path.exists(path):
        raise RuntimeError(f'{path} is missing: the save was interrupted or the directory is incomplete')
    try:
        blob = torch.load(path, map_location='cpu', weights_only=False)
    except Exception as exc:    # noqa: BLE001  (torch.load raises many kinds on a damaged file)
        raise RuntimeError(f'{path} is unreadable: {type(exc).__name__}: {exc}') from exc
    if not isinstance(blob, dict) or 'state' not in blob:
        raise RuntimeError(f'{path} is not a training-state file')
    want = {'format_version': FORMAT_VERSION, 'rank': int(rank), 'epoch': int(epoch)}
    bad = {k: blob.get(k) for k, v in want.items() if blob.get(k) != v}
    if bad:
        raise RuntimeError(f'{path}: {bad} where {want} was expected')
    return blob['state']
