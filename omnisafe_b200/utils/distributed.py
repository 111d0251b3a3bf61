"""Process-group helpers: one process per GPU, torch.distributed for bootstrap, NCCL for the data
path.  Mirrors the surface of omnisafe/utils/distributed.py (fork / world_size / get_rank /
dist_avg / dist_sum / avg_grads semantics); the hot-loop gradient all-reduce is issued from C through
the communicator created here (csrc/epoch.cu).
"""
from __future__ import annotations

import ctypes
import os
import subprocess
import sys

import torch
import torch.distributed as dist

_COMM = None  # ctypes.c_void_p of the NCCL communicator used from C
_P2P = {}     # param count -> (device ptr-array of peer buffers, device ptr-array of peer flags, error flag)


def world_size() -> int:
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def get_rank() -> int:
    return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0


def is_master() -> bool:
    return get_rank() == 0


def nccl_comm():
    return _COMM if _COMM is not None else 0


def nccl_library_path() -> str:
    base = os.path.dirname(torch.__file__)
    cand = os.path.join(base, '..', 'nvidia', 'nccl', 'lib', 'libnccl.so.2')
    return os.path.abspath(cand) if os.path.exists(cand) else 'libnccl.so.2'


def fork(parallel: int, device: str = 'cuda', manual_args: list[str] | None = None) -> bool:
    """Re-exec under torchrun when `parallel > 1` and no process group exists yet
    (omnisafe/utils/distributed.py:L83-139).  Returns True in the parent (which should exit)."""
    if parallel > 1 and os.getenv('RANK') is None:
        args = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1',
                f'--nproc-per-node={parallel}', '--master-addr', '127.0.0.1', '--master-port',
                os.getenv('MASTER_PORT', '29511')]
        args += manual_args if manual_args is not None else sys.argv
        subprocess.check_call(args, env=os.environ)
        return True
    init_process_group(device)
    return False


def init_process_group(device: str = 'cuda') -> None:
    """Join the torchrun-provided group (nccl for CUDA, gloo for CPU host-logic tests)."""
    global _COMM
    if os.getenv('RANK') is None or (dist.is_available() and dist.is_initialized()):
        return
    backend = 'nccl' if str(device).startswith('cuda') else 'gloo'
    if backend == 'nccl':
        torch.cuda.set_device(int(os.getenv('LOCAL_RANK', '0')))
    dist.init_process_group(backend=backend)
    if backend == 'nccl' and dist.get_world_size() > 1:
        _COMM = _create_nccl_comm()


def _create_nccl_comm():
    from omnisafe_b200._lib import lib  # noqa: PLC0415

    path = nccl_library_path().encode()
    uid = (ctypes.c_ubyte * 128)()
    if get_rank() == 0:
        lib().osb_nccl_unique_id(path, uid)
    t = torch.tensor(list(uid), dtype=torch.uint8, device='cuda')
    dist.broadcast(t, 0)
    uid = (ctypes.c_ubyte * 128)(*t.cpu().tolist())
    comm = ctypes.c_void_p()
    lib().osb_nccl_init(path, uid, dist.get_world_size(), dist.get_rank(), ctypes.byref(comm))
    return comm


def p2p_exchange(n_params: int):
    """NVLink peer-memory exchange buffers for the fused reduce+clip+all-reduce+Adam kernel: every
    rank allocates [2][P] floats + [2][world] flags with cudaMalloc, the cudaIpc handles travel
    through torch.distributed, peers map them.  Returns (peer_buf_array_ptr, peer_flag_array_ptr,
    error_flag_ptr) as ints, or (0, 0, 0) for a single rank / when OSB_NO_P2P is set."""
    if world_size() == 1 or os.getenv('OSB_NO_P2P'):
        return 0, 0, 0
    if n_params in _P2P:
        bufs, flags, err = _P2P[n_params]
        return bufs.data_ptr(), flags.data_ptr(), err.data_ptr()
    from omnisafe_b200._lib import lib  # noqa: PLC0415

    w, r = world_size(), get_rank()
    ptrs = []
    # receive buffers [2][world][P] (the persistent bf16x3 kernel pushes slices; the per-step kernel uses the first
    # [2][P]); flags: [2][world] (per-step kernel) + [2][world][160] (one flag per CTA of the persistent kernel)
    # (8 bytes per parameter slot: the persistent kernel sends {step tag, value} words)
    for nbytes in (2 * w * n_params * 8, (2 * w + 2 * w * 160) * 4):
        mine = ctypes.c_void_p()
        handle = (ctypes.c_ubyte * 64)()
        lib().osb_p2p_alloc(nbytes, ctypes.byref(mine), handle)
        t = torch.tensor(list(handle), dtype=torch.uint8, device='cuda')
        gathered = [torch.zeros_like(t) for _ in range(w)]
        dist.all_gather(gathered, t)
        addr = []
        for peer in range(w):
            if peer == r:
                addr.append(mine.value)
            else:
                h = (ctypes.c_ubyte * 64)(*gathered[peer].cpu().tolist())
                p = ctypes.c_void_p()
                lib().osb_p2p_open(h, ctypes.byref(p))
                addr.append(p.value)
        ptrs.append(torch.tensor(addr, dtype=torch.int64, device='cuda'))
    err = torch.zeros(1, dtype=torch.int32, device='cuda')
    dist.barrier()
    _P2P[n_params] = (ptrs[0], ptrs[1], err)
    return ptrs[0].data_ptr(), ptrs[1].data_ptr(), err.data_ptr()


def p2p_check() -> None:
    for bufs, flags, err in _P2P.values():
        assert int(err.item()) == 0, 'NVLink gradient exchange timed out waiting for a peer rank'


def all_reduce_(t: torch.Tensor) -> torch.Tensor:
    """In-place SUM all-reduce (no-op for a single rank)."""
    if world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return t


def avg_grads(module) -> None:
    """Average the gradients of `module.parameters()` over ranks (omnisafe/utils/distributed.py:L167-198): the
    all-reduce SUM and 1/world scale the update kernels apply after clipping."""
    if world_size() > 1:
        for param in module.parameters():
            if param.grad is not None:
                dist.all_reduce(param.grad, op=dist.ReduceOp.SUM)
                param.grad.mul_(1.0 / world_size())


def barrier() -> None:
    if world_size() > 1:
        dist.barrier()


def broadcast_object(obj):
    """Rank 0's `obj` on every rank (a picklable host object)."""
    if world_size() == 1:
        return obj
    box = [obj]
    dist.broadcast_object_list(box, src=0)
    return box[0]


def dist_avg(value: torch.Tensor | float) -> torch.Tensor:
    """Average over ranks (omnisafe/utils/distributed.py:L231-260)."""
    t = torch.as_tensor(value, dtype=torch.float32).clone()
    if world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
        t /= world_size()
    return t


def local_steps(steps_per_epoch: int, vector_env_nums: int) -> int:
    """steps_per_epoch is GLOBAL: per-rank steps per env = steps_per_epoch // world // num_envs
    (algorithms/on_policy/base/policy_gradient.py:L70-77)."""
    assert steps_per_epoch % (world_size() * vector_env_nums) == 0, (
        'The number of steps per epoch is not divisible by the number of environments.')
    return steps_per_epoch // world_size() // vector_env_nums
