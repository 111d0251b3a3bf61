"""CUDA-event timing of the dual-GAE launch (training configuration: no discounted_ret slab) at several horizons."""
import json, sys
import torch
sys.path.insert(0, '.')
from omnisafe_b200.common.buffer import VectorOnPolicyBuffer

out = {'kernel': 'gae_stream_kernel<TMA>'}
for T, N in ((128, 4096), (512, 4096), (2048, 4096), (4096, 4096), (128, 32768)):
    buf = VectorOnPolicyBuffer(4, 2, T, 0.99, 0.95, 0.95, 'gae', 0.0, True, True, num_envs=N, device='cuda', keep_discounted_ret=False)
    for k in ('reward', 'cost', 'value_r', 'value_c', 'boot_r', 'boot_c'):
        buf.data[k].normal_()
    buf.data['flags'].copy_((torch.rand(T, N, device='cuda') < 0.02).to(torch.uint8) * 2)
    for _ in range(5):
        buf.finish_paths()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(50):
        buf.finish_paths()
    b.record(); torch.cuda.synchronize()
    us = a.elapsed_time(b) / 50 * 1e3
    out[f'T{T}_N{N}'] = {'us': round(us, 2), 'GBps': round(33 * T * N / us / 1e3, 1)}
print(json.dumps(out))
