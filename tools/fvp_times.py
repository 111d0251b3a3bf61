"""CUDA-event timing of the Fisher-vector product and full-batch actor gradient, fp32 FMA tiles vs tf32 and
bf16x3 wgmma tiles (headline batch 4096 x 128, O = 60, A = 8)."""
import json
import sys

import torch

sys.path.insert(0, '.')
import omnisafe_b200
from omnisafe_b200.algorithms.engine import LOSS_RATIO

N, T = 4096, 128
agent = omnisafe_b200.Agent('CPO', 'SyntheticBox-v0', custom_cfgs={
    'seed': 0, 'train_cfgs': {'device': 'cuda', 'vector_env_nums': N, 'total_steps': N * T * 4},
    'algo_cfgs': {'steps_per_epoch': N * T, 'batch_size': 16384, 'update_iters': 8},
    'logger_cfgs': {'use_tensorboard': False, 'log_dir': '/tmp/osb_fvp', 'save_model_freq': 10 ** 9},
    'env_cfgs': {'obs_dim': 60, 'act_dim': 8, 'max_episode_steps': 64}})
algo = agent.agent
algo.train_epoch()
eng = algo._engine
vec = torch.randn(eng.Pa, device='cuda')
out = torch.zeros(eng.Pa, device='cuda')
g = torch.zeros(eng.Pa, device='cuda')


def timeit(fn, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e3


res = {}
for prec, name in ((0, 'fp32'), (1, 'tf32'), (2, 'bf16x3')):
    eng.precision = prec
    res[f'fvp_{name}_us'] = round(timeit(lambda: eng.fvp(vec, out, 0.1)), 1)
    res[f'actor_loss_grad_{name}_us'] = round(timeit(lambda: eng.actor_loss_grad(LOSS_RATIO, None, g)), 1)
flops = 6 * 2 * (60 * 64 + 64 * 64 + 64 * 8) * N * T          # tangent fwd + fwd + bwd, 2 flop per MAC
for name in ('tf32', 'bf16x3'):
    res[f'fvp_{name}_TFLOPs'] = round(flops / (res[f'fvp_{name}_us'] * 1e-6) / 1e12, 1)
print(json.dumps(res))
