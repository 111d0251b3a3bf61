"""CUDA-event timing of the update-side kernels at a given obs dim (default 376), fp32 FMA tiles vs wgmma
tiles: minibatch gradient (16384 rows, 3 networks), Fisher-vector product, full-batch evaluation."""
import json
import sys

import torch

sys.path.insert(0, '.')
import omnisafe_b200
from omnisafe_b200._lib import current_stream as s, lib, ptr
from omnisafe_b200.algorithms.engine import LOSS_RATIO

O = int(sys.argv[1]) if len(sys.argv) > 1 else 376
N, T, A = 4096, 128, 8
agent = omnisafe_b200.Agent('CPO', 'SyntheticBox-v0', custom_cfgs={
    'seed': 0, 'train_cfgs': {'device': 'cuda', 'vector_env_nums': N, 'total_steps': N * T * 4},
    'algo_cfgs': {'steps_per_epoch': N * T, 'batch_size': 16384, 'update_iters': 8},
    'logger_cfgs': {'use_tensorboard': False, 'log_dir': '/tmp/osb_chunk', 'save_model_freq': 10 ** 9},
    'env_cfgs': {'obs_dim': O, 'act_dim': A, 'max_episode_steps': 64}})
algo = agent.agent
algo._env.rollout(T, algo._actor_critic, algo._buf, algo._logger)
algo._buf.finish_paths(); algo._reduce_epoch_statistics()
eng, buf, ac = algo._engine, algo._buf, algo._actor_critic
d = buf.data
total, bs = N * T, 16384
vec = torch.randn(eng.Pa, device='cuda')
out = torch.zeros(eng.Pa, device='cuda')
eng.snapshot_old_policy()


def timeit(fn, iters=10):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return round(a.elapsed_time(b) / iters * 1e3, 1)


def grad(fn):
    return lambda: fn(ptr(ac.theta), O, A, ptr(d['obs']), ptr(d['act']), ptr(d['logp']), ptr(d['adv_r']), ptr(d['adv_c']),
                      ptr(d['target_value_r']), ptr(d['target_value_c']), ptr(eng.mu_old), ptr(buf.adv_moments), 0, total, 1,
                      0, bs, 0, 0.2, 0.0, 1.0, 0.0, 0, ptr(eng.logstd_old), 7, ptr(eng.gpart), ptr(eng.stats_part), 0, s())


res = {'obs_dim': O}
res['grad_fp32_us'] = timeit(grad(lib().osb_minibatch_grad))
res['grad_tc_us'] = timeit(grad(lib().osb_minibatch_grad_tc))
for prec, name in ((0, 'fp32'), (1, 'tc')):
    eng.precision = prec
    res[f'fvp_{name}_us'] = timeit(lambda: eng.fvp(vec, out, 0.1), 5)
    res[f'eval_{name}_us'] = timeit(lambda: eng.evaluate(ac.theta, None), 5)
a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
a.record()
algo._env.rollout(T, algo._actor_critic, algo._buf, algo._logger)
b.record(); torch.cuda.synchronize()
res['rollout_epoch_ms'] = round(a.elapsed_time(b), 2)
print(json.dumps(res))
