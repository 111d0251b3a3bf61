"""CUDA-event times of the bf16x3 full-batch actor evaluation at the bench workload, against the update it sits in.

Times osb_actor_eval_x3 in mu_store mode (the old-policy snapshot) and in KL mode (the per-iteration full-batch KL
check, with its fp64 reduction), osb_kl_check, one persistent update iteration (osb_ppo_update_iter_x3 with zero
learning rates, as bench.py times it) and one algo._update(), and sets each evaluation pass against its two bounds:
the bf16 tensor-core time of the 6 bf16 products per padded fp32 product, and the HBM time of the bytes it must move.
Prints the card name and power limit of the measurement, then one JSON line."""
import json
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import bench
import omnisafe_b200
from omnisafe_b200._lib import current_stream, lib, ptr

PEAK_BF16_TFLOPS, PEAK_HBM_GBS = 989.0, 3350.0    # H100 SXM data sheet (700 W), dense bf16 / HBM3

assert torch.cuda.is_available(), 'actor_eval_times needs a CUDA device'
card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                      capture_output=True, text=True).stdout.strip().splitlines()[0]
w = bench.WORKLOAD
agent = omnisafe_b200.Agent(w['algo'], w['env'], custom_cfgs=bench._custom_cfgs(1, tempfile.mkdtemp(), 50, None, 'bf16x3'))
algo = agent.agent
for _ in range(2):
    algo.train_epoch()
torch.cuda.synchronize()
eng, buf, ac, d = algo._engine, algo._buf, algo._actor_critic, algo._buf.data
assert eng.precision == 2
O, A, total, bs = w['obs_dim'], w['act_dim'], buf.T * buf.N, w['batch_size']
lag = algo._lagrange.state
s = current_stream


def timeit(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3


mu_scratch = torch.empty_like(eng.mu_old)


def eval_mu():
    rc = lib().osb_actor_eval_x3(ptr(ac.theta), O, A, ptr(d['obs']), 0, 0, 0, 0, 0, 0, 0, 0, total, 1, ptr(mu_scratch),
                                 0, 0, s())
    assert rc == 0


def eval_kl():
    rc = lib().osb_actor_eval_x3(ptr(ac.theta), O, A, ptr(d['obs']), ptr(d['act']), ptr(d['logp']), ptr(d['adv_r']),
                                 ptr(d['adv_c']), ptr(eng.mu_old), ptr(eng.logstd_old), ptr(buf.adv_moments), ptr(lag),
                                 total, 1, 0, ptr(eng.eval_ws), ptr(eng.eval_out), s())
    assert rc == 0


kl_state = torch.zeros_like(eng.kl_state)
stop_flag = torch.zeros_like(eng.stop_flag)


def kl_check():
    lib().osb_kl_check(ptr(eng.eval_out), 0.02, 0, ptr(stop_flag), ptr(kl_state), s())


def iter_x3():
    lib().osb_ppo_update_iter_x3(ptr(ac.theta), ptr(ac.grad), ptr(ac.adam_m), ptr(ac.adam_v), ptr(ac.adam_step), O, A,
                                 ptr(d['obs']), ptr(d['act']), ptr(d['logp']), ptr(d['adv_r']), ptr(d['adv_c']),
                                 ptr(d['target_value_r']), ptr(d['target_value_c']), ptr(buf.adv_moments), 0, total, 12345,
                                 bs, 0, 0.2, 0.0, ptr(lag), 7, 0.001, 40.0, 0.0, 0.0, 0.0, ptr(eng.gpart),
                                 ptr(eng.stats_part), ptr(eng.train_stats), 0, 0, 0, 1, 0, 0, s())


res = {'card': card, 'O': O, 'A': A, 'rows': total}
res['eval_mu_store_us'] = timeit(eval_mu, 50)
res['eval_kl_us'] = timeit(eval_kl, 50)
res['kl_check_us'] = timeit(kl_check, 200)
res['update_iter_x3_us'] = timeit(iter_x3, 10)
res['update_ms'] = timeit(algo._update, 5) * 1e-3
res['us_per_minibatch_step'] = res['update_iter_x3_us'] / (total // bs)
res['nine_passes_ms'] = (res['eval_mu_store_us'] + 8 * (res['eval_kl_us'] + res['kl_check_us'])) * 1e-3
# every row runs the padded forward: K 64 -> 64 -> 64 -> 16 columns, 6 bf16 products per fp32-level product
flop = 6 * 2 * (64 * 64 + 64 * 64 + 64 * 16) * total
bytes_mu = (O + A) * 4 * total                        # obs in, mu out
bytes_kl = (O + 2 * A + 3) * 4 * total                # obs, act, mu_old, logp, adv_r, adv_c in
t_flop = flop / (PEAK_BF16_TFLOPS * 1e12) * 1e6
for mode, nbytes in (('mu_store', bytes_mu), ('kl', bytes_kl)):
    us = res[f'eval_{mode}_us']
    t_hbm = nbytes / (PEAK_HBM_GBS * 1e9) * 1e6
    res[f'eval_{mode}'] = {'bf16_tflops': flop / (us * 1e-6) / 1e12, 'gbs': nbytes / (us * 1e-6) / 1e9,
                           'compute_bound_us': t_flop, 'hbm_bound_us': t_hbm,
                           'share_of_compute_bound': t_flop / us, 'share_of_hbm_bound': t_hbm / us}
print(f'card: {card}')
for k in ('eval_mu_store_us', 'eval_kl_us', 'kl_check_us', 'update_iter_x3_us', 'us_per_minibatch_step'):
    print(f'{k:24s} {res[k]:10.1f}')
print(f'{"update_ms":24s} {res["update_ms"]:10.3f}')
print(f'{"nine_passes_ms":24s} {res["nine_passes_ms"]:10.3f}')
print(json.dumps(res))
