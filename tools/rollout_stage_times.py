"""Where one step of the persistent rollout kernel goes: clock64 stamps of thread 0 of actor CTA (0,0) and critic CTA (0,1)."""
import os, sys, tempfile
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import omnisafe_b200, bench
from omnisafe_b200._lib import lib, ptr
cfg = bench._custom_cfgs(1, tempfile.mkdtemp(), 40)
cfg['train_cfgs']['matmul_precision'] = os.environ.get('PREC', 'bf16x3')
algo = omnisafe_b200.Agent('PPOLag', 'SyntheticBox-v0', custom_cfgs=cfg).agent
for _ in range(2): algo.train_epoch()
dbg = torch.zeros(1024, dtype=torch.int64, device='cuda')
torch.cuda.synchronize()
lib().osb_rollout_debug_buffer(ptr(dbg))
algo._env.rollout(algo._steps_per_epoch, algo._actor_critic, algo._buf, algo._logger)
torch.cuda.synchronize()
lib().osb_rollout_debug_buffer(0)
NAMES = {1: 'step start', 2: 'obs tile staged', 3: 'layer 1 MMAs done', 4: 'E1 + layer 2 MMAs done', 5: 'E2 + layer 3 MMAs done', 6: 'outputs written',
         7: 'sampled + log-prob', 8: 'env transition', 9: 'normaliser sums', 10: 'grid barrier', 11: 'normaliser fold'}
for which, off in (('actor CTA', 0), ('reward-critic CTA', 512)):
    d = dbg[off:off + 512].cpu().tolist()
    n = d[0]
    print(f'== {which}: {n} stamps')
    prev = t0 = d[2]
    for i in range(min(n, 48)):
        id_, clk = d[1 + 2 * i], d[2 + 2 * i]
        print(f'  {NAMES.get(id_, id_):28s} +{clk - prev:7d} cyc   t={clk - t0:8d}')
        prev = clk
