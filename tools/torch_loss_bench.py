"""Cost of objectives written in PyTorch: device time of one PPOLag update (the bench.py workload: obs 60 / act 8,
4096 envs x T = 128, batch 16384, update_iters 8) on the fused kernels and on the PyTorch path, plus whole epochs.
--hook actor: a subclass whose `_loss_pi` returns super()'s; --hook critic: whose `_update_reward_critic` and
`_update_cost_critic` call super()'s (the actor stays on its kernel step); --hook both.  Alternates the two, prints the
GPU and its power limit.

    python tools/torch_loss_bench.py [--precision bf16x3] [--hook actor|critic|both] [--reps 5] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402
import omnisafe_b200  # noqa: E402
from omnisafe_b200.algorithms import registry  # noqa: E402


def timed(fn, k):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(k):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--precision', default='bf16x3')
    ap.add_argument('--hook', default='actor', choices=('actor', 'critic', 'both'))
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'this measurement needs a GPU'
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    base = registry.get('PPOLag')
    body = {}
    if args.hook in ('actor', 'both'):
        body['_loss_pi'] = lambda self, o, a, lp, adv: base._loss_pi(self, o, a, lp, adv)
    if args.hook in ('critic', 'both'):
        body['_update_reward_critic'] = lambda self, o, t: base._update_reward_critic(self, o, t)
        body['_update_cost_critic'] = lambda self, o, t: base._update_cost_critic(self, o, t)
    user = type('UserPPOLag', (base,), body)
    algos = {}
    for tag, cls in (('fused', base), ('torch', user)):
        registry._classes['PPOLag'] = cls
        cfg = bench._custom_cfgs(1, tempfile.mkdtemp(), 200)
        cfg['train_cfgs']['matmul_precision'] = args.precision
        algos[tag] = omnisafe_b200.Agent('PPOLag', 'SyntheticBox-v0', custom_cfgs=cfg).agent
    registry._classes['PPOLag'] = base
    assert not algos['fused']._torch_hooks and algos['torch']._torch_hooks
    for a in algos.values():
        for _ in range(2):
            a.train_epoch()
    res = {tag: {'update_ms': [], 'epoch_ms': []} for tag in algos}
    for _ in range(args.reps):              # alternate the two paths
        for tag, a in algos.items():
            res[tag]['update_ms'].append(timed(a._update, 1))
            res[tag]['epoch_ms'].append(timed(a.train_epoch, 1))
    out = {'gpu': gpu, 'precision': args.precision, 'hook': args.hook, 'workload': 'PPOLag obs60/act8, 4096 envs x T=128, batch 16384, '
           'update_iters 8 (KL early stop may end an update early)'}
    for tag, r in res.items():
        for k, v in r.items():
            v = sorted(v)
            out[f'{tag}_{k}_median'] = v[len(v) // 2]
            out[f'{tag}_{k}_min'] = v[0]
    out['update_ratio'] = out['torch_update_ms_median'] / out['fused_update_ms_median']
    print(json.dumps(out, indent=1))
    if args.out:
        with open(args.out, 'w') as fh:
            json.dump(out, fh, indent=1)


if __name__ == '__main__':
    main()
