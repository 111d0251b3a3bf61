"""Where one CTA of the persistent bf16x3 update kernel spends its time: clock64 stamps of CTA (0, 0)
(thread 0 = warp 0: rows 0-63, statistics and actions 0 .. AP / 4 - 1 of the loss; thread 320 = warp 10: rows 64-127;
thread 512 = the MMA-issue warpgroup)."""
import os, sys, tempfile
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import omnisafe_b200, bench
from omnisafe_b200._lib import lib, ptr
cfg = bench._custom_cfgs(1, tempfile.mkdtemp(), 40)
cfg['train_cfgs']['matmul_precision'] = 'bf16x3'
algo = omnisafe_b200.Agent('PPOLag', 'SyntheticBox-v0', custom_cfgs=cfg).agent
for _ in range(2): algo.train_epoch()
dbg = torch.zeros(3072, dtype=torch.int64, device='cuda')
torch.cuda.synchronize()
lib().osb_x3_debug_buffer(ptr(dbg))
algo._update()
torch.cuda.synchronize()
lib().osb_x3_debug_buffer(0)
NAMES = {0: 'E0 start', 1: 'X free', 2: 'X stored+sync', 3: 'C1 ok', 4: 'E1 done', 5: 'C2 ok', 6: 'E2 done', 7: 'C3 ok', 8: 'dOUT stored', 9: 'E3 done',
         10: 'C4A ok', 11: 'E4 computed', 12: 'C4B ok', 13: 'E4 stored', 14: 'C5A ok', 15: 'E5 computed', 16: 'C5B ok', 17: 'E5 stored', 20: 'tiles done',
         21: 'C6 ok', 22: 'partials out', 23: 'barrier1', 29: 'partials loaded', 30: 'norm published', 31: 'Adam state in',
         24: 'Adam stored', 25: 'barrier2', 26: 'adam done', 27: 'barrier3', 28: 'restaged',
         200: 'dW3 read H2', 201: 'dW2 read H2, H1', 202: 'dW1 read X', 203: 'gradients committed'}
# MMA-issue warpgroup: 100 + 20 k for product k, + 4 r + event for row half r
for k, prod in enumerate(('Z1', 'Z2', 'OUT', "dZ2'", "dZ1'")):
    for r in range(2):
        for ev, what in enumerate(('operands ready', 'MMAs complete', 'stored', 'committed')):
            NAMES[100 + 20 * k + 4 * r + ev] = f'{prod}[{r}] {what}'
for which, off in (('thread 0 (rows 0-63)', 0), ('thread 320 (rows 64-127)', 1024)):
    d = dbg[off:off + 1024].cpu().tolist()
    n = d[0]
    print(f'== {which}: {n} stamps (last update iteration kept the buffer)')
    prev = None
    # print the first minibatch only (until second id 28) ... stamps restart every launch: take the tail launch
    rows = [(d[1 + 2 * i], d[2 + 2 * i]) for i in range(n)]
    # first minibatch of the (last) launch
    t0 = rows[0][1]
    cnt28 = 0
    for id_, clk in rows:
        dt = 0 if prev is None else clk - prev
        print(f'  {NAMES.get(id_, id_):16s} +{dt:7d} cyc   t={clk - t0:8d}')
        prev = clk
        if id_ == 28:
            cnt28 += 1
            if cnt28 == 2: break
# the first minibatch above is one sample of each hop: the median over every stamped tile is steadier
import statistics
for which, off in (('thread 0', 0), ('thread 320', 1024)):
    d = dbg[off:off + 1024].cpu().tolist()
    rows = [(d[1 + 2 * i], d[2 + 2 * i]) for i in range(d[0])]
    hops = {}
    for (_, c0), (id1, c1) in zip(rows, rows[1:]):
        hops.setdefault(id1, []).append(c1 - c0)
    print(f'== {which}: median cycles from the previous stamp, over all stamps of the launch')
    for id_ in sorted(hops):
        print(f'  {NAMES.get(id_, id_):16s} {statistics.median(hops[id_]):8.0f} cyc  (n = {len(hops[id_])})')
    per_tile, start = [], None
    for id_, clk in rows:
        if id_ == 0:
            if start is not None: per_tile.append(clk - start)
            start = clk
        elif id_ == 20:                    # the optimiser phases follow: not a tile
            start = None
    if per_tile:
        print(f'  cycles per tile (E0 start to E0 start inside a minibatch): median {statistics.median(per_tile):.0f}  (n = {len(per_tile)})')
d = dbg[2048:3072].cpu().tolist()
rows = [(d[1 + 2 * i], d[2 + 2 * i]) for i in range(d[0])]
hops = {}
for (_, c0), (id1, c1) in zip(rows, rows[1:]):
    hops.setdefault(id1, []).append(c1 - c0)
print('== MMA-issue warpgroup (thread 512): median cycles from its previous stamp')
for id_ in sorted(hops):
    print(f'  {NAMES.get(id_, id_):24s} {statistics.median(hops[id_]):8.0f} cyc  (n = {len(hops[id_])})')
