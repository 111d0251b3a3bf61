"""Where one CTA of the persistent bf16x3 update kernel spends its time: clock64 stamps of the selected CTA
(thread 0 = warp 0: rows 0-63, statistics and actions 0 .. AP / 4 - 1 of the loss; thread 320 = warp 10: rows 64-127;
thread 512 = the MMA-issue warpgroup).  All three threads run on one SM, so their clocks are comparable.

    python tools/x3_stage_times.py [--cta X Y] ...     (default: --cta 0 0 --cta 0 1, an actor CTA and a critic CTA)
"""
import argparse, os, statistics, sys, tempfile
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import omnisafe_b200, bench
from omnisafe_b200._lib import lib, ptr

REGION = 4096                 # X3_DBG_REGION (csrc/update_x3.cu); the selected CTA follows the three regions
NAMES = {0: 'E0 start', 1: 'X free', 2: 'X stored+sync', 3: 'C1 ok', 4: 'E1 done', 5: 'C2 ok', 6: 'E2 done', 7: 'C3 ok', 8: 'dOUT stored', 9: 'E3 done',
         10: 'C4A ok', 11: 'E4 computed', 12: 'C4B ok', 13: 'E4 stored', 14: 'C5A ok', 15: 'E5 computed', 16: 'C5B ok', 17: 'E5 stored', 20: 'tiles done',
         32: 'stats stored', 35: 'next rows', 21: 'C6 ok', 22: 'partials out', 23: 'barrier1', 29: 'partials loaded', 30: 'norm published', 31: 'Adam state in',
         24: 'Adam stored', 25: 'barrier2', 26: 'adam done', 27: 'barrier3', 28: 'restaged',
         200: 'dW3 read H2', 201: 'dW2 read H2, H1', 202: 'dW1 read X', 203: 'gradients committed', 204: 'dW2 stored',
         205: 'dZ1 ready', 206: 'dW1 stored', 207: 'db2 stored'}
# MMA-issue warpgroup: 100 + 20 k for product k, + 4 r + event for row half r
for k, prod in enumerate(('Z1', 'Z2', 'OUT', "dZ2'", "dZ1'")):
    for r in range(2):
        for ev, what in enumerate(('operands ready', 'MMAs complete', 'stored', 'committed')):
            NAMES[100 + 20 * k + 4 * r + ev] = f'{prod}[{r}] {what}'


def rows_of(d, region):
    d = d[region * REGION:(region + 1) * REGION]
    return [(d[1 + 2 * i], d[2 + 2 * i]) for i in range(d[0])]


def report(d):
    epi = rows_of(d, 0)
    mma = rows_of(d, 2)
    for which, rows in (('thread 0', epi), ('thread 320', rows_of(d, 1)), ('MMA-issue warpgroup (thread 512)', mma)):
        hops = {}
        for (_, c0), (id1, c1) in zip(rows, rows[1:]):
            hops.setdefault(id1, []).append(c1 - c0)
        print(f'== {which}: {len(rows)} stamps, median cycles from the previous stamp')
        for id_ in sorted(hops):
            print(f'  {NAMES.get(id_, id_):24s} {statistics.median(hops[id_]):8.0f} cyc  (n = {len(hops[id_])})')
    per_tile, start = [], None
    for id_, clk in epi:
        if id_ == 0:
            if start is not None: per_tile.append(clk - start)
            start = clk
        elif id_ == 20:
            start = None
    if per_tile:
        print(f'  cycles per tile (thread 0, E0 start to E0 start inside a minibatch): median {statistics.median(per_tile):.0f}  (n = {len(per_tile)})')
    # the minibatch boundary on one clock: every stamp of thread 0 from its last 'E5 stored' of a minibatch to 'restaged',
    # and those of the MMA-issue warpgroup in that window, relative to thread 0's 'E5 stored'
    bounds = []
    for i, (id_, clk) in enumerate(epi):
        if id_ == 20:
            j = i
            while j > 0 and epi[j][0] != 17: j -= 1
            k = i
            while k < len(epi) and epi[k][0] != 28: k += 1
            if k < len(epi): bounds.append((epi[j][1], epi[j:k + 1]))
    # the first minibatch of the launch is left out, and so are those past the MMA-issue warpgroup's last stamp
    bounds = [b for b in bounds[1:] if mma and mma[-1][1] >= b[1][-1][1]]
    events = {}
    for t0, seg in bounds:
        t1 = seg[-1][1]
        for id_, clk in seg: events.setdefault(('epi', id_), []).append(clk - t0)
        last = {}
        for id_, clk in mma:
            if t0 - 15000 <= clk <= t1: last[id_] = clk - t0        # its last occurrence in the window
        for id_, dt in last.items(): events.setdefault(('mma', id_), []).append(dt)
    if bounds:
        print(f'== boundary on one clock: median cycles after thread 0\'s last "E5 stored" (n = {len(bounds)} minibatches)')
        for (who, id_), v in sorted(events.items(), key=lambda kv: statistics.median(kv[1])):
            if len(v) == len(bounds):
                print(f'  {who:3s} {NAMES.get(id_, id_):24s} {statistics.median(v):8.0f}')
        total = [seg[-1][1] - seg[0][1] for _, seg in bounds]
        print(f'  boundary, "E5 stored" to "restaged": median {statistics.median(total):.0f} cycles')


ap = argparse.ArgumentParser()
ap.add_argument('--cta', nargs=2, type=int, action='append', metavar=('X', 'Y'), help='blockIdx.x, blockIdx.y (y = network)')
args = ap.parse_args()
ctas = args.cta or [(0, 0), (0, 1)]
cfg = bench._custom_cfgs(1, tempfile.mkdtemp(), 40)
cfg['train_cfgs']['matmul_precision'] = 'bf16x3'
algo = omnisafe_b200.Agent('PPOLag', 'SyntheticBox-v0', custom_cfgs=cfg).agent
for _ in range(2): algo.train_epoch()
print(torch.cuda.get_device_name(), 'power limit / max SM clock:', os.popen('nvidia-smi --query-gpu=power.limit,clocks.max.sm --format=csv,noheader').read().strip())
for x, y in ctas:
    dbg = torch.zeros(3 * REGION + 1, dtype=torch.int64, device='cuda')
    dbg[3 * REGION] = x | (y << 16)
    torch.cuda.synchronize()
    lib().osb_x3_debug_buffer(ptr(dbg))
    algo._update()
    torch.cuda.synchronize()
    lib().osb_x3_debug_buffer(0)
    print(f'######## CTA ({x}, {y}): {"actor" if y == 0 else "critic"} (stamps of the last update iteration)')
    report(dbg.cpu().tolist())
