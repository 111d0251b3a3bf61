"""GPU: the slice reduction of the persistent bf16x3 update kernel, bit for bit.

After a minibatch every CTA of the persistent kernel holds its partial gradient in its accumulator image (b3 and log_std
in its row of gpart), and the owners of each parameter slice sum the G partials in a fixed order: two halves of
Gh = ceil(G / 2) CTAs, each a sequence of 32-wide pairwise trees, then half 0 + half 1.  CTAs without a tile in a short
minibatch add 0.f.  The stepwise kernel (osb_minibatch_grad_x3) assigns tiles to CTAs the same strided way and writes
each CTA's partial to gpart [CTA][P], so summing its rows in float32 in that order must give exactly the gradient the
persistent kernel stores (log_std aside, see below) (lr 0 keeps theta fixed across minibatches, max_grad_norm 0 and critic_norm_coef 0 leave the
stored gradient as reduced).  Covers the ones column (O < 64) and the db1 column (O = 64), one and sixteen actions,
three networks and one network (G up to every SM: several trees per half), a full and a short last minibatch."""
import numpy as np
import pytest
import torch

from oracle import actor_critic as oac
from test_update_gpu import _rand_data, _setup

pytestmark = pytest.mark.gpu

NETS = ('actor', 'reward_critic', 'cost_critic')
PSTR = 9472                  # row stride of the persistent kernel's gpart rows
SHORT = 4 * 128 + 77         # rows of the short last minibatch: 5 tiles, the last one partial


def _fused_sum(parts, G):
    """parts [G][n] float32 (rows of CTAs without a tile are 0) -> the persistent kernel's fixed-order sum."""
    Gh = (G + 1) // 2
    halves = []
    for h in range(2):
        b0, b1 = h * Gh, min(G, (h + 1) * Gh)
        sacc = np.zeros(parts.shape[1], np.float32)
        for b in range(b0, b1, 32):
            t = np.zeros((32, parts.shape[1]), np.float32)
            k = min(32, b1 - b)
            t[:k] = parts[b:b + k]
            w = 16
            while w:
                t[:w] = t[:w] + t[w:2 * w]
                w //= 2
            sacc = sacc + t[0]
        halves.append(sacc)
    return halves[0] + halves[1]


@pytest.mark.parametrize('short', [False, True], ids=['full', 'short'])
@pytest.mark.parametrize('mask', [7, 2])
@pytest.mark.parametrize('O,A', [(60, 8), (64, 16), (17, 6), (33, 1)])
def test_persistent_x3_reduction_bitwise(cuda, O, A, mask, short):
    from omnisafe_b200._lib import current_stream, lib, ptr

    L, stream = lib(), current_stream()
    cap = L.osb_tc_grid_blocks(1 << 40, mask)
    batch = 128 * cap * (2 if mask == 7 else 1)
    total = batch + (SHORT if short else 0)
    N, T = 64, 288
    assert N * T >= total
    rng = np.random.default_rng(O + 10 * A + mask)
    theta = oac.init_theta(O, A, seed=O + A)
    data = _rand_data(rng, N, T, O, A, theta)
    agent, buf, eng = _setup(cuda, data, N, T, O, A, theta)
    buf.adv_moments.copy_(torch.tensor([0.37, 2.3, -0.41, 1.0]))
    perm = torch.as_tensor(rng.permutation(N * T)[:total].astype(np.int32)).to(cuda)
    lag = torch.tensor([0.37, 0, 0, 0], dtype=torch.float32, device=cuda)
    d, a, P = buf.data, agent, eng.P
    start, count = (batch, SHORT) if short else (0, batch)

    # per-CTA partials of the last minibatch from the stepwise kernel
    nb = L.osb_tc_grid_blocks(count, mask)
    gpart = torch.zeros(nb * P, dtype=torch.float32, device=cuda)
    stats = torch.zeros(148 * 3 * 8, dtype=torch.float32, device=cuda)
    assert L.osb_minibatch_grad_x3(
        ptr(a.theta), O, A, ptr(d['obs']), ptr(d['act']), ptr(d['logp']), ptr(d['adv_r']), ptr(d['adv_c']),
        ptr(d['target_value_r']), ptr(d['target_value_c']), ptr(eng.mu_old), ptr(buf.adv_moments), ptr(perm), total, 0,
        start, count, 0, 0.2, 0.0, 1.0, 0.0, ptr(lag), ptr(eng.logstd_old), mask, ptr(gpart), ptr(stats),
        ptr(eng.stop_flag), stream) == 0
    torch.cuda.synchronize()
    parts = gpart.cpu().numpy().reshape(nb, P)

    # the persistent kernel over every minibatch, nothing moved: lr 0, no clipping, no critic L2 term
    G = L.osb_tc_grid_blocks(min(batch, total), mask)
    fused_gpart = torch.zeros(3 * G * PSTR, dtype=torch.float32, device=cuda)
    a.grad.fill_(float('nan'))
    assert L.osb_ppo_update_iter_x3(
        ptr(a.theta), ptr(a.grad), ptr(a.adam_m), ptr(a.adam_v), ptr(a.adam_step), O, A, ptr(d['obs']), ptr(d['act']),
        ptr(d['logp']), ptr(d['adv_r']), ptr(d['adv_c']), ptr(d['target_value_r']), ptr(d['target_value_c']),
        ptr(buf.adv_moments), ptr(perm), total, 0, batch, 0, 0.2, 0.0, ptr(lag), mask, 0.0, 0.0, 0.0, 0.0, 0.0,
        ptr(fused_gpart), ptr(eng.stats_part), ptr(eng.train_stats), ptr(eng.stop_flag), 0, 0, 1, 0, 0, stream) == 0
    torch.cuda.synchronize()
    got = a.grad.cpu().numpy()
    assert np.array_equal(a.theta.cpu().numpy(), theta.astype(np.float32))

    assert nb == (-(-count // 128) if short else G), (nb, G, count)
    lay = oac.layout(O, A)
    for j, net in enumerate(NETS):
        if not (mask >> j) & 1:
            continue
        sl = slice(lay[net]['start'], lay[net]['start'] + lay[net]['size'])
        rows = np.zeros((G, sl.stop - sl.start), np.float32)
        rows[:nb] = parts[:, sl]
        want = _fused_sum(rows, G)
        # log_std's partial is the loss epilogue's own sum, which the stepwise kernel's extended loss rounds differently
        # (last bits, with two tiles per CTA); it is checked against float64 in test_optimizer_gpu
        keep = np.arange(sl.stop - sl.start) >= (A if net == 'actor' else 0)
        bad = np.flatnonzero((got[sl].view(np.uint32) != want.view(np.uint32)) & keep)
        assert bad.size == 0, (net, G, nb, bad[:8], got[sl][bad[:8]], want[bad[:8]])
    print(f'[O={O} A={A} mask={mask} {"short" if short else "full"}] G={G}, {nb} CTAs with tiles: bit-identical')
