"""Generate tests/golden/update_x3_bits.npz: what the bf16x3 kernels compute, bit for bit, on seeded inputs whose last
minibatch is short -- tests/test_update_x3_bits_gpu.py holds every later build to the same bits.

  ppolag : the parameters after one fused update iteration of PPOLag (loss PPO-clip, all three networks, obs 60,
           act 8: the AP = 8 kernel), minibatches 320, 320, 128
  cpo    : the same after one fused critics-only iteration (CPO's critic update) on the same data
  focops : the parameters after one stepwise FOCOPS pass (forward-only statistics pass + gradient launch per minibatch,
           obs 33, act 16: the AP = 16 kernel), minibatches 288, 288, 144
  mu_old : the actor's mean over the FOCOPS slab from the bf16x3 actor-evaluation kernel at the initial parameters

    python tests/golden/make_golden_update_x3_bits.py [--out PATH]

Needs an H100 and a built library (python -c "import __graft_entry__ as g; g.build()")."""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.dirname(HERE)):
    if p not in sys.path:
        sys.path.insert(0, p)

FNAME = os.path.join(HERE, 'update_x3_bits.npz')
CASES = {
    # name: (N, T, O, A, batch)
    'ppo': (32, 24, 60, 8, 320),
    'focops': (24, 30, 33, 16, 288),
}
DATA_KEYS = ('obs', 'act', 'logp', 'adv_r', 'adv_c', 'target_value_r', 'target_value_c')


def make_inputs(seed: int = 20261017) -> dict:
    """Seeded parameters, env-major slabs and minibatch orders of both cases (CPU, numpy)."""
    from oracle import actor_critic as oac
    from test_update_gpu import _rand_data

    out = {}
    for i, (name, (N, T, O, A, _)) in enumerate(CASES.items()):
        rng = np.random.default_rng(seed + i)
        theta = oac.init_theta(O, A, seed=seed % 1000 + i)
        data = _rand_data(rng, N, T, O, A, theta)
        out[f'{name}_theta0'] = theta.astype(np.float32)
        for k in DATA_KEYS:
            out[f'{name}_{k}'] = np.asarray(data[k], np.float32)
        out[f'{name}_perm'] = rng.permutation(N * T).astype(np.int64)
    return out


def run(inp: dict, dev) -> dict:
    """The kernels' outputs on `inp` (make_inputs' dict, or the fixture's copy of it)."""
    import torch

    from test_update_gpu import _rows, _setup

    out = {}
    # PPOLag: one fused iteration of every network; CPO: one fused iteration of the two critics
    N, T, O, A, batch = CASES['ppo']
    data = {k: inp[f'ppo_{k}'] for k in DATA_KEYS}
    perm = torch.as_tensor(_rows(inp['ppo_perm'], N, T)[None]).to(dev)
    for name, loss_kind, net_mask in (('ppolag', 0, 7), ('cpo', 1, 6)):
        agent, buf, eng = _setup(dev, data, N, T, O, A, inp['ppo_theta0'])
        lag = torch.tensor([0.37, 0.0, 0.0, 0.0], dtype=torch.float32, device=dev)
        eng.ppo_epoch(loss_kind=loss_kind, lagrange=lag, net_mask=net_mask, batch_size=batch, update_iters=1, clip=0.2,
                      entropy_coef=0.0, critic_norm_coef=0.001, max_grad_norm=40.0, lr_actor=3e-4, lr_critic=3e-4,
                      target_kl=10.0, kl_early_stop=False, perm=perm, precision=2)
        torch.cuda.synchronize()
        out[f'{name}_theta'] = agent.theta.cpu().numpy()
    # FOCOPS, stepwise: the old policy from the actor-evaluation kernel, then per minibatch the statistics pass, the
    # gradient launch and the optimiser
    N, T, O, A, batch = CASES['focops']
    data = {k: inp[f'focops_{k}'] for k in DATA_KEYS}
    perm = torch.as_tensor(_rows(inp['focops_perm'], N, T)[None]).to(dev)
    agent, buf, eng = _setup(dev, data, N, T, O, A, inp['focops_theta0'])
    eng.precision = 2
    eng.snapshot_old_policy()
    torch.cuda.synchronize()
    out['mu_old'] = eng.mu_old.cpu().numpy()
    lag = torch.tensor([0.37, 0.0, 0.0, 0.0], dtype=torch.float32, device=dev)
    eng.stepwise_epoch({}, loss_kind=2, lagrange=lag, net_mask=1, batch_size=batch, update_iters=1, clip=0.2,
                       focops_lam=1.5, focops_eta=0.02, max_grad_norm=40.0, lr_actor=3e-4, lr_critic=3e-4,
                       target_kl=10.0, kl_early_stop=False, perm=perm)
    torch.cuda.synchronize()
    out['focops_theta'] = agent.theta.cpu().numpy()
    return out


def main() -> None:
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=FNAME)
    args = ap.parse_args()
    import omnisafe_b200  # noqa: F401  (binds the built library)

    inp = make_inputs()
    out = run(inp, torch.device('cuda:0'))
    np.savez_compressed(args.out, **inp, **{f'out_{k}': v for k, v in out.items()},
                        device=np.array(torch.cuda.get_device_name(0)))
    print('wrote', args.out, {k: v.shape for k, v in out.items()})


if __name__ == '__main__':
    main()
