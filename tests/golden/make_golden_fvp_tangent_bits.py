"""Generate tests/golden/fvp_tangent_bits.npz: what the tensor-core Fisher-vector product computes, bit for bit, on
seeded inputs -- tests/test_fvp_tangent_bits_gpu.py holds every later build to the same bits.

For each case and precision (tf32: osb_fvp_partials_tc, bf16x3: osb_fvp_partials_x3) it records F v, the partials
reduced by osb_reduce_partials, and the SHA-256 of the bytes of the tangent scratch dmu [total][A] (rows 0, stride,
2 stride, ... written, the others left zero): the scratch of the large cases would make the fixture megabytes.  The
inputs are not stored; they are drawn again from the seed, and the fixture keeps the SHA-256 of their bytes so that a
change of numpy's streams shows as such.

  o17     : O % 4 != 0 (scalar row gathers)
  a1      : one action dimension
  o64_a16 : the widest bf16x3 shape
  many    : about 40 000 rows, more tiles than CTAs, a short last tile
  stride3 : every third row
  o111    : tf32 only, layer 1 over two K chunks, O % 4 != 0
  o376    : tf32 only, layer 1 over six K chunks

    python tests/golden/make_golden_fvp_tangent_bits.py [--out PATH]

Needs an H100 and a built library (python -c "import __graft_entry__ as g; g.build()")."""
from __future__ import annotations

import argparse
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

FNAME = os.path.join(HERE, 'fvp_tangent_bits.npz')
CASES = {
    # name: (O, A, total, stride, precisions)
    'o17': (17, 8, 3001, 1, ('tf32', 'bf16x3')),
    'a1': (60, 1, 2050, 1, ('tf32', 'bf16x3')),
    'o64_a16': (64, 16, 4000, 1, ('tf32', 'bf16x3')),
    'many': (60, 8, 40001, 1, ('tf32', 'bf16x3')),
    'stride3': (60, 8, 9001, 3, ('tf32', 'bf16x3')),
    'o111': (111, 8, 3001, 1, ('tf32',)),
    'o376': (376, 6, 2000, 1, ('tf32',)),
}


def make_inputs(seed: int = 20261017) -> dict:
    """Seeded actor parameters (random log_std), directions and observations of every case (CPU, numpy)."""
    from oracle import actor_critic as oac

    out = {}
    for i, (name, (O, A, total, _, _)) in enumerate(CASES.items()):
        rng = np.random.default_rng(seed + i)
        Pa = oac.layout(O, A)['actor']['size']
        theta = oac.init_theta(O, A, seed=seed % 1000 + i)[:Pa].copy()
        theta[:A] = rng.uniform(-0.5, 0.5, A)
        out[f'{name}_theta'] = theta.astype(np.float32)
        out[f'{name}_vec'] = rng.standard_normal(Pa).astype(np.float32)
        out[f'{name}_obs'] = rng.standard_normal((total, O)).astype(np.float32)
    return out


def inputs_sha256(inp: dict) -> str:
    h = hashlib.sha256()
    for k in sorted(inp):
        h.update(k.encode())
        h.update(np.ascontiguousarray(inp[k]).tobytes())
    return h.hexdigest()


def run(inp: dict, dev) -> dict:
    """The kernels' outputs on `inp` (make_inputs' dict)."""
    import torch

    from omnisafe_b200._lib import current_stream, lib, ptr

    out = {}
    for name, (O, A, total, stride, precs) in CASES.items():
        theta = torch.as_tensor(inp[f'{name}_theta']).to(dev)
        vec = torch.as_tensor(inp[f'{name}_vec']).to(dev)
        obs = torch.as_tensor(inp[f'{name}_obs']).to(dev)
        Pa = theta.numel()
        nb = lib().osb_tc_grid_blocks((total + stride - 1) // stride, 1)
        for prec in precs:
            fn = lib().osb_fvp_partials_tc if prec == 'tf32' else lib().osb_fvp_partials_x3
            dmu = torch.zeros(total * A, dtype=torch.float32, device=dev)
            gpart = torch.zeros(nb * Pa, dtype=torch.float32, device=dev)
            stats = torch.zeros(nb * 24, dtype=torch.float32, device=dev)
            fv = torch.zeros(Pa, dtype=torch.float32, device=dev)
            fn(ptr(theta), ptr(vec), O, A, ptr(obs), total, stride, ptr(dmu), ptr(gpart), ptr(stats), current_stream())
            lib().osb_reduce_partials(ptr(gpart), nb, Pa, Pa, 1.0, 0, 0.0, ptr(fv), current_stream())
            torch.cuda.synchronize()
            out[f'{name}_{prec}_dmu_sha256'] = np.array(hashlib.sha256(dmu.cpu().numpy().tobytes()).hexdigest())
            out[f'{name}_{prec}_fv'] = fv.cpu().numpy()
    return out


def main() -> None:
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=FNAME)
    args = ap.parse_args()
    import omnisafe_b200  # noqa: F401  (binds the built library)

    inp = make_inputs()
    out = run(inp, torch.device('cuda:0'))
    np.savez_compressed(args.out, inputs_sha256=np.array(inputs_sha256(inp)), **{f'out_{k}': v for k, v in out.items()},
                        device=np.array(torch.cuda.get_device_name(0)))
    print('wrote', args.out, {k: v.shape for k, v in out.items()})


if __name__ == '__main__':
    main()
