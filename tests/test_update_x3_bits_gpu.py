"""GPU: the bf16x3 kernels compute, bit for bit, what the build that wrote tests/golden/update_x3_bits.npz computed on
the same seeded inputs (tests/golden/make_golden_update_x3_bits.py): the parameters after one fused update
iteration of PPOLag (AP = 8) and of CPO's critics, the parameters after one stepwise FOCOPS pass (AP = 16, with
its forward-only statistics launches), and the actor-evaluation kernel's mu_old.  Where a product is staged between
its MMAs and its epilogue is not part of what these kernels compute, so moving it must leave every bit in place."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import make_golden_update_x3_bits as mk  # noqa: E402


@pytest.fixture(scope='module')
def bits(cuda, golden_dir):
    g = np.load(os.path.join(golden_dir, 'update_x3_bits.npz'))
    inp = {k: g[k] for k in g.files if not k.startswith('out_') and k != 'device'}
    want = {k[4:]: g[k] for k in g.files if k.startswith('out_')}
    return mk.run(inp, cuda), want


@pytest.mark.timeout(300)
@pytest.mark.parametrize('key', ['ppolag_theta', 'cpo_theta', 'focops_theta', 'mu_old'])
def test_same_bits_as_the_fixture(bits, key):
    got, want = bits
    assert got[key].shape == want[key].shape
    diff = got[key].view(np.uint32) != want[key].view(np.uint32)
    assert not diff.any(), f'{key}: {int(diff.sum())} of {diff.size} values differ, max |diff| ' \
                           f'{np.abs(got[key].astype(np.float64) - want[key]).max():.3e}'
