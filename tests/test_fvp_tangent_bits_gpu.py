"""GPU: the tensor-core Fisher-vector product (tangent pass and LOSS_FVP backward, tf32 and bf16x3) computes, bit for
bit, what the build that wrote tests/golden/fvp_tangent_bits.npz computed on the same seeded inputs
(tests/golden/make_golden_fvp_tangent_bits.py): the reduced F v and the tangent scratch dmu, at O % 4 != 0, A = 1,
O = 64 / A = 16, more tiles than CTAs, stride 3 and (tf32) the K-chunked layer 1."""
import hashlib
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import make_golden_fvp_tangent_bits as mk  # noqa: E402


@pytest.fixture(scope='module')
def bits(cuda, golden_dir):
    g = np.load(os.path.join(golden_dir, 'fvp_tangent_bits.npz'))
    inp = mk.make_inputs()
    assert mk.inputs_sha256(inp) == str(g['inputs_sha256']), 'the seeded inputs are not the ones the fixture was made from'
    want = {k[4:]: g[k] for k in g.files if k.startswith('out_')}
    return mk.run(inp, cuda), want


KEYS = [f'{name}_{prec}' for name, (*_, precs) in mk.CASES.items() for prec in precs]


@pytest.mark.timeout(300)
@pytest.mark.parametrize('key', KEYS)
def test_same_bits_as_the_fixture(bits, key):
    got, want = bits
    g, w = got[f'{key}_fv'], want[f'{key}_fv']
    assert g.shape == w.shape
    diff = g.view(np.uint32) != w.view(np.uint32)
    assert not diff.any(), f'{key} F v: {int(diff.sum())} of {diff.size} values differ, max |diff| ' \
                           f'{np.abs(g.astype(np.float64) - w).max():.3e}'
    assert str(got[f'{key}_dmu_sha256']) == str(want[f'{key}_dmu_sha256']), f'{key}: the dmu scratch differs'
