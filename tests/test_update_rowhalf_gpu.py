"""The bf16x3 update kernel issues every product of its forward / backward chain once per row half of the 128-sample
tile (`gemm_x3_rows`, csrc/x3.cuh): one m64 block over the whole K, for K = 64 as two wgmma chains whose fp32 sum is
stored.  Pinned here on real hardware: the row-half product meets the fp64 product at the fp32 bar of the other bf16x3
shapes, and it is bit for bit what the M = 128 product leaves in the accumulator image when it is issued in two
column-half phases of which the second adds to the first -- so a kernel may switch between the two schedules without
changing a result."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# (N, K, b_mn, a_sw, b_sw) -- the row-half products of one tile of the update kernel
CASES = [
    (64, 64, 0, 128, 128),     # Z1 / Z2      = X  W^T     (B K-major)
    (64, 64, 1, 128, 128),     # dZ1 pre-act  = dZ2 W2     (B: W2 tile MN-major)
    (16, 64, 0, 128, 128),     # OUT          = H2 W3^T
    (64, 16, 1, 32, 128),      # dZ2 pre-act  = dOUT W3    (A: SW32, one k-step: a single chain)
]


@pytest.mark.parametrize('N,K,b_mn,a_sw,b_sw', CASES)
def test_row_half_product(cuda, N, K, b_mn, a_sw, b_sw):
    from omnisafe_b200._lib import current_stream, lib, ptr

    rng = np.random.default_rng(11 * N + 5 * K + b_mn)
    A = (rng.standard_normal((128, K)) * np.exp(rng.uniform(-4, 4, (128, 1)))).astype(np.float32)
    B = rng.standard_normal((N, K)).astype(np.float32)
    out = torch.full((128, N), float('nan'), dtype=torch.float32, device=cuda)
    phases = torch.full((128, N), float('nan'), dtype=torch.float32, device=cuda)
    a_dev, b_dev = torch.as_tensor(A).to(cuda), torch.as_tensor(B).to(cuda)     # keep both alive across the launch
    lib().osb_x3_rows_selftest(ptr(a_dev), ptr(b_dev), N, K, b_mn, a_sw, b_sw, ptr(out), ptr(phases), current_stream())
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    want = A.astype(np.float64) @ B.astype(np.float64).T
    scale = np.abs(A).astype(np.float64) @ np.abs(B).astype(np.float64).T
    err = np.abs(got.astype(np.float64) - want) / scale
    print(f'x3 row halves 128x{N}x{K}: max err / (|A||B|^T) = {err.max():.3e}')
    assert err.max() < 1e-6
    assert np.array_equal(got.view(np.uint32), phases.cpu().numpy().view(np.uint32)), \
        'row-half product differs from the column-half phases in the last bits'


def test_other_shapes_are_refused(cuda):
    from omnisafe_b200._lib import OsbError, current_stream, lib, ptr

    a = torch.zeros((128, 64), dtype=torch.float32, device=cuda)
    out = torch.zeros((128, 64), dtype=torch.float32, device=cuda)
    with pytest.raises(OsbError):
        lib().osb_x3_rows_selftest(ptr(a), ptr(a), 64, 32, 0, 128, 128, ptr(out), ptr(out), current_stream())
