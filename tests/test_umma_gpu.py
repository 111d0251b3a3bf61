"""Pins the wgmma conventions (smem descriptors, 128B swizzle, K-/MN-major views of one tile,
accumulator lane mapping) with a single-CTA GEMM against numpy."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _tf32(x):
    u = np.asarray(x, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)
    return u.view(np.float32)


# K-major operands only: for tf32 wgmma an MN-major operand needs the SWIZZLE_128B_BASE32B layout
# (32-byte swizzle base), i.e. it cannot share a physical tile with the K-major view -- which is why
# the kernels produce transposed activations with role-swapped MMAs instead (csrc/update_tc.cu).
@pytest.mark.parametrize('M,N,K,a_mn,b_mn', [
    (128, 64, 64, 0, 0), (128, 16, 64, 0, 0), (128, 64, 16, 0, 0), (128, 192, 64, 0, 0), (128, 64, 128, 0, 0),
    (64, 64, 64, 0, 0), (64, 128, 64, 0, 0), (64, 64, 128, 0, 0), (64, 128, 16, 0, 0),
])
def test_umma_gemm(cuda, M, N, K, a_mn, b_mn):
    from omnisafe_b200._lib import current_stream, lib, ptr

    rng = np.random.default_rng(M + N + K + a_mn * 2 + b_mn)
    A = rng.standard_normal((M, K)).astype(np.float32)
    B = rng.standard_normal((N, K)).astype(np.float32)
    a_dev = torch.as_tensor(np.ascontiguousarray(A.T if a_mn else A)).to(cuda)
    b_dev = torch.as_tensor(np.ascontiguousarray(B.T if b_mn else B)).to(cuda)
    out = torch.full((128, N), float('nan'), dtype=torch.float32, device=cuda)
    lib().osb_umma_selftest(ptr(a_dev), ptr(b_dev), M, N, K, a_mn, b_mn, ptr(out), current_stream())
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    want = _tf32(A).astype(np.float64) @ _tf32(B).astype(np.float64).T
    if M == 128:
        np.testing.assert_allclose(got, want, rtol=2e-3, atol=2e-3)
    else:
        # M = 64: report where the 64 rows land in the accumulator image (lane mapping), then check values
        rows = [32 * (r // 16) + r % 16 for r in range(64)]   # M = 64: row r -> accumulator lane 32*(r/16) + r%16
        np.testing.assert_allclose(got[rows], want, rtol=2e-3, atol=2e-3)
