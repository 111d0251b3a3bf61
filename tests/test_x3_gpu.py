"""Pins the split-bf16 ("bf16x3", bf16 wgmma) building blocks of csrc/x3.cuh on real hardware:
the K-major and MN-major views of one physical SW128 / SW32 bf16 tile, the six-product compensation,
and its fp32-level accuracy (the parity-grade tensor-core mode rests on these conventions)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# (M, N, K, a_mn, b_mn, a_sw, b_sw, b_ones) -- the eight GEMM shapes of one 128-sample tile of the update kernel
CASES = [
    (128, 64, 64, 0, 0, 128, 128, 0),    # Z1 / Z2      = X  W^T        (both K-major)
    (128, 16, 64, 0, 0, 128, 128, 0),    # OUT          = H2 W3^T
    (128, 64, 16, 0, 1, 32, 128, 0),     # dZ2 pre-act  = dOUT W3       (A: SW32 K-major, B: W3 tile MN-major)
    (128, 64, 64, 0, 1, 128, 128, 0),    # dZ1 pre-act  = dZ2 W2        (B: W2 tile MN-major)
    (64, 64, 128, 1, 1, 128, 128, 0),    # dW2 / dW1    = dZ^T H        (both MN-major: contraction over samples)
    (64, 16, 128, 1, 1, 128, 32, 0),     # dW3^T        = H2^T dOUT     (B: SW32 MN-major)
    (64, 16, 128, 1, 1, 128, 32, 1),     # bias grads   = dZ^T 1        (ones tile)
    (64, 64, 64, 0, 0, 128, 128, 0),     # M = 64 lane mapping
]


@pytest.mark.parametrize('M,N,K,a_mn,b_mn,a_sw,b_sw,b_ones', CASES)
def test_x3_gemm(cuda, M, N, K, a_mn, b_mn, a_sw, b_sw, b_ones):
    from omnisafe_b200._lib import current_stream, lib, ptr

    rng = np.random.default_rng(M + 3 * N + 7 * K + a_mn * 2 + b_mn + a_sw)
    A = (rng.standard_normal((M, K)) * np.exp(rng.uniform(-4, 4, (M, 1)))).astype(np.float32)
    B = rng.standard_normal((N, K)).astype(np.float32)
    if b_ones:
        B[:] = 1.0
    out = torch.full((128, N), float('nan'), dtype=torch.float32, device=cuda)
    a_dev, b_dev = torch.as_tensor(A).to(cuda), torch.as_tensor(B).to(cuda)     # keep both alive across the launch
    lib().osb_x3_selftest(ptr(a_dev), ptr(b_dev), M, N, K, a_mn, b_mn, a_sw, b_sw, b_ones, ptr(out), current_stream())
    torch.cuda.synchronize()
    got = out.cpu().numpy().astype(np.float64)
    want = A.astype(np.float64) @ B.astype(np.float64).T
    scale = np.abs(A).astype(np.float64) @ np.abs(B).astype(np.float64).T
    rows = list(range(128)) if M == 128 else [32 * (r // 16) + r % 16 for r in range(64)]   # M = 64: row r -> lane 32*(r/16) + r%16
    err = np.abs(got[rows] - want) / scale
    print(f'x3 gemm {M}x{N}x{K}: max err / (|A||B|^T) = {err.max():.3e}')
    assert err.max() < 1e-6      # fp32-level: K = 128 fp32 accumulation noise included (a tf32 product sits at 5e-4)
