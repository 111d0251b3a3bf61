// Self-test of the tf32 wgmma building blocks: D[M][N] = A * B^T on one warpgroup, used by
// tests/test_umma_gpu.py to pin the descriptor / swizzle / accumulator-lane conventions on real hardware.
#include "common.cuh"
#include "umma.cuh"

namespace osb {

// A[M][K], B[N][K] (row-major fp32), both staged K-major.  out[128][N]: dump of accumulator lanes 0..127.
__global__ void __launch_bounds__(128, 1) umma_selftest_kernel(const float* __restrict__ A,
                                                               const float* __restrict__ B, int M, int N,
                                                               int K, float* __restrict__ scratch,
                                                               float* __restrict__ out) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int Kp = (K + 31) & ~31;
    uint8_t* sA = smem;
    uint8_t* sB = smem + (size_t)(Kp / 32) * M * 128;
    const int tid = threadIdx.x;
    for (int i = tid; i < M * Kp; i += 128) {
        const int r = i / Kp, c = i % Kp;
        *reinterpret_cast<float*>(sA + umma::sw128_offset(r, c, M)) = (c < K) ? A[(size_t)r * K + c] : 0.f;
    }
    for (int i = tid; i < N * Kp; i += 128) {
        const int r = i / Kp, c = i % Kp;
        *reinterpret_cast<float*>(sB + umma::sw128_offset(r, c, N)) = (c < K) ? B[(size_t)r * K + c] : 0.f;
    }
    umma::fence_async_smem();
    __syncthreads();
    const umma::Acc acc = umma::acc_cta(scratch, (uint32_t)N);
    umma::tc_gemm(acc, 0u, umma::smem_u32(sA), M, umma::smem_u32(sB), N, M, N, K, false);
    __threadfence_block();
    __syncthreads();
    for (int c0 = 0; c0 < N; c0 += 16) {
        float v[16];
        umma::acc_ld16(acc, ((uint32_t)(tid & ~31) << 16) + (uint32_t)c0, v);
        for (int j = 0; j < 16; ++j) out[(size_t)tid * N + c0 + j] = v[j];
    }
}

}  // namespace osb

extern "C" int osb_umma_selftest(const float* A, const float* B, int M, int N, int K, int a_mn, int b_mn,
                                 float* out, void* stream) {
    OSB_CHECK_ARG(A && B && out, "null pointer");
    OSB_CHECK_ARG(!a_mn && !b_mn, "tf32 wgmma reads both operands K-major");
    OSB_CHECK_ARG((M == 64 || M == 128) && (N == 16 || (N % 64 == 0 && N <= 256)) && K % 8 == 0 && K >= 8 && K <= 128,
                  "bad shape");
    float* scratch = osb::acc_scratch(osb::ACC_SELFTEST, (size_t)128 * N * sizeof(float));
    if (!scratch) return OSB_ERR_CUDA;
    const size_t smem = 1024 + (size_t)((K + 31) / 32) * (M + N) * 128;
    OSB_CUDA(cudaFuncSetAttribute(osb::umma_selftest_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    osb::umma_selftest_kernel<<<1, 128, smem, (cudaStream_t)stream>>>(A, B, M, N, K, scratch, out);
    OSB_LAUNCH_CHECK();
    return OSB_OK;
}
