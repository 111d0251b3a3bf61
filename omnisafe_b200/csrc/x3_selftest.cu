// Self-test of the split-bf16 tensor-core building blocks of csrc/x3.cuh: pins on real hardware the K-major /
// MN-major views of one SW128 or SW32 bf16 tile, the 6-product compensation and its accuracy
// (tests/test_x3_gpu.py).
#include "common.cuh"
#include "x3.cuh"

namespace osb {

// A: row-major fp32 [M][K], B: row-major fp32 [N][K].  out[128][N]: dump of accumulator lanes 0..127.
// a_mn / b_mn: operand consumed MN-major (tile rows = K index) instead of K-major (tile rows = M/N index).
// a_sw / b_sw: 128 (tile rows of 64 bf16) or 32 (tile rows of 16 bf16).  b_ones: B is the all-ones tile
// (exact in bf16: three MMAs per k-step).
__global__ void __launch_bounds__(128, 1) x3_selftest_kernel(const float* __restrict__ A, const float* __restrict__ B,
                                                             int M, int N, int K, int a_mn, int b_mn, int a_sw,
                                                             int b_sw, int b_ones, float* __restrict__ scratch,
                                                             float* __restrict__ out) {
    using namespace x3;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const uint32_t pad = (1024u - (smem_u32(smem_raw) & 1023u)) & 1023u;
    const uint32_t sA = smem_u32(smem_raw) + pad;
    const int tid = threadIdx.x;
    const int rowsA = a_mn ? K : M, colsA = a_mn ? M : K;
    const int rowsB = b_mn ? K : N, colsB = b_mn ? N : K;
    const uint32_t splitA = (uint32_t)((rowsA * a_sw + 1023) & ~1023), splitB = (uint32_t)((rowsB * b_sw + 1023) & ~1023);
    const uint32_t sB = sA + 3 * splitA;
    for (uint32_t i = tid; i < (3 * splitA + 3 * splitB) / 4; i += 128)
        reinterpret_cast<uint32_t*>(smem_raw + pad)[i] = 0u;
    __syncthreads();
    for (int i = tid; i < rowsA * colsA; i += 128) {
        const int r = i / colsA, c = i % colsA;
        const float v = a_mn ? A[(size_t)c * K + r] : A[(size_t)r * K + c];
        store1_x3(sA, splitA, a_sw == 128 ? off128(r, c) : off32(r, c), v);
    }
    for (int i = tid; i < rowsB * colsB; i += 128) {
        const int r = i / colsB, c = i % colsB;
        const float v = b_ones ? 1.0f : (b_mn ? B[(size_t)c * K + r] : B[(size_t)r * K + c]);
        store1_x3(sB, splitB, b_sw == 128 ? off128(r, c) : off32(r, c), v);
    }
    fence_async_smem();
    __syncthreads();
    const Acc acc = acc_cta(scratch, (uint32_t)N);
    const uint64_t a0 = a_sw == 128 ? desc128(sA) : desc32(sA), b0 = b_sw == 128 ? desc128(sB) : desc32(sB);
    gemm_x3(acc, 0u, a0, splitA, a_mn ? 16u * (uint32_t)a_sw : 32u, b0, b_ones ? 0u : splitB,
            b_mn ? 16u * (uint32_t)b_sw : 32u, idesc_bf16(M, N, a_mn, b_mn), K / 16, false);
    __threadfence_block();
    __syncthreads();
    for (int c0 = 0; c0 < N; c0 += 8) {
        float v[8];
        acc_ld8(acc, ((uint32_t)(tid & ~31) << 16) + (uint32_t)c0, v);
        for (int j = 0; j < 8; ++j) out[(size_t)tid * N + c0 + j] = v[j];
    }
}

}  // namespace osb

extern "C" int osb_x3_selftest(const float* A, const float* B, int M, int N, int K, int a_mn, int b_mn, int a_sw,
                               int b_sw, int b_ones, float* out, void* stream) {
    OSB_CHECK_ARG(A && B && out, "null pointer");
    OSB_CHECK_ARG((M == 64 || M == 128) && (N == 16 || N == 64) && K % 16 == 0 && K >= 16 && K <= 128, "bad shape");
    OSB_CHECK_ARG((a_sw == 128 || a_sw == 32) && (b_sw == 128 || b_sw == 32), "swizzle must be 128 or 32");
    OSB_CHECK_ARG((a_mn ? M : K) <= (a_sw == 128 ? 64 : 16) && (b_mn ? N : K) <= (b_sw == 128 ? 64 : 16), "tile wider than one swizzle atom");
    OSB_CHECK_ARG(!(a_mn && M == 128), "an MN-major A has 64 rows");
    float* scratch = osb::acc_scratch(osb::ACC_SELFTEST, (size_t)128 * N * sizeof(float));
    if (!scratch) return OSB_ERR_CUDA;
    const size_t smem = 1024 + 3 * 16384 + 3 * 16384;
    OSB_CUDA(cudaFuncSetAttribute(osb::x3_selftest_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    osb::x3_selftest_kernel<<<1, 128, smem, (cudaStream_t)stream>>>(A, B, M, N, K, a_mn, b_mn, a_sw, b_sw, b_ones, scratch, out);
    OSB_LAUNCH_CHECK();
    return OSB_OK;
}
