// Self-test of the split-bf16 tensor-core building blocks of csrc/x3.cuh: pins on real hardware the K-major /
// MN-major views of one SW128 or SW32 bf16 tile, the 6-product compensation and its accuracy
// (tests/test_x3_gpu.py), and the row-half products of the update kernel against the column-half phases they replace
// (tests/test_update_rowhalf_gpu.py).
#include "common.cuh"
#include "x3.cuh"

namespace osb {

// The GEMM shapes the kernels issue (gemm_x3 takes its shape as template arguments).
struct X3TestShape { int M, N, K, a_mn, b_mn, b_ones; };
constexpr X3TestShape X3_TEST_SHAPES[] = {
    {128, 64, 64, 0, 0, 0}, {128, 16, 64, 0, 0, 0}, {128, 64, 16, 0, 1, 0}, {128, 64, 64, 0, 1, 0},
    {64, 64, 128, 1, 1, 0}, {64, 16, 128, 1, 1, 0}, {64, 16, 128, 1, 1, 1}, {64, 64, 64, 0, 0, 0},
};
constexpr int X3_NSHAPES = sizeof(X3_TEST_SHAPES) / sizeof(X3_TEST_SHAPES[0]);

// A: row-major fp32 [M][K], B: row-major fp32 [N][K].  out[128][N]: dump of accumulator lanes 0..127.
// a_mn / b_mn: operand consumed MN-major (tile rows = K index) instead of K-major (tile rows = M/N index).
// a_sw / b_sw: 128 (tile rows of 64 bf16) or 32 (tile rows of 16 bf16).  b_ones: B is the all-ones tile
// (exact in bf16: three MMAs per k-step).
// Stages A (rowsA x colsA) and B (rowsB x colsB) as bf16x3 tiles behind the 1024-byte-aligned base of the dynamic shared
// memory; returns through sA / splitA / sB / splitB where they lie.  All 128 threads; ends in a block barrier.
__device__ __forceinline__ void selftest_stage(uint8_t* smem_raw, const float* __restrict__ A, const float* __restrict__ B,
                                               int M, int N, int K, int a_mn, int b_mn, int b_ones, int a_sw, int b_sw,
                                               uint32_t& sA, uint32_t& splitA, uint32_t& sB, uint32_t& splitB) {
    using namespace x3;
    const uint32_t pad = (1024u - (smem_u32(smem_raw) & 1023u)) & 1023u;
    sA = smem_u32(smem_raw) + pad;
    const int tid = threadIdx.x;
    const int rowsA = a_mn ? K : M, colsA = a_mn ? M : K;
    const int rowsB = b_mn ? K : N, colsB = b_mn ? N : K;
    splitA = (uint32_t)((rowsA * a_sw + 1023) & ~1023);
    splitB = (uint32_t)((rowsB * b_sw + 1023) & ~1023);
    sB = sA + 3 * splitA;
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
}

template <int S>
__global__ void __launch_bounds__(128, 1) x3_selftest_kernel(const float* __restrict__ A, const float* __restrict__ B,
                                                             int a_sw, int b_sw, float* __restrict__ scratch,
                                                             float* __restrict__ out) {
    using namespace x3;
    constexpr X3TestShape sh = X3_TEST_SHAPES[S];
    constexpr int M = sh.M, N = sh.N, K = sh.K, a_mn = sh.a_mn, b_mn = sh.b_mn, b_ones = sh.b_ones;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const int tid = threadIdx.x;
    uint32_t sA, splitA, sB, splitB;
    selftest_stage(smem_raw, A, B, M, N, K, a_mn, b_mn, b_ones, a_sw, b_sw, sA, splitA, sB, splitB);
    const Acc acc = acc_cta(scratch, (uint32_t)N);
    const uint64_t a0 = a_sw == 128 ? desc128(sA) : desc32(sA), b0 = b_sw == 128 ? desc128(sB) : desc32(sB);
    gemm_x3<M, N, K / 16, a_mn, b_mn, b_ones != 0>(acc, 0u, a0, splitA, a_mn ? 16u * (uint32_t)a_sw : 32u, b0, splitB,
                                                   b_mn ? 16u * (uint32_t)b_sw : 32u, false);
    __threadfence_block();
    __syncthreads();
    for (int c0 = 0; c0 < N; c0 += 8) {
        float v[8];
        acc_ld8(acc, ((uint32_t)(tid & ~31) << 16) + (uint32_t)c0, v);
        for (int j = 0; j < 8; ++j) out[(size_t)tid * N + c0 + j] = v[j];
    }
}

// The row-half products of the update kernel: A [128][K] K-major, B [N][K] K-major or MN-major; K = 64 as two chains of
// two k-steps whose sum is stored, K = 16 as one chain.
struct X3RowsShape { int N, K, b_mn; };
constexpr X3RowsShape X3_ROWS_SHAPES[] = {{64, 64, 0}, {64, 64, 1}, {16, 64, 0}, {64, 16, 1}};
constexpr int X3_NROWS_SHAPES = sizeof(X3_ROWS_SHAPES) / sizeof(X3_ROWS_SHAPES[0]);

// out[128][N]: the product issued as gemm_x3_rows on rows 0-63 and on rows 64-127; out_phases[128][N]: the same product
// issued as gemm_x3<128, ...>, for K = 64 in two column-half phases of which the second adds to the image.
template <int S>
__global__ void __launch_bounds__(128, 1) x3_rows_selftest_kernel(const float* __restrict__ A, const float* __restrict__ B,
                                                                  int a_sw, int b_sw, float* __restrict__ scratch,
                                                                  float* __restrict__ out, float* __restrict__ out_phases) {
    using namespace x3;
    constexpr X3RowsShape sh = X3_ROWS_SHAPES[S];
    constexpr int N = sh.N, K = sh.K, b_mn = sh.b_mn, NC = K == 16 ? 1 : 2, NK = K / 16 / NC;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const int tid = threadIdx.x;
    uint32_t sA, splitA, sB, splitB;
    selftest_stage(smem_raw, A, B, 128, N, K, 0, b_mn, 0, a_sw, b_sw, sA, splitA, sB, splitB);
    const Acc acc = acc_cta(scratch, 2u * N);
    const uint64_t a0 = a_sw == 128 ? desc128(sA) : desc32(sA), b0 = b_sw == 128 ? desc128(sB) : desc32(sB);
    const uint32_t bkstep = b_mn ? 16u * (uint32_t)b_sw : 32u;
    for (int r = 0; r < 2; ++r) gemm_x3_rows<N, NK, NC, b_mn>(acc, 0u, r, a0, splitA, 32u, b0, splitB, bkstep);
    for (int ph = 0; ph < NC; ++ph)
        gemm_x3<128, N, NK, 0, b_mn>(acc, (uint32_t)N, desc_add(a0, (uint32_t)ph * NK * 32u), splitA, 32u,
                                     desc_add(b0, (uint32_t)ph * NK * bkstep), splitB, bkstep, ph > 0);
    __threadfence_block();
    __syncthreads();
    for (int c0 = 0; c0 < 2 * N; c0 += 8) {
        float v[8];
        acc_ld8(acc, ((uint32_t)(tid & ~31) << 16) + (uint32_t)c0, v);
        float* dst = c0 < N ? out + (size_t)tid * N + c0 : out_phases + (size_t)tid * N + (c0 - N);
        for (int j = 0; j < 8; ++j) dst[j] = v[j];
    }
}

}  // namespace osb

extern "C" int osb_x3_selftest(const float* A, const float* B, int M, int N, int K, int a_mn, int b_mn, int a_sw,
                               int b_sw, int b_ones, float* out, void* stream) {
    OSB_CHECK_ARG(A && B && out, "null pointer");
    int shape = -1;
    for (int i = 0; i < osb::X3_NSHAPES; ++i) {
        const osb::X3TestShape& t = osb::X3_TEST_SHAPES[i];
        if (t.M == M && t.N == N && t.K == K && t.a_mn == a_mn && t.b_mn == b_mn && t.b_ones == b_ones) shape = i;
    }
    OSB_CHECK_ARG(shape >= 0, "not a GEMM shape of the kernels");
    OSB_CHECK_ARG((a_sw == 128 || a_sw == 32) && (b_sw == 128 || b_sw == 32), "swizzle must be 128 or 32");
    OSB_CHECK_ARG((a_mn ? M : K) <= (a_sw == 128 ? 64 : 16) && (b_mn ? N : K) <= (b_sw == 128 ? 64 : 16), "tile wider than one swizzle atom");
    using Kernel = void (*)(const float*, const float*, int, int, float*, float*);
    const Kernel kernels[osb::X3_NSHAPES] = {osb::x3_selftest_kernel<0>, osb::x3_selftest_kernel<1>, osb::x3_selftest_kernel<2>,
                                             osb::x3_selftest_kernel<3>, osb::x3_selftest_kernel<4>, osb::x3_selftest_kernel<5>,
                                             osb::x3_selftest_kernel<6>, osb::x3_selftest_kernel<7>};
    float* scratch = osb::acc_scratch(osb::ACC_SELFTEST, (size_t)128 * N * sizeof(float));
    if (!scratch) return OSB_ERR_CUDA;
    const size_t smem = 1024 + 3 * 16384 + 3 * 16384;
    OSB_CUDA(cudaFuncSetAttribute(kernels[shape], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernels[shape]<<<1, 128, smem, (cudaStream_t)stream>>>(A, B, a_sw, b_sw, scratch, out);
    OSB_LAUNCH_CHECK();
    return OSB_OK;
}

extern "C" int osb_x3_rows_selftest(const float* A, const float* B, int N, int K, int b_mn, int a_sw, int b_sw, float* out,
                                    float* out_phases, void* stream) {
    OSB_CHECK_ARG(A && B && out && out_phases, "null pointer");
    int shape = -1;
    for (int i = 0; i < osb::X3_NROWS_SHAPES; ++i) {
        const osb::X3RowsShape& t = osb::X3_ROWS_SHAPES[i];
        if (t.N == N && t.K == K && t.b_mn == b_mn) shape = i;
    }
    OSB_CHECK_ARG(shape >= 0, "not a row-half GEMM shape of the update kernel");
    OSB_CHECK_ARG((a_sw == 128 || a_sw == 32) && (b_sw == 128 || b_sw == 32), "swizzle must be 128 or 32");
    OSB_CHECK_ARG(K <= (a_sw == 128 ? 64 : 16) && (b_mn ? N : K) <= (b_sw == 128 ? 64 : 16), "tile wider than one swizzle atom");
    using Kernel = void (*)(const float*, const float*, int, int, float*, float*, float*);
    const Kernel kernels[osb::X3_NROWS_SHAPES] = {osb::x3_rows_selftest_kernel<0>, osb::x3_rows_selftest_kernel<1>,
                                                  osb::x3_rows_selftest_kernel<2>, osb::x3_rows_selftest_kernel<3>};
    float* scratch = osb::acc_scratch(osb::ACC_SELFTEST, (size_t)128 * 2 * N * sizeof(float));
    if (!scratch) return OSB_ERR_CUDA;
    const size_t smem = 1024 + 3 * 16384 + 3 * 16384;
    OSB_CUDA(cudaFuncSetAttribute(kernels[shape], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernels[shape]<<<1, 128, smem, (cudaStream_t)stream>>>(A, B, a_sw, b_sw, scratch, out, out_phases);
    OSB_LAUNCH_CHECK();
    return OSB_OK;
}
