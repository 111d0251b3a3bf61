// wgmma / mbarrier helpers (inline PTX, sm_90a) for the tensor-core MLP tiles.
//
// Operand tiles live in shared memory as fp32 in the canonical 128-byte-swizzled layout
// (rows of 128 B = 32 floats, 8-row groups of 1024 B, 16-byte chunks XOR-ed with row % 8), consumed K-major
// (rows = M/N index, the 32 floats of a row run along K); wgmma reads tf32 operands from shared memory
// K-major only, which is why the kernels produce transposed activations with role-swapped MMAs.
// kind tf32 reads the fp32 words directly (10-bit mantissa used).
//
// Accumulators.  A GEMM D[M][N] (M = 128 or 64) is issued by one warpgroup (128 threads) as m64 wgmma
// instructions with fp32 register accumulators; when they complete, every thread writes its fragment to the
// CTA's accumulator image in global memory (L2 resident): fp32 [128 lanes][pitch columns], row m of an
// M = 128 product in lane m, row m of an M = 64 product in lane 32 (m / 16) + m % 16.  An accumulator address
// `taddr` is (lane << 16) | column.  Epilogue threads read the rows they own with vector loads (acc_ld8 / acc_ld16 / acc_ld32);
// a GEMM with accumulate = true adds its product to what the image holds.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace osb {
namespace umma {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// byte offset of element (r, c) inside a tile of R rows x C floats (C % 32 == 0) stored as C/32 atoms
// of [R][32] floats, each atom 128B-swizzled.  Tile base must be 1024-byte aligned.
__device__ __forceinline__ uint32_t sw128_offset(int r, int c, int R) {
    const int atom = c >> 5, cc = c & 31;
    return (uint32_t)(atom * R * 128 + r * 128 + ((((cc >> 2) ^ (r & 7)) << 4) | ((cc & 3) << 2)));
}

// Shared-memory matrix descriptor, 128B swizzle (wgmma descriptor: start address [0,14), leading byte
// offset [16,30), stride byte offset [32,46), base offset [49,52) = 0, layout type [62,64): 1 = SW128).
__device__ __forceinline__ uint64_t desc_sw128(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (uint64_t)((saddr >> 4) & 0x3FFFu) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) |
           ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32) | (1ull << 62);
}
// K-major operand: 8-row groups are 1024 B apart; LBO is unused for swizzled K-major (set to 16 B).
__device__ __forceinline__ uint64_t desc_kmajor(uint32_t saddr) { return desc_sw128(saddr, 16, 1024); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_init_fence() {
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}
// the same on 32-bit shared addresses, for barriers placed in dynamic shared memory by offset
__device__ __forceinline__ void mbar_init_a(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(bar) : "memory");
}
// one arrival that also makes the current phase wait for `bytes` of asynchronous (TMA) copies to land
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait_a(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}\n"
            : "=r"(ok)
            : "r"(bar), "r"(parity)
            : "memory");
    } while (!ok);
}

// generic-proxy smem writes -> visible to the async proxy (tensor core operand reads)
__device__ __forceinline__ void fence_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
}
// ---- wgmma (one warpgroup) --------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_tf32_n64(float (&d)[32], uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(scale_d) : "memory");
}
__device__ __forceinline__ void wgmma_tf32_n16(float (&d)[8], uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, "
        "%8, %9, p, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a), "l"(b), "r"(scale_d) : "memory");
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_n64(float (&d)[32], uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1, %35, %36;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB) : "memory");
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_n16(float (&d)[8], uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, "
        "%8, %9, p, 1, 1, %11, %12;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB) : "memory");
}

// The same with A from registers: the m64k16 fragment of the thread, a[0] / a[1] = rows l / 4 and l / 4 + 8 of the
// warp's 16 rows at k = 2 (l % 4) + {0, 1}, a[2] / a[3] the same at k + 8 (bf16x2 words, lower k in the low half).
template <int TB>
__device__ __forceinline__ void wgmma_bf16_n64_ra(float (&d)[32], const uint32_t (&a)[4], uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %38, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "{%32, %33, %34, %35}, %36, p, 1, 1, %37;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "n"(TB), "r"(scale_d) : "memory");
}
template <int TB>
__device__ __forceinline__ void wgmma_bf16_n16_ra(float (&d)[8], const uint32_t (&a)[4], uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %14, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, "
        "{%8, %9, %10, %11}, %12, p, 1, 1, %13;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "n"(TB), "r"(scale_d) : "memory");
}

// Warpgroup of the calling thread, taken from lane 0 so that ptxas can prove a branch on it uniform over the warp.
// A wgmma-issuing branch must test this value: on a test of threadIdx.x itself ptxas assumes a divergent path and
// waits on every wgmma before issuing the next (C7520).
__device__ __forceinline__ int warpgroup_index() { return __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0); }

// Per-warpgroup register budget (all 128 threads of the warpgroup): the calling warpgroup's registers per thread become
// N (a multiple of 8).  `inc` waits until the CTA's pool, the launch allocation, has N free per thread, so the warpgroups
// that give registers up must `dec` first or concurrently.
template <int N>
__device__ __forceinline__ void wg_regs_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void wg_regs_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(N)); }

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
// wait until at most N committed groups of this warpgroup are pending
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory"); }
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// ---- accumulator image ------------------------------------------------------------------------------------
struct Acc {
    float* p;          // this CTA's [128][pitch] fp32 image
    uint32_t pitch;    // columns per lane
};
// the CTA's slice of a scratch buffer holding one [128][pitch] image per CTA of the grid
__device__ __forceinline__ Acc acc_cta(float* scratch, uint32_t pitch) {
    const size_t cta = (size_t)blockIdx.y * gridDim.x + blockIdx.x;
    return Acc{scratch + cta * 128 * pitch, pitch};
}

// Where row rr (0 or 1) of the m64 fragment of this warpgroup thread starts in the image: rows 64 half .. 64 half + 63
// of an M-row product, columns from the accumulator address taddr.  Element (rr, j, e) lies at [8 j + e].
__device__ __forceinline__ float* frag_row(const Acc& acc, uint32_t taddr, int M, int half, int rr) {
    const int t = threadIdx.x & 127, w = t >> 5, l = t & 31;
    const int m = 64 * half + 16 * w + (l >> 2) + 8 * rr;
    const uint32_t lane = (taddr >> 16) + (uint32_t)(M == 128 ? m : 32 * (m >> 4) + (m & 15));
    return acc.p + (size_t)lane * acc.pitch + (taddr & 0xFFFFu) + 2u * (uint32_t)(l & 3);
}

// One row of the fragment (rr = 0 or 1, see frag_row), NB float2 of it from column pair j0 on: the image values under
// them, read as independent loads that are all in flight together; the fragment registers d written there; and d + o
// written there, one fp32 add per element.  A product that adds to the image reads a batch before it adds and stores:
// a load, add, store chain per element would put one image round trip after another.
template <int NB>
__device__ __forceinline__ void row_load(const float* row, int j0, float2 (&o)[NB]) {
#pragma unroll
    for (int j = 0; j < NB; ++j) o[j] = *reinterpret_cast<const float2*>(row + 8 * (j0 + j));
}
template <int ND, int NB>
__device__ __forceinline__ void row_add_store(float* row, int rr, const float (&d)[ND], int j0, const float2 (&o)[NB]) {
#pragma unroll
    for (int j = 0; j < NB; ++j) {
        const int i = 4 * (j0 + j) + 2 * rr;
        *reinterpret_cast<float2*>(row + 8 * (j0 + j)) = make_float2(d[i] + o[j].x, d[i + 1] + o[j].y);
    }
}

// The m64 x (8 NJ) fragment of this warpgroup thread: the image values under it (both rows in flight), the fragment
// written, and the fragment written as d + o.
template <int NJ>
__device__ __forceinline__ void frag_load(const Acc& acc, uint32_t taddr, int M, int half, float2 (&o)[2][NJ]) {
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) row_load(frag_row(acc, taddr, M, half, rr), 0, o[rr]);
}
template <int NJ>
__device__ __forceinline__ void frag_store(const Acc& acc, uint32_t taddr, int M, int half, const float (&d)[4 * NJ]) {
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
        float* row = frag_row(acc, taddr, M, half, rr);
#pragma unroll
        for (int j = 0; j < NJ; ++j)
            *reinterpret_cast<float2*>(row + 8 * j) = make_float2(d[4 * j + 2 * rr], d[4 * j + 2 * rr + 1]);
    }
}
template <int NJ>
__device__ __forceinline__ void frag_add_store(const Acc& acc, uint32_t taddr, int M, int half, const float (&d)[4 * NJ],
                                               const float2 (&o)[2][NJ]) {
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) row_add_store(frag_row(acc, taddr, M, half, rr), rr, d, 0, o[rr]);
}

// The issuing warpgroup's image writes -> visible to the CTA, then one arrival on the mbarrier (count 1).
// Called by all 128 threads of the warpgroup that issued the GEMMs (named barrier 3).
__device__ __forceinline__ void mma_commit(uint64_t* bar) {
    __threadfence_block();
    asm volatile("bar.sync 3, 128;\n" ::: "memory");
    if ((threadIdx.x & 127) == 0)
        asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}

// vector loads of NV consecutive columns: like a 32-lane tensor-memory load, taddr names the warp's first lane and
// thread i of the warp reads lane (taddr >> 16) + i
template <int NV>
__device__ __forceinline__ void acc_ld(const Acc& acc, uint32_t taddr, float* v) {
    const uint32_t lane = (taddr >> 16) + (threadIdx.x & 31u);
    const float4* s = reinterpret_cast<const float4*>(acc.p + (size_t)lane * acc.pitch + (taddr & 0xFFFFu));
#pragma unroll
    for (int i = 0; i < NV / 4; ++i) {
        const float4 x = s[i];
        v[4 * i] = x.x; v[4 * i + 1] = x.y; v[4 * i + 2] = x.z; v[4 * i + 3] = x.w;
    }
}
__device__ __forceinline__ void acc_ld32(const Acc& acc, uint32_t taddr, float (&v)[32]) { acc_ld<32>(acc, taddr, v); }
__device__ __forceinline__ void acc_ld16(const Acc& acc, uint32_t taddr, float (&v)[16]) { acc_ld<16>(acc, taddr, v); }

// D[acc] (+)= A * B^T, both K-major SW128 tf32 tiles with RA / RB rows (M = 64 or 128, N = 16 or a multiple
// of 64, K % 8 == 0); called by all 128 threads of one warpgroup.  With accumulate, the image values under a
// fragment are read while its MMAs run.
__device__ __forceinline__ void tc_gemm(const Acc& acc, uint32_t d_addr, uint32_t a_base, int RA, uint32_t b_base,
                                        int RB, int M, int N, int K, bool accumulate) {
#pragma unroll 1
    for (int half = 0; half < M / 64; ++half) {
        const uint32_t a_half = a_base + (uint32_t)half * 64u * 128u;
        if (N == 16) {
            float d[8] = {};
            float2 old[2][2];
            wg_fence();
            acc_fence(d);
#pragma unroll 1
            for (int ks = 0; ks < K / 8; ++ks) {
                const uint32_t offA = (uint32_t)((ks >> 2) * RA * 128 + (ks & 3) * 32);
                const uint32_t offB = (uint32_t)((ks >> 2) * RB * 128 + (ks & 3) * 32);
                wgmma_tf32_n16(d, desc_kmajor(a_half + offA), desc_kmajor(b_base + offB), ks > 0 ? 1u : 0u);
            }
            wg_commit();
            if (accumulate) frag_load<2>(acc, d_addr, M, half, old);
            wg_wait<0>();
            acc_fence(d);
            if (accumulate) frag_add_store<2>(acc, d_addr, M, half, d, old);
            else frag_store<2>(acc, d_addr, M, half, d);
        } else {
#pragma unroll 1
            for (int nc = 0; nc < N / 64; ++nc) {
                float d[32] = {};
                float2 old[2][8];
                wg_fence();
                acc_fence(d);
#pragma unroll 1
                for (int ks = 0; ks < K / 8; ++ks) {
                    const uint32_t offA = (uint32_t)((ks >> 2) * RA * 128 + (ks & 3) * 32);
                    const uint32_t offB = (uint32_t)((ks >> 2) * RB * 128 + (ks & 3) * 32 + nc * 64 * 128);
                    wgmma_tf32_n64(d, desc_kmajor(a_half + offA), desc_kmajor(b_base + offB), ks > 0 ? 1u : 0u);
                }
                wg_commit();
                if (accumulate) frag_load<8>(acc, d_addr + (uint32_t)(64 * nc), M, half, old);
                wg_wait<0>();
                acc_fence(d);
                if (accumulate) frag_add_store<8>(acc, d_addr + (uint32_t)(64 * nc), M, half, d, old);
                else frag_store<8>(acc, d_addr + (uint32_t)(64 * nc), M, half, d);
            }
        }
    }
}

// round-to-nearest TF32 (the MMA would otherwise truncate the low 13 mantissa bits: biased)
__device__ __forceinline__ float tf32r(float x) {
    uint32_t u;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
    return __uint_as_float(u);
}
__device__ __forceinline__ float tanh_fast(float x) {
    float y;
    asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
struct TanhFast {
    __device__ __forceinline__ float operator()(float x) const { return tanh_fast(x); }
};
// explicit shared-window (32-bit address) accessors: keeps every tile access an LDS/STS
__device__ __forceinline__ float lds(uint32_t a) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ void sts(uint32_t a, float v) {
    asm volatile("st.shared.f32 [%0], %1;" ::"r"(a), "f"(v) : "memory");
}
__device__ __forceinline__ uint32_t tile_addr(uint32_t base, int r, int c, int R) {
    return base + sw128_offset(r, c, R);
}
// store / load 32 consecutive columns [c0, c0+32) (c0 % 32 == 0) of row r
__device__ __forceinline__ void store_row32(uint32_t base, int r, int c0, int R, const float (&v)[32]) {
    const uint32_t row = base + (uint32_t)((c0 >> 5) * R * 128 + r * 128);
#pragma unroll
    for (int i = 0; i < 8; ++i)
        asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(row + (uint32_t)((i ^ (r & 7)) << 4)),
                     "f"(tf32r(v[4 * i])), "f"(tf32r(v[4 * i + 1])), "f"(tf32r(v[4 * i + 2])), "f"(tf32r(v[4 * i + 3]))
                     : "memory");
}
__device__ __forceinline__ void load_row32(uint32_t base, int r, int c0, int R, float (&v)[32]) {
    const uint32_t row = base + (uint32_t)((c0 >> 5) * R * 128 + r * 128);
#pragma unroll
    for (int i = 0; i < 8; ++i)
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                     : "=f"(v[4 * i]), "=f"(v[4 * i + 1]), "=f"(v[4 * i + 2]), "=f"(v[4 * i + 3])
                     : "r"(row + (uint32_t)((i ^ (r & 7)) << 4)));
}


}  // namespace umma
}  // namespace osb
