// Split-bf16 ("bf16x3") tensor-core arithmetic: the parity-grade mode of the MLP tiles.
//
// Every fp32 operand x is stored as three bf16 tiles x0 + x1 + x2 == x (exactly: x0 = rn_bf16(x),
// x1 = rn_bf16(x - x0), x2 = x - x0 - x1 which has <= 8 significant bits).  A product A * B is issued as the
// six bf16 wgmmas  sum_{i+j<=2} A_i B_j  (the dropped terms are <= 2^-26 relative) with fp32 accumulation
// in registers, small terms first.  Every bf16 x bf16 product is exact in fp32, so the result carries fp32-level
// accuracy -- unlike tf32 wgmma (10-bit mantissa), this mode meets the reference's fp32 Linear layers
// (omnisafe/utils/model.py:L105-111) at the tolerance of the exact-FMA path.
//
// Unlike tf32, 16-bit operands have an MN-major view under the ordinary 128-byte swizzle, so ONE stored
// activation tile [sample][feature] serves the forward GEMM (K-major, contraction over features) and the
// weight-gradient GEMM (MN-major, contraction over samples): no transposed copies, no role-swapped MMAs.
//
// Tile formats (base 1024-byte aligned):
//   SW128: [R][64] bf16, row pitch 128 B, 16-byte chunk index XOR (row & 7)            (layout code 2)
//   SW32 : [R][16] bf16, row pitch  32 B, 16-byte chunk index XOR ((row >> 2) & 1)     (layout code 6)
// (the layout code sits at descriptor bits [61,64); the wgmma layout field is bits [62,64): 1 = SW128, 3 = SW32)
// An x3 tile is three such sub-tiles back to back (hi, mid, lo), `split` bytes apart.
#pragma once
#include "umma.cuh"

namespace osb {
namespace x3 {

using namespace umma;

// ---- descriptors ------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t desc_make(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t layout) {
    return (uint64_t)((saddr >> 4) & 0x3FFFu) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) |
           ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32) | ((uint64_t)layout << 61);
}
// SW128 tile: 8-row groups 1024 B apart, both as K-major (rows = M/N index) and MN-major (rows = K index,
// one 64-element atom along M/N, so the leading offset is never used).
constexpr int LBO_DEFAULT = 16;
__device__ __forceinline__ uint64_t desc128(uint32_t saddr) { return desc_make(saddr, LBO_DEFAULT, 1024, 2); }
// SW32 tile: 8-row groups 256 B apart.
__device__ __forceinline__ uint64_t desc32(uint32_t saddr) { return desc_make(saddr, LBO_DEFAULT, 256, 6); }
// descriptor + byte offset (start-address field only; all tiles live below 256 KB of shared memory)
__device__ __forceinline__ uint64_t desc_add(uint64_t d, uint32_t bytes) { return d + (uint64_t)(bytes >> 4); }

// GEMM shape word, bf16 x bf16 -> fp32: M (64 or 128), N, and which operands are read MN-major
__device__ __forceinline__ constexpr uint32_t idesc_bf16(int M, int N, int a_mn, int b_mn) {
    return ((uint32_t)a_mn << 15) | ((uint32_t)b_mn << 16) | ((uint32_t)(N >> 3) << 17) | ((uint32_t)(M >> 4) << 24);
}

// One m64 x N block over nk k-steps of 16, six split products per k-step (three when B is exact).
template <int TA, int TB, int NJ>
__device__ __forceinline__ void x3_block(float (&d)[4 * NJ], uint64_t a0, uint32_t asplit, uint32_t akstep, uint64_t b0,
                                         uint32_t bsplit, uint32_t bkstep, int nk) {
    wg_fence();
    acc_fence(d);
#pragma unroll 1
    for (int ks = 0; ks < nk; ++ks) {
        const uint64_t a = desc_add(a0, (uint32_t)ks * akstep), b = desc_add(b0, (uint32_t)ks * bkstep);
        const uint64_t a1 = desc_add(a, asplit), a2 = desc_add(a, 2 * asplit);
        const uint32_t s = ks > 0 ? 1u : 0u;
        if constexpr (NJ == 8) {
            if (bsplit == 0) {
                wgmma_bf16_n64<TA, TB>(d, a2, b, s);
                wgmma_bf16_n64<TA, TB>(d, a1, b, 1u);
                wgmma_bf16_n64<TA, TB>(d, a, b, 1u);
            } else {
                const uint64_t b1 = desc_add(b, bsplit), b2 = desc_add(b, 2 * bsplit);
                wgmma_bf16_n64<TA, TB>(d, a2, b, s);
                wgmma_bf16_n64<TA, TB>(d, a, b2, 1u);
                wgmma_bf16_n64<TA, TB>(d, a1, b1, 1u);
                wgmma_bf16_n64<TA, TB>(d, a1, b, 1u);
                wgmma_bf16_n64<TA, TB>(d, a, b1, 1u);
                wgmma_bf16_n64<TA, TB>(d, a, b, 1u);
            }
        } else {
            if (bsplit == 0) {
                wgmma_bf16_n16<TA, TB>(d, a2, b, s);
                wgmma_bf16_n16<TA, TB>(d, a1, b, 1u);
                wgmma_bf16_n16<TA, TB>(d, a, b, 1u);
            } else {
                const uint64_t b1 = desc_add(b, bsplit), b2 = desc_add(b, 2 * bsplit);
                wgmma_bf16_n16<TA, TB>(d, a2, b, s);
                wgmma_bf16_n16<TA, TB>(d, a, b2, 1u);
                wgmma_bf16_n16<TA, TB>(d, a1, b1, 1u);
                wgmma_bf16_n16<TA, TB>(d, a1, b, 1u);
                wgmma_bf16_n16<TA, TB>(d, a, b1, 1u);
                wgmma_bf16_n16<TA, TB>(d, a, b, 1u);
            }
        }
    }
    wg_commit_wait();
    acc_fence(d);
}

template <int TA, int TB>
__device__ __forceinline__ void gemm_x3_t(const Acc& acc, uint32_t d_addr, uint64_t a0, uint32_t asplit, uint32_t akstep,
                                          uint64_t b0, uint32_t bsplit, uint32_t bkstep, int M, int N, int nk,
                                          bool accumulate) {
    // rows 64..127 of a K-major A: 64 rows further down the tile (row pitch 128 B for SW128, 32 B for SW32)
    const uint32_t a_half_bytes = 64u * (((a0 >> 61) & 7u) == 2u ? 128u : 32u);
#pragma unroll 1
    for (int half = 0; half < M / 64; ++half) {
        const uint64_t ah = desc_add(a0, (uint32_t)half * a_half_bytes);
        if (N == 16) {
            float d[8] = {};
            x3_block<TA, TB, 2>(d, ah, asplit, akstep, b0, bsplit, bkstep, nk);
            frag_store<2>(acc, d_addr, M, half, d, accumulate);
        } else {
#pragma unroll 1
            for (int nc = 0; nc < N / 64; ++nc) {       // N > 64: K-major SW128 B, 64 rows per block
                float d[32] = {};
                x3_block<TA, TB, 8>(d, ah, asplit, akstep, desc_add(b0, (uint32_t)nc * 8192u), bsplit, bkstep, nk);
                frag_store<8>(acc, d_addr + (uint32_t)(64 * nc), M, half, d, accumulate);
            }
        }
    }
}

// D[acc] (+)= A * B over `nk` k-steps of 16, with the six split products (small terms first); called by all
// 128 threads of one warpgroup.
//   a0 / b0: descriptors of the hi sub-tiles at k-step 0; asplit / bsplit: bytes between sub-tiles;
//   akstep / bkstep: bytes per k-step (K-major: 32; MN-major: 16 rows * pitch); shape: idesc_bf16(M, N, a_mn, b_mn)
//   (an MN-major A has M = 64; N is 16 or a multiple of 64, and a multiple of 64 above 64 only for a K-major B).
//   bsplit == 0 marks an exactly representable B (e.g. the ones tile): only the three A terms are issued.
__device__ __forceinline__ void gemm_x3(const Acc& acc, uint32_t d_addr, uint64_t a0, uint32_t asplit, uint32_t akstep,
                                        uint64_t b0, uint32_t bsplit, uint32_t bkstep, uint32_t shape, int nk,
                                        bool accumulate) {
    const int M = (int)((shape >> 24) & 31u) << 4, N = (int)((shape >> 17) & 63u) << 3;
    switch ((shape >> 15) & 3u) {
        case 0: gemm_x3_t<0, 0>(acc, d_addr, a0, asplit, akstep, b0, bsplit, bkstep, M, N, nk, accumulate); break;
        case 1: gemm_x3_t<1, 0>(acc, d_addr, a0, asplit, akstep, b0, bsplit, bkstep, M, N, nk, accumulate); break;
        case 2: gemm_x3_t<0, 1>(acc, d_addr, a0, asplit, akstep, b0, bsplit, bkstep, M, N, nk, accumulate); break;
        default: gemm_x3_t<1, 1>(acc, d_addr, a0, asplit, akstep, b0, bsplit, bkstep, M, N, nk, accumulate); break;
    }
}

// ---- fp32 <-> three bf16 ----------------------------------------------------------------------------
// pack two floats into one bf16x2 word (lo half = a, hi half = b), round to nearest even
__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
    return r;
}
__device__ __forceinline__ float bf16lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf16hi(uint32_t w) { return __uint_as_float(w & 0xFFFF0000u); }
// (a, b) -> words w0, w1, w2 with a == lo(w0) + lo(w1) + lo(w2), b == hi(w0) + hi(w1) + hi(w2)
__device__ __forceinline__ void split2(float a, float b, uint32_t& w0, uint32_t& w1, uint32_t& w2) {
    w0 = pack_bf16x2(a, b);
    const float ra = a - bf16lo(w0), rb = b - bf16hi(w0);
    w1 = pack_bf16x2(ra, rb);
    w2 = pack_bf16x2(ra - bf16lo(w1), rb - bf16hi(w1));
}

// byte offset of element (r, c) of a SW128 / SW32 sub-tile
__device__ __forceinline__ uint32_t off128(int r, int c) {
    return (uint32_t)(r * 128 + ((((c >> 3) ^ (r & 7)) << 4) | ((c & 7) << 1)));
}
__device__ __forceinline__ uint32_t off32(int r, int c) {
    return (uint32_t)(r * 32 + ((((c >> 3) ^ ((r >> 2) & 1)) << 4) | ((c & 7) << 1)));
}
__device__ __forceinline__ void sts128(uint32_t a, uint32_t x, uint32_t y, uint32_t z, uint32_t w) {
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}
__device__ __forceinline__ void lds128(uint32_t a, uint32_t& x, uint32_t& y, uint32_t& z, uint32_t& w) {
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(x), "=r"(y), "=r"(z), "=r"(w) : "r"(a));
}
__device__ __forceinline__ void sts16(uint32_t a, uint16_t v) {
    asm volatile("st.shared.u16 [%0], %1;" ::"r"(a), "h"(v) : "memory");
}

// store 16 consecutive columns [c0, c0 + 16) (c0 % 16 == 0) of row r of a SW128 x3 tile
__device__ __forceinline__ void store16_x3(uint32_t base, uint32_t split, int r, int c0, const float (&v)[16]) {
    uint32_t w0[8], w1[8], w2[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) split2(v[2 * i], v[2 * i + 1], w0[i], w1[i], w2[i]);
    const uint32_t row = base + (uint32_t)(r * 128);
    const int ch = c0 >> 3;
    const uint32_t o0 = row + (uint32_t)(((ch) ^ (r & 7)) << 4), o1 = row + (uint32_t)(((ch + 1) ^ (r & 7)) << 4);
    sts128(o0, w0[0], w0[1], w0[2], w0[3]); sts128(o1, w0[4], w0[5], w0[6], w0[7]);
    sts128(o0 + split, w1[0], w1[1], w1[2], w1[3]); sts128(o1 + split, w1[4], w1[5], w1[6], w1[7]);
    sts128(o0 + 2 * split, w2[0], w2[1], w2[2], w2[3]); sts128(o1 + 2 * split, w2[4], w2[5], w2[6], w2[7]);
}
// load them back as fp32 (exact reconstruction)
__device__ __forceinline__ void load16_x3(uint32_t base, uint32_t split, int r, int c0, float (&v)[16]) {
    const uint32_t row = base + (uint32_t)(r * 128);
    const int ch = c0 >> 3;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        const uint32_t o = row + (uint32_t)(((ch + half) ^ (r & 7)) << 4);
        uint32_t a[4], b[4], c[4];
        lds128(o, a[0], a[1], a[2], a[3]);
        lds128(o + split, b[0], b[1], b[2], b[3]);
        lds128(o + 2 * split, c[0], c[1], c[2], c[3]);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            v[8 * half + 2 * i] = (bf16lo(a[i]) + bf16lo(b[i])) + bf16lo(c[i]);
            v[8 * half + 2 * i + 1] = (bf16hi(a[i]) + bf16hi(b[i])) + bf16hi(c[i]);
        }
    }
}
// store the 16 columns of row r of a SW32 x3 tile ([R][16])
__device__ __forceinline__ void store16_x3_sw32(uint32_t base, uint32_t split, int r, const float (&v)[16]) {
    uint32_t w0[8], w1[8], w2[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) split2(v[2 * i], v[2 * i + 1], w0[i], w1[i], w2[i]);
    const uint32_t row = base + (uint32_t)(r * 32);
    const int x = (r >> 2) & 1;
    const uint32_t o0 = row + (uint32_t)(x << 4), o1 = row + (uint32_t)((x ^ 1) << 4);
    sts128(o0, w0[0], w0[1], w0[2], w0[3]); sts128(o1, w0[4], w0[5], w0[6], w0[7]);
    sts128(o0 + split, w1[0], w1[1], w1[2], w1[3]); sts128(o1 + split, w1[4], w1[5], w1[6], w1[7]);
    sts128(o0 + 2 * split, w2[0], w2[1], w2[2], w2[3]); sts128(o1 + 2 * split, w2[4], w2[5], w2[6], w2[7]);
}

// single element stores (weight staging)
__device__ __forceinline__ void store1_x3(uint32_t base, uint32_t split, uint32_t off, float x) {
    uint32_t w0, w1, w2;
    split2(x, 0.f, w0, w1, w2);
    sts16(base + off, (uint16_t)w0); sts16(base + split + off, (uint16_t)w1); sts16(base + 2 * split + off, (uint16_t)w2);
}

// ---- mbarrier / issue helpers on 32-bit shared addresses ----------------------------------------------
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(bar) : "memory");
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
// mma_commit on a 32-bit shared address
__device__ __forceinline__ void mma_commit_a(uint32_t bar) {
    __threadfence_block();
    asm volatile("bar.sync 3, 128;\n" ::: "memory");
    if ((threadIdx.x & 127) == 0) mbar_arrive(bar);
}
__device__ __forceinline__ void acc_ld8(const Acc& acc, uint32_t taddr, float (&v)[8]) { acc_ld<8>(acc, taddr, v); }
// 8 consecutive columns [c0, c0 + 8) (c0 % 8 == 0) of row r of a SW128 x3 tile
__device__ __forceinline__ void store8_x3(uint32_t base, uint32_t split, int r, int c0, const float (&v)[8]) {
    uint32_t w0[4], w1[4], w2[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) split2(v[2 * i], v[2 * i + 1], w0[i], w1[i], w2[i]);
    const uint32_t o = base + (uint32_t)(r * 128 + (((c0 >> 3) ^ (r & 7)) << 4));
    sts128(o, w0[0], w0[1], w0[2], w0[3]);
    sts128(o + split, w1[0], w1[1], w1[2], w1[3]);
    sts128(o + 2 * split, w2[0], w2[1], w2[2], w2[3]);
}
__device__ __forceinline__ void load8_x3(uint32_t base, uint32_t split, int r, int c0, float (&v)[8]) {
    const uint32_t o = base + (uint32_t)(r * 128 + (((c0 >> 3) ^ (r & 7)) << 4));
    uint32_t a[4], b[4], c[4];
    lds128(o, a[0], a[1], a[2], a[3]);
    lds128(o + split, b[0], b[1], b[2], b[3]);
    lds128(o + 2 * split, c[0], c[1], c[2], c[3]);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        v[2 * i] = (bf16lo(a[i]) + bf16lo(b[i])) + bf16lo(c[i]);
        v[2 * i + 1] = (bf16hi(a[i]) + bf16hi(b[i])) + bf16hi(c[i]);
    }
}


// tanh with fp32-level accuracy (the MUFU tanh.approx has 2^-11 relative error):
//   |x| <  1: x + x^3 p(x^2), p = degree-6 minimax fit (relative error of the result 5e-9 before rounding);
//   otherwise 1 - 2 / (exp(2|x|) + 1) with ex2.approx / rcp.approx.  Max relative error 1.2e-7 (2 ulp).
__device__ __forceinline__ float tanh_acc(float x) {
    const float ax = fabsf(x);
    const float x2 = x * x;
    float p = fmaf(x2, -3.497081634e-04f, 2.272918122e-03f);
    p = fmaf(p, x2, -7.910109125e-03f);
    p = fmaf(p, x2, 2.146438509e-02f);
    p = fmaf(p, x2, -5.387288332e-02f);
    p = fmaf(p, x2, 1.333224624e-01f);
    p = fmaf(p, x2, -3.333328962e-01f);
    const float small = fmaf(p * x2, x, x);
    float e;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(ax * 2.8853900817779268f));   // exp(2|x|)
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(e + 1.0f));
    const float big = copysignf(fmaf(-2.0f, r, 1.0f), x);
    return ax < 1.0f ? small : big;
}

}  // namespace x3
}  // namespace osb
