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

// d, hidden from loop-invariant code motion (see gemm_x3)
__device__ __forceinline__ uint64_t desc_fresh(uint64_t d) {
    asm volatile("" : "+l"(d));
    return d;
}

// One m64 x (8 NJ) block over NK k-steps of 16, six split products per k-step (three when B is exact), small terms
// first: one fence, an unbroken run of wgmmas and one commit.  The caller waits on the group.
template <int TA, int TB, int NJ, int NK, bool B_EXACT>
__device__ __forceinline__ void x3_block(float (&d)[4 * NJ], uint64_t a0, uint32_t asplit, uint32_t akstep, uint64_t b0,
                                         uint32_t bsplit, uint32_t bkstep) {
    auto mma = [&](uint64_t a, uint64_t b, uint32_t s) {
        if constexpr (NJ == 8) wgmma_bf16_n64<TA, TB>(d, a, b, s);
        else wgmma_bf16_n16<TA, TB>(d, a, b, s);
    };
    wg_fence();
    acc_fence(d);
#pragma unroll
    for (int ks = 0; ks < NK; ++ks) {
        const uint64_t a = desc_add(a0, (uint32_t)ks * akstep), b = desc_add(b0, (uint32_t)ks * bkstep);
        const uint64_t a1 = desc_add(a, asplit), a2 = desc_add(a, 2 * asplit);
        const uint32_t s = ks > 0 ? 1u : 0u;
        if constexpr (B_EXACT) {
            mma(a2, b, s);
            mma(a1, b, 1u);
            mma(a, b, 1u);
        } else {
            const uint64_t b1 = desc_add(b, bsplit), b2 = desc_add(b, 2 * bsplit);
            mma(a2, b, s);
            mma(a, b2, 1u);
            mma(a1, b1, 1u);
            mma(a1, b, 1u);
            mma(a, b1, 1u);
            mma(a, b, 1u);
        }
    }
    wg_commit();
}

// x3_block<0, TB, NJ, NK, false> with A from registers: a[p][ks] is the m64k16 fragment (wgmma_bf16_n64_ra) of piece p
// (0 hi, 1 mid, 2 lo) at k-step ks.  The same products in the same order as with A read from a shared-memory tile.
template <int TB, int NJ, int NK>
__device__ __forceinline__ void x3_block_ra(float (&d)[4 * NJ], const uint32_t (&a)[3][NK][4], uint64_t b0, uint32_t bsplit,
                                            uint32_t bkstep) {
    auto mma = [&](const uint32_t (&ap)[4], uint64_t b, uint32_t s) {
        if constexpr (NJ == 8) wgmma_bf16_n64_ra<TB>(d, ap, b, s);
        else wgmma_bf16_n16_ra<TB>(d, ap, b, s);
    };
    wg_fence();
    acc_fence(d);
#pragma unroll
    for (int ks = 0; ks < NK; ++ks) {
        const uint64_t b = desc_add(b0, (uint32_t)ks * bkstep), b1 = desc_add(b, bsplit), b2 = desc_add(b, 2 * bsplit);
        const uint32_t s = ks > 0 ? 1u : 0u;
        mma(a[2][ks], b, s);
        mma(a[0][ks], b2, 1u);
        mma(a[1][ks], b1, 1u);
        mma(a[1][ks], b, 1u);
        mma(a[0][ks], b1, 1u);
        mma(a[0][ks], b, 1u);
    }
    wg_commit();
}

// D[acc] (+)= A * B over NK k-steps of 16, with the six split products (small terms first); called by all 128 threads
// of one warpgroup.
//   M = 64 or 128, N = 16 or 64; TA / TB: A / B read MN-major (an MN-major A has M = 64); B_EXACT: B is exactly
//   representable in bf16 (e.g. the ones tile), only the three A terms are issued and bsplit is not read.
//   a0 / b0: descriptors of the hi sub-tiles at k-step 0; asplit / bsplit: bytes between sub-tiles;
//   akstep / bkstep: bytes per k-step (K-major: 32; MN-major: 16 rows * pitch).
// M = 128 issues both m64 halves before draining the first: half 0 is stored while half 1 runs.  A product that adds
// to the image reads the old values in batches of independent loads, the first batch before it waits on its MMAs.
// Either way the stored value is d, or d + old, as one fp32 add.
// `waited(half)` is called when the MMAs of m64 half `half` have completed and before the image is written: for
// stage-time stamps, and for releasing the operands to their next writer (nothing by default).
struct NoStamp {
    __device__ __forceinline__ void operator()(int) const {}
};
template <int M, int N, int NK, int TA, int TB, bool B_EXACT = false, class Stamp = NoStamp>
__device__ __forceinline__ void gemm_x3(const Acc& acc, uint32_t d_addr, uint64_t a0, uint32_t asplit, uint32_t akstep,
                                        uint64_t b0, uint32_t bsplit, uint32_t bkstep, bool accumulate,
                                        Stamp waited = Stamp()) {
    static_assert((M == 64 || (M == 128 && TA == 0)) && (N == 16 || N == 64), "unsupported bf16x3 GEMM shape");
    constexpr int NJ = N / 8;
    // Every descriptor of the unrolled k-steps is invariant in the callers' tile loops; computed once there and held
    // across them, they would not fit in registers next to the accumulators.  Derive them afresh at every call.
    a0 = desc_fresh(a0);
    b0 = desc_fresh(b0);
    // rows 64..127 of a K-major A: 64 rows further down the tile (row pitch 128 B for SW128, 32 B for SW32)
    const uint32_t a_half_bytes = 64u * (((a0 >> 61) & 7u) == 2u ? 128u : 32u);
    if constexpr (M == 64) {
        float d[4 * NJ] = {};
        float2 old[2][NJ];
        x3_block<TA, TB, NJ, NK, B_EXACT>(d, a0, asplit, akstep, b0, bsplit, bkstep);
        if (accumulate) frag_load<NJ>(acc, d_addr, M, 0, old);
        wg_wait<0>();
        acc_fence(d);
        waited(0);
        if (accumulate) frag_add_store<NJ>(acc, d_addr, M, 0, d, old);
        else frag_store<NJ>(acc, d_addr, M, 0, d);
    } else {
        float d0[4 * NJ] = {}, d1[4 * NJ] = {};
        x3_block<TA, TB, NJ, NK, B_EXACT>(d0, a0, asplit, akstep, b0, bsplit, bkstep);
        x3_block<TA, TB, NJ, NK, B_EXACT>(d1, desc_add(a0, a_half_bytes), asplit, akstep, b0, bsplit, bkstep);
        if (accumulate) {
            // The two fragments leave the 640-thread update kernel (96 registers) room for half a row of old values.
            // So the four fragment rows go in turn, each batch of old values read as soon as registers are free for it:
            // half of the first row while the MMAs run, the other half after it, and from then on whole rows into the
            // registers that the stored rows have given up.
            constexpr int NH = NJ / 2;
            float* r00 = frag_row(acc, d_addr, M, 0, 0);
            float* r01 = r00 + 8 * acc.pitch;                 // M = 128: fragment row m lies in image lane m
            float* r10 = r00 + 64 * acc.pitch;
            float* r11 = r00 + 72 * acc.pitch;
            float2 oa[NH], ob[NH], oc[NJ], od[NJ], oe[NJ];
            row_load(r00, 0, oa);
            wg_wait<1>();
            acc_fence(d0);
            waited(0);
            row_add_store(r00, 0, d0, 0, oa);
            row_load(r00, NH, ob);
            row_add_store(r00, 0, d0, NH, ob);
            row_load(r01, 0, oc);
            row_add_store(r01, 1, d0, 0, oc);
            row_load(r10, 0, od);
            row_load(r11, 0, oe);
            wg_wait<0>();
            acc_fence(d1);
            waited(1);
            row_add_store(r10, 0, d1, 0, od);
            row_add_store(r11, 1, d1, 0, oe);
        } else {
            wg_wait<1>();
            acc_fence(d0);
            waited(0);
            frag_store<NJ>(acc, d_addr, M, 0, d0);
            wg_wait<0>();
            acc_fence(d1);
            waited(1);
            frag_store<NJ>(acc, d_addr, M, 1, d1);
        }
    }
}

// ---- products staged in shared memory ------------------------------------------------------------------
// A product of N = 64 (16) columns that its epilogue turns into a [128][N] bf16x3 operand tile can be staged as fp32 in
// that tile's own footprint instead of the image: three SW128 (SW32) sub-tiles `split` bytes apart, of which row r's fp32
// values take the 128 (32) bytes of row r in sub-tiles 0 and 1 -- columns 0-31 (0-7) in sub-tile 0, 32-63 (8-15) in
// sub-tile 1 -- with the sub-tile's 16-byte-chunk XOR swizzle.  So the fp32 values of rows 32 q .. 32 q + 31 lie inside
// those rows' bytes of the tile, and the epilogue warps of those rows alone can read them, meet, and store the bf16x3
// pieces over them.  The MMA-issue warpgroup writes them only past the wgmma wait that follows the last read of the tile.
struct Staged {
    uint32_t base;     // shared address of sub-tile 0 (1024-byte aligned)
    uint32_t split;    // bytes between the sub-tiles
};
template <int N>
__host__ __device__ constexpr uint32_t staged_off(int r, int c, uint32_t split) {
    static_assert(N == 16 || N == 64, "staged products are N = 16 (SW32) or N = 64 (SW128)");
    if constexpr (N == 64) return (uint32_t)(c >> 5) * split + (uint32_t)(r * 128 + ((((c >> 2) & 7) ^ (r & 7)) << 4) + ((c & 3) << 2));
    else return (uint32_t)(c >> 3) * split + (uint32_t)(r * 32 + ((((c >> 2) & 1) ^ ((r >> 2) & 1)) << 4) + ((c & 3) << 2));
}
// every fp32 value of every row r of a [128][N] product staged in sub-tiles `split` bytes apart lies in row r's bytes of
// sub-tile 0 or 1, 4-byte aligned, and no two values share bytes (for the static_asserts of the kernels that stage)
template <int N>
constexpr bool staged_in_own_rows(uint32_t split) {
    constexpr uint32_t pitch = N == 64 ? 128u : 32u;
    if (split < 128u * pitch) return false;
    for (int r = 0; r < 128; ++r) {
        uint32_t seen[N / 32 + 1] = {};      // bit per float slot of the row in sub-tiles 0 and 1
        for (int c = 0; c < N; ++c) {
            const uint32_t off = staged_off<N>(r, c, split), sub = off / split, in = off % split;
            if (sub > 1u || in / pitch != (uint32_t)r || (in & 3u) != 0u) return false;
            const uint32_t slot = sub * (pitch / 4u) + (in % pitch) / 4u;
            if ((seen[slot / 32u] >> (slot % 32u)) & 1u) return false;
            seen[slot / 32u] |= 1u << (slot % 32u);
        }
    }
    return true;
}
// the m64 fragment of rows 64 half .. 64 half + 63 of this warpgroup thread: element (rr, j, e) is row
// 64 half + 16 w + l / 4 + 8 rr, column 8 j + 2 (l % 4) + e
template <int N>
__device__ __forceinline__ void staged_store(const Staged& s, int half, const float (&d)[N / 2]) {
    const int t = threadIdx.x & 127, w = t >> 5, l = t & 31;
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
        const int m = 64 * half + 16 * w + (l >> 2) + 8 * rr;
#pragma unroll
        for (int j = 0; j < N / 8; ++j)
            asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(s.base + staged_off<N>(m, 8 * j + 2 * (l & 3), s.split)),
                         "f"(d[4 * j + 2 * rr]), "f"(d[4 * j + 2 * rr + 1]) : "memory");
    }
}
// NV consecutive columns [c0, c0 + NV) (c0 % 4 == 0, NV % 4 == 0) of row r
template <int N, int NV>
__device__ __forceinline__ void staged_load(const Staged& s, int r, int c0, float (&v)[NV]) {
#pragma unroll
    for (int i = 0; i < NV / 4; ++i)
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                     : "=f"(v[4 * i]), "=f"(v[4 * i + 1]), "=f"(v[4 * i + 2]), "=f"(v[4 * i + 3])
                     : "r"(s.base + staged_off<N>(r, c0 + 4 * i, s.split)));
}

// gemm_x3<128, N, NK, 0, TB> without accumulation, stored into the staging footprint s instead of the image: the same
// wgmmas in the same order, half 0 stored while half 1 runs.  Half 0's rows of the footprint are not rows that half 1's
// MMAs read, so A may be the tile being staged over.
template <int N, int NK, int TB>
__device__ __forceinline__ void gemm_x3_staged(const Staged& s, uint64_t a0, uint32_t asplit, uint32_t akstep, uint64_t b0,
                                        uint32_t bsplit, uint32_t bkstep) {
    static_assert(N == 16 || N == 64, "unsupported bf16x3 GEMM shape");
    constexpr int NJ = N / 8;
    a0 = desc_fresh(a0);
    b0 = desc_fresh(b0);
    float d0[4 * NJ] = {}, d1[4 * NJ] = {};
    x3_block<0, TB, NJ, NK, false>(d0, a0, asplit, akstep, b0, bsplit, bkstep);
    x3_block<0, TB, NJ, NK, false>(d1, desc_add(a0, 64u * (((a0 >> 61) & 7u) == 2u ? 128u : 32u)), asplit, akstep, b0, bsplit, bkstep);
    wg_wait<1>();
    acc_fence(d0);
    staged_store<N>(s, 0, d0);
    wg_wait<0>();
    acc_fence(d1);
    staged_store<N>(s, 1, d1);
}

// Rows 64 r .. 64 r + 63 (r = 0 or 1) of a 128-row product with a K-major A, as one m64 block over the whole K, stored
// once: into the image rows of the M = 128 product at d_addr (row m in lane m), or into the staging footprint s.  The two
// row halves of a product share nothing but B, so each can be issued, stored and announced on its own.
//   NC = 2: K is split into two runs of NK k-steps; each run is its own wgmma chain, started from zero into its own
//   fragment and both in flight together, and the stored value is the fp32 sum of the two chains, one add per element.
//   That is the value two column-half phases of gemm_x3<128, ...> leave in the image (the second accumulating), bit for
//   bit, without the image read.  One chain over all 2 NK k-steps would save the add and a fragment and round differently.
//   NC = 1: one chain of NK k-steps, stored as it is.
// a0 / b0 and the strides as for gemm_x3; `waited(r)` is called when the MMAs have completed.
template <int N, int NK, int NC, int TB, class Stamp>
__device__ __forceinline__ void rows_x3(float (&d)[N / 2], int r, uint64_t a0, uint32_t asplit, uint32_t akstep,
                                        uint64_t b0, uint32_t bsplit, uint32_t bkstep, Stamp waited) {
    static_assert((N == 16 || N == 64) && (NC == 1 || NC == 2), "unsupported bf16x3 row-half GEMM shape");
    constexpr int NJ = N / 8;
    a0 = desc_fresh(a0);
    b0 = desc_fresh(b0);
    a0 = desc_add(a0, (uint32_t)r * 64u * (((a0 >> 61) & 7u) == 2u ? 128u : 32u));
#pragma unroll
    for (int i = 0; i < 4 * NJ; ++i) d[i] = 0.f;
    x3_block<0, TB, NJ, NK, false>(d, a0, asplit, akstep, b0, bsplit, bkstep);
    if constexpr (NC == 2) {
        float d1[4 * NJ] = {};
        x3_block<0, TB, NJ, NK, false>(d1, desc_add(a0, NK * akstep), asplit, akstep, desc_add(b0, NK * bkstep), bsplit, bkstep);
        wg_wait<0>();
        acc_fence(d);
        acc_fence(d1);
        waited(r);
#pragma unroll
        for (int i = 0; i < 4 * NJ; ++i) d[i] += d1[i];
    } else {
        wg_wait<0>();
        acc_fence(d);
        waited(r);
    }
}
template <int N, int NK, int NC, int TB, class Stamp = NoStamp>
__device__ __forceinline__ void gemm_x3_rows(const Acc& acc, uint32_t d_addr, int r, uint64_t a0, uint32_t asplit,
                                             uint32_t akstep, uint64_t b0, uint32_t bsplit, uint32_t bkstep,
                                             Stamp waited = Stamp()) {
    float d[N / 2];
    rows_x3<N, NK, NC, TB>(d, r, a0, asplit, akstep, b0, bsplit, bkstep, waited);
    frag_store<N / 8>(acc, d_addr, 128, r, d);
}
template <int N, int NK, int NC, int TB, class Stamp = NoStamp>
__device__ __forceinline__ void gemm_x3_rows(const Staged& s, int r, uint64_t a0, uint32_t asplit, uint32_t akstep,
                                             uint64_t b0, uint32_t bsplit, uint32_t bkstep, Stamp waited = Stamp()) {
    float d[N / 2];
    rows_x3<N, NK, NC, TB>(d, r, a0, asplit, akstep, b0, bsplit, bkstep, waited);
    staged_store<N>(s, r, d);
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

// store the column pair (c, c + 1) (c even) of row r of a SW32 x3 tile: the words store16_x3_sw32 writes there
__device__ __forceinline__ void store2_x3_sw32(uint32_t base, uint32_t split, int r, int c, float a, float b) {
    uint32_t w0, w1, w2;
    split2(a, b, w0, w1, w2);
    const uint32_t o = base + off32(r, c);
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(o), "r"(w0) : "memory");
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(o + split), "r"(w1) : "memory");
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(o + 2 * split), "r"(w2) : "memory");
}

// single element stores (weight staging)
__device__ __forceinline__ void store1_x3(uint32_t base, uint32_t split, uint32_t off, float x) {
    uint32_t w0, w1, w2;
    split2(x, 0.f, w0, w1, w2);
    sts16(base + off, (uint16_t)w0); sts16(base + split + off, (uint16_t)w1); sts16(base + 2 * split + off, (uint16_t)w2);
}

// ---- issue helpers on 32-bit shared addresses ---------------------------------------------------------
// mma_commit on a 32-bit shared address
__device__ __forceinline__ void mma_commit_a(uint32_t bar) {
    __threadfence_block();
    asm volatile("bar.sync 3, 128;\n" ::: "memory");
    if ((threadIdx.x & 127) == 0) mbar_arrive(bar);
}
// The warpgroup's MMAs have read their operands: one arrival for the warps that overwrite them.  Called by all 128
// threads once each is past its wgmma wait; nothing those warps read was written here, so there is no fence.
__device__ __forceinline__ void mma_release_a(uint32_t bar) {
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
struct TanhAcc {
    __device__ __forceinline__ float operator()(float x) const { return tanh_acc(x); }
};

}  // namespace x3
}  // namespace osb
