// The tensor-core MLP forward (obs -> 64 -> 64 -> out <= 16, tanh hidden layers) on tiles of 128 rows, shared by
// rollout_step_tc_kernel (csrc/rollout.cu), policy_tc_kernel (csrc/policy.cu) and actor_eval_tc_kernel
// (csrc/eval_tc.cu), so that the rollout, the policy step and the evaluation compute one function bit for bit.
//   X3 = false: tf32 wgmma tiles (csrc/umma.cuh), layer 1 as a K loop over 64-column chunks for inputs up to 512 wide;
//   X3 = true : split-bf16 tiles (csrc/x3.cuh), inputs up to 64 wide, one activation buffer (X, H1 and H2 overwrite
//               each other in place: every epilogue starts after its layer's MMAs completed), accurate tanh.
// 256 threads: warpgroup 0 issues the MMAs; in the epilogues thread (warp w, lane l) owns tile row 32 (w % 4) + l and
// the 32-column half w / 4.  The OUT product lands in accumulator columns [TC_C_OUT, TC_C_OUT + 16) without its bias.
#pragma once
#include <type_traits>

#include "mlp.cuh"
#include "umma.cuh"
#include "x3.cuh"

namespace osb {

constexpr int TC_ROWS = 128;                                    // rows per tile
constexpr uint32_t TC_C_Z = 0, TC_C_OUT = 64, TC_COLS = 80;     // accumulator columns: Z [0, 64), OUT [64, 80)

// Operand tiles, byte offsets from the 1024-byte aligned base of the dynamic shared memory.  tf32: X / H2 [128][64],
// H1 [128][64], W1 [64][64] (one 64-column chunk), W2 [64][64], W3 [16][64]; bf16x3: the activation buffer and the
// weights, three bf16 sub-tiles each, SUB / WSUB / W3SUB bytes apart.  The caller's own region starts at FLOATS.
template <bool X3>
struct TcTiles {
    static constexpr uint32_t SUB = TC_ROWS * 128, WSUB = 64 * 128, W3SUB = 16 * 128;
    static constexpr uint32_t X = 0;
    static constexpr uint32_t H1 = X3 ? X : TC_ROWS * 256;
    static constexpr uint32_t W1 = X3 ? 3 * SUB : 2 * TC_ROWS * 256;
    static constexpr uint32_t W2 = W1 + (X3 ? 3 * WSUB : 16384u);
    static constexpr uint32_t W3 = W2 + (X3 ? 3 * WSUB : 16384u);
    static constexpr uint32_t FLOATS = W3 + (X3 ? 3 * W3SUB : 4096u);
};

// W1 [64][In], W2 [64][64], W3 [out][64] of one network into the tiles, b1, b2 and b3 (zero padded to 16) into shared
// floats.  tf32 with In > 64: W1 is left to tc_stage_rows, chunk by chunk.  All loads are in flight before the stores;
// bf16x3 issues them in groups of BATCH items (of 8) per thread, for kernels whose staging would otherwise set their
// register count.
template <bool X3, int BATCH = 8>
__device__ __forceinline__ void tc_stage_weights(uint32_t base, const float* theta, const NetLayout& L, int In, float* sB1,
                                                 float* sB2, float* sB3) {
    using namespace umma;
    using T = TcTiles<X3>;
    const int tid = threadIdx.x;
    const uint32_t sW1 = base + T::W1, sW2 = base + T::W2, sW3 = base + T::W3;
    if constexpr (X3) {
        for (int i0 = tid; i0 < 64 * 32; i0 += BATCH * NTHREADS) {   // W1, W2: item i = row i / 32, columns 2 (i % 32) + {0, 1}
            float a1[BATCH], b1[BATCH], a2[BATCH], b2[BATCH];
#pragma unroll
            for (int j = 0; j < BATCH; ++j) {
                const int i = i0 + j * NTHREADS, n = i >> 5, k = (i & 31) << 1;
                a1[j] = (k < In) ? __ldg(theta + L.off_w1 + n * In + k) : 0.f;
                b1[j] = (k + 1 < In) ? __ldg(theta + L.off_w1 + n * In + k + 1) : 0.f;
                a2[j] = __ldg(theta + L.off_w2 + n * 64 + k); b2[j] = __ldg(theta + L.off_w2 + n * 64 + k + 1);
            }
#pragma unroll
            for (int j = 0; j < BATCH; ++j) {
                const int i = i0 + j * NTHREADS, n = i >> 5, k = (i & 31) << 1;
                uint32_t w0, w1, w2;
                const uint32_t off = x3::off128(n, k);
                x3::split2(a1[j], b1[j], w0, w1, w2);
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(sW1 + off), "r"(w0) : "memory");
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(sW1 + T::WSUB + off), "r"(w1) : "memory");
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(sW1 + 2 * T::WSUB + off), "r"(w2) : "memory");
                x3::split2(a2[j], b2[j], w0, w1, w2);
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(sW2 + off), "r"(w0) : "memory");
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(sW2 + T::WSUB + off), "r"(w1) : "memory");
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(sW2 + 2 * T::WSUB + off), "r"(w2) : "memory");
            }
        }
        constexpr int B3 = BATCH < 2 ? BATCH : 2;
        for (int i0 = tid; i0 < 16 * 32; i0 += B3 * NTHREADS) {      // W3
            float a3[B3], b3[B3];
#pragma unroll
            for (int j = 0; j < B3; ++j) {
                const int i = i0 + j * NTHREADS, o = i >> 5, k = (i & 31) << 1;
                a3[j] = (o < L.out) ? __ldg(theta + L.off_w3 + o * 64 + k) : 0.f;
                b3[j] = (o < L.out) ? __ldg(theta + L.off_w3 + o * 64 + k + 1) : 0.f;
            }
#pragma unroll
            for (int j = 0; j < B3; ++j) {
                const int i = i0 + j * NTHREADS, o = i >> 5, k = (i & 31) << 1;
                uint32_t w0, w1, w2;
                const uint32_t off = x3::off128(o, k);
                x3::split2(a3[j], b3[j], w0, w1, w2);
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(sW3 + off), "r"(w0) : "memory");
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(sW3 + T::W3SUB + off), "r"(w1) : "memory");
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(sW3 + 2 * T::W3SUB + off), "r"(w2) : "memory");
            }
        }
    } else {
        float w1v[16], w2v[16], w3v[4];
        const int k = tid & 63;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const int n = (tid >> 6) + 4 * j;
            w1v[j] = (k < In && In <= 64) ? __ldg(theta + L.off_w1 + n * In + k) : 0.f;
            w2v[j] = __ldg(theta + L.off_w2 + n * 64 + k);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int o = (tid >> 6) + 4 * j;
            w3v[j] = (o < L.out) ? __ldg(theta + L.off_w3 + o * 64 + k) : 0.f;
        }
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const int n = (tid >> 6) + 4 * j;
            sts(tile_addr(sW1, n, k, 64), tf32r(w1v[j]));
            sts(tile_addr(sW2, n, k, 64), tf32r(w2v[j]));
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) sts(tile_addr(sW3, (tid >> 6) + 4 * j, k, 16), tf32r(w3v[j]));
    }
    if (tid < 64) { sB1[tid] = __ldg(theta + L.off_b1 + tid); sB2[tid] = __ldg(theta + L.off_b2 + tid); }
    if (tid < 16) sB3[tid] = (tid < L.out) ? __ldg(theta + L.off_b3 + tid) : 0.f;
}

// X tile rows gathered from obs [*][O]: row_of(m) is the obs row of tile row m, or -1 for a zero row.
//   bf16x3: the whole tile; thread -> row tid / 2, 32-column half; 128-bit loads when vec (O % 4 == 0, obs 16-byte
//           aligned).  The previous tile's MMAs have completed: the buffer is free.
//   tf32  : chunk c (columns [64 c, 64 c + 64)) of X, and of W1 when O > 64; thread -> column tid % 64.
template <bool X3, class Row>
__device__ __forceinline__ void tc_stage_rows(uint32_t base, const float* obs, int O, bool vec, int c, const float* theta,
                                              const NetLayout& L, Row&& row_of) {
    using namespace umma;
    const int tid = threadIdx.x;
    if constexpr (X3) {
        const int xm = tid >> 1, xh = (tid & 1) << 5;
        const long long row = row_of(xm);
#pragma unroll
        for (int c8 = 0; c8 < 4; ++c8) {
            const int c0 = xh + 8 * c8;
            float v[8];
            if (vec) {
#pragma unroll
                for (int v4 = 0; v4 < 2; ++v4) {
                    const int cc = c0 + 4 * v4;
                    const float4 x = (row >= 0 && cc < O) ? __ldg(reinterpret_cast<const float4*>(obs + row * O + cc))
                                                          : make_float4(0.f, 0.f, 0.f, 0.f);
                    v[4 * v4] = x.x; v[4 * v4 + 1] = x.y; v[4 * v4 + 2] = x.z; v[4 * v4 + 3] = x.w;
                }
            } else {
#pragma unroll
                for (int i = 0; i < 8; ++i) v[i] = (row >= 0 && c0 + i < O) ? __ldg(obs + row * O + c0 + i) : 0.f;
            }
            x3::store8_x3(base + TcTiles<true>::X, TcTiles<true>::SUB, xm, c0, v);
        }
    } else {
        const int k = tid & 63, col = c * 64 + k;
        if (O > 64) {
            const uint32_t sW1 = base + TcTiles<false>::W1;
            float w1c[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) w1c[j] = (col < O) ? __ldg(theta + L.off_w1 + ((tid >> 6) + 4 * j) * O + col) : 0.f;
#pragma unroll
            for (int j = 0; j < 16; ++j) sts(tile_addr(sW1, (tid >> 6) + 4 * j, k, 64), tf32r(w1c[j]));
        }
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            float xv[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const long long row = row_of((tid >> 6) + 4 * (16 * half + j));
                xv[j] = (row >= 0 && col < O) ? __ldg(obs + row * O + col) : 0.f;
            }
#pragma unroll
            for (int j = 0; j < 16; ++j)
                sts(tile_addr(base + TcTiles<false>::X, (tid >> 6) + 4 * (16 * half + j), k, TC_ROWS), tf32r(xv[j]));
        }
    }
}

struct TcNop {
    template <class... Ts>
    __device__ __forceinline__ void operator()(Ts...) const {}
};

// The forward of one tile: layer 1, tanh(. + b1), layer 2, tanh(. + b2), then the OUT GEMM.  Returns after the OUT
// MMAs completed; `phase` is the mbarrier parity, carried across calls.
// stage(c) stages chunk c of X (bf16x3: the whole tile, c = 0) right before layer 1 consumes it; tf32 runs layer 1 as a
// K loop over nchunks chunks.  stage = TcNop: the caller has staged, fenced and synchronised the whole X tile.
// after(l) runs in every thread once layer l's MMAs completed (l = 1, 2, 3).
template <bool X3, class Stage, class After = TcNop>
__device__ __forceinline__ void tc_forward(uint32_t base, const umma::Acc& tm, uint64_t* bar, uint32_t& phase,
                                           const float* sB1, const float* sB2, int nchunks, Stage&& stage,
                                           After&& after = After{}) {
    using namespace umma;
    using T = TcTiles<X3>;
    constexpr bool staged = std::is_same<typename std::decay<Stage>::type, TcNop>::value;
    auto stage_chunk = [&](int c) {
        if constexpr (!staged) {
            stage(c);
            fence_async_smem();
            __syncthreads();
        }
    };
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q = warp & 3, h = warp >> 2;
    const uint32_t lane_base = (uint32_t)(q * 32) << 16;
    if constexpr (X3) {
        const uint64_t dAct = x3::desc128(base + T::X), dW1 = x3::desc128(base + T::W1), dW2 = x3::desc128(base + T::W2),
                       dW3 = x3::desc128(base + T::W3);
        auto hidden = [&](const float* sB) {   // tanh(Z + b) over the activation buffer
#pragma unroll
            for (int c8 = 0; c8 < 4; ++c8) {
                const int c0 = 32 * h + 8 * c8;
                float v[8];
                x3::acc_ld8(tm, lane_base + TC_C_Z + (uint32_t)c0, v);
#pragma unroll
                for (int i = 0; i < 8; ++i) v[i] = x3::tanh_acc(v[i] + sB[c0 + i]);
                x3::store8_x3(base + T::X, T::SUB, 32 * q + lane, c0, v);
            }
            fence_async_smem();
            __syncthreads();
        };
        stage_chunk(0);
        if (warp < 4) {
            x3::gemm_x3(tm, TC_C_Z, dAct, T::SUB, 32u, dW1, T::WSUB, 32u, x3::idesc_bf16(128, 64, 0, 0), 4, false);
            mma_commit(bar);
        }
        mbar_wait(bar, phase); phase ^= 1;
        after(1);
        hidden(sB1);
        if (warp < 4) {
            x3::gemm_x3(tm, TC_C_Z, dAct, T::SUB, 32u, dW2, T::WSUB, 32u, x3::idesc_bf16(128, 64, 0, 0), 4, false);
            mma_commit(bar);
        }
        mbar_wait(bar, phase); phase ^= 1;
        after(2);
        hidden(sB2);
        if (warp < 4) {
            x3::gemm_x3(tm, TC_C_OUT, dAct, T::SUB, 32u, dW3, T::W3SUB, 32u, x3::idesc_bf16(128, 16, 0, 0), 4, false);
            mma_commit(bar);
        }
        mbar_wait(bar, phase); phase ^= 1;
        after(3);
    } else {
        const uint32_t sX = base + T::X, sH1 = base + T::H1;
        auto hidden = [&](const float* sB, uint32_t dst) {   // tanh(Z + b) into the next layer's operand tile
            float v[32];
            acc_ld32(tm, lane_base + TC_C_Z + 32 * h, v);
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] = tanh_fast(v[i] + sB[32 * h + i]);
            store_row32(dst, 32 * q + lane, 32 * h, TC_ROWS, v);
            fence_async_smem();
            __syncthreads();
        };
#pragma unroll 1
        for (int c = 0; c < nchunks; ++c) {
            stage_chunk(c);
            if (warp < 4) { tc_gemm(tm, TC_C_Z, sX, TC_ROWS, base + T::W1, 64, 128, 64, 64, c > 0); mma_commit(bar); }
            mbar_wait(bar, phase); phase ^= 1;
        }
        after(1);
        hidden(sB1, sH1);
        if (warp < 4) { tc_gemm(tm, TC_C_Z, sH1, TC_ROWS, base + T::W2, 64, 128, 64, 64, false); mma_commit(bar); }
        mbar_wait(bar, phase); phase ^= 1;
        after(2);
        hidden(sB2, sX);
        if (warp < 4) { tc_gemm(tm, TC_C_OUT, sX, TC_ROWS, base + T::W3, 16, 128, 16, 64, false); mma_commit(bar); }
        mbar_wait(bar, phase); phase ^= 1;
        after(3);
    }
}

}  // namespace osb
