// Tensor-core Fisher-vector product, forward half: the tangent of the policy mean along a parameter direction v, for
// every sampled row.
//
//   NaturalPG._fvp (algorithms/on_policy/base/natural_pg.py:L74-119):  F v = grad( (grad KL)^T v ), which for the
//   Gaussian actor at theta = theta_old is  [ (2 / A) v_logsigma ;  (1 / (B A)) sum_s J(s)^T diag(sigma^-2) J(s) v_mu ]
//   (SURVEY §8a row 13).  This kernel computes d mu(s) = J(s) v_mu by forward-mode differentiation of the MLP:
//       T1 = X V1^T + bv1,              dH1 = f'(H1) T1
//       T2 = dH1 W2^T + H1 V2^T + bv2,  dH2 = f'(H2) T2
//       dmu = dH2 W3^T + H2 V3^T + bv3
//   next to the ordinary forward (Z1 = X W1^T + b1, H1 = f(Z1), ...; f the hidden activation of csrc/activation.cuh),
//   on the tiles of csrc/tc_forward.cuh:
//     X3 = false: tf32 wgmma (O <= 512; CHUNKED: layer 1 as a K loop over 64-column chunks of X, W1 and V1), tanh_fast;
//     X3 = true : split-bf16, six bf16 wgmma products per product (O <= 64), tanh_acc.
//   The backward half J^T diag(sigma^-2) dmu / (B A) is the precision's update kernel with loss kind LOSS_FVP
//   (fvp_backward_tc in csrc/update_tc.cu, fvp_backward_x3 in csrc/update_x3.cu).
//
// One CTA per SM, tiles of 128 rows, FVP_NT<X3> threads: 256 for bf16x3, 512 for tf32 (measured faster than 256 for
// it on an H100 SXM at 700 W).  Warpgroup 0 issues the MMAs; in the epilogues thread (warp w, lane l) owns tile row
// 32 (w % 4) + l and the column group w / 4.  The weights and the direction's V1 V2 V3 are staged by the first 256
// threads with tc_stage_weights, V1 V2 V3 FvpTiles::V bytes past W1 W2 W3 (the tf32 K chunks of W1 and V1 by the two
// halves of the CTA side by side); the tangent activations (dH1, then dH2 over it) have their own buffer.
#include "common.cuh"
#include "loss.cuh"
#include "tc_forward.cuh"

namespace osb {

using namespace umma;

template <bool X3>
struct FvpTiles {
    using T = TcTiles<X3>;
    static constexpr uint32_t V = T::FLOATS - T::W1;                          // V1, V2, V3 = W1, W2, W3 + V
    static constexpr uint32_t D = T::FLOATS + V;                              // tangent activations
    static constexpr uint32_t FLOATS = D + (X3 ? 3 * T::SUB : TC_ROWS * 256);
};
// accumulator columns: Z [0, 64), T [64, 128), OUT [128, 144)
constexpr uint32_t FVP_C_Z = 0, FVP_C_T = 64, FVP_C_OUT = 128, FVP_COLS = 144;
// the region after the tiles: floats b1[64] b2[64] b3[16] (b3 unused), then bv1[64] bv2[64] bv3[16]
constexpr int FVP_B = 0, FVP_BV = 144, FVP_WORDS = 288;

template <bool X3>
constexpr int FVP_NT = X3 ? NTHREADS : 2 * NTHREADS;

struct FvpTanArgs {
    const float* obs; long long total; int stride;
    const float* theta; const float* vec; float* dmu;
    int O, A;
    float* acc;         // accumulator images, [gridDim.x][128][FVP_COLS]
};

// D[col] (+)= A B^T: A a [128][64] activation tile, B a [N][64] weight tile (N = 64, or 16 for layer 3)
template <bool X3, int N>
__device__ __forceinline__ void fvp_gemm(const Acc& tm, uint32_t col, uint32_t a, uint32_t b, bool accumulate) {
    using T = TcTiles<X3>;
    if constexpr (X3)
        x3::gemm_x3<128, N, 4, 0, 0>(tm, col, x3::desc128(a), T::SUB, 32u, x3::desc128(b), N == 64 ? T::WSUB : T::W3SUB, 32u,
                                     accumulate);
    else
        tc_gemm(tm, col, a, TC_ROWS, b, N, 128, N, 64, accumulate);
}

// columns [c0, c0 + 8) of row r of a [128][64] activation tile
template <bool X3>
__device__ __forceinline__ void fvp_store8(uint32_t tile, int r, int c0, const float (&v)[8]) {
    if constexpr (X3) {
        x3::store8_x3(tile, TcTiles<true>::SUB, r, c0, v);
    } else {
#pragma unroll
        for (int i = 0; i < 2; ++i)
            asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(tile_addr(tile, r, c0 + 4 * i, TC_ROWS)),
                         "f"(tf32r(v[4 * i])), "f"(tf32r(v[4 * i + 1])), "f"(tf32r(v[4 * i + 2])), "f"(tf32r(v[4 * i + 3]))
                         : "memory");
    }
}

template <bool X3, bool CHUNKED, int ACT>
__global__ void __launch_bounds__(FVP_NT<X3>, 1) fvp_tangent_kernel(FvpTanArgs p, NetSpec spec) {
    using T = TcTiles<X3>;
    using F = FvpTiles<X3>;
    constexpr int EC = 64 * 128 / FVP_NT<X3>;      // epilogue columns per thread
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const uint32_t pad = (1024u - (smem_u32(smem_raw) & 1023u)) & 1023u;
    const uint32_t B0 = smem_u32(smem_raw) + pad;
    float* sB = reinterpret_cast<float*>(smem_raw + pad + F::FLOATS) + FVP_B;
    float* sBv = reinterpret_cast<float*>(smem_raw + pad + F::FLOATS) + FVP_BV;
    __shared__ uint64_t bar;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int q = warp & 3, h = warp >> 2;
    const int O = p.O, A = p.A;
    const NetLayout L = actor_layout(O, A);
    if (FVP_NT<X3> == NTHREADS || tid < NTHREADS) {
        tc_stage_weights<X3>(B0, p.theta, L, O, sB, sB + 64, sB + 128);
        tc_stage_weights<X3>(B0 + F::V, p.vec, L, O, sBv, sBv + 64, sBv + 128);
    }
    if (tid == 0) { mbar_init(&bar, 1); mbar_init_fence(); }
    fence_async_smem();
    __syncthreads();
    const Acc tm = acc_cta(p.acc, FVP_COLS);
    const uint32_t lane_base = (uint32_t)(q * 32) << 16;
    const bool mma_wg = warpgroup_index() == 0;
    uint32_t phase = 0;
    const uint32_t sX = B0 + T::X, sH1 = B0 + T::H1, sD = B0 + F::D;
    const uint32_t sW1 = B0 + T::W1, sW2 = B0 + T::W2, sW3 = B0 + T::W3;

    const long long nrows = (p.total + p.stride - 1) / p.stride;
    const long long ntiles = (nrows + TC_ROWS - 1) / TC_ROWS;
    const int nchunks = CHUNKED ? (O + 63) >> 6 : 1;
    const bool vec = (O & 3) == 0;
    const int s_row = 32 * q + lane;

    // X is gathered into registers one chunk ahead, then stored into the X tile.
    //   bf16x3: thread -> row tid / 2, 32 columns; the next tile's first chunk flies under layers 2 and 3 (the layer-1
    //           epilogue has no registers to spare for it).
    //   tf32  : 16 values per thread, 128-bit loads by 16 threads per row (vec) or one column per thread; the next chunk,
    //           or the next tile's first, flies under the layer-1 MMAs and on through layers 2 and 3.
    float xpre[X3 ? 4 : 2][8];
    auto x_row = [&](long long tile, int m) -> long long {
        const long long k = tile * TC_ROWS + m;
        return (tile < ntiles && k < nrows) ? k * p.stride : -1;
    };
    auto gather = [&](long long tile, int c) {
        if constexpr (X3) {
            const long long row = x_row(tile, tid >> 1);
#pragma unroll
            for (int c8 = 0; c8 < 4; ++c8) tc_gather8(p.obs, O, vec, row, ((tid & 1) << 5) + 8 * c8, xpre[c8]);
        } else if (vec) {
            const int col = 64 * c + ((tid & 15) << 2);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const long long row = x_row(tile, (tid >> 4) + 32 * j);
                const float4 x = (row >= 0 && col < O) ? __ldg(reinterpret_cast<const float4*>(p.obs + row * O + col))
                                                       : make_float4(0.f, 0.f, 0.f, 0.f);
                float* v = &xpre[j >> 1][4 * (j & 1)];
                v[0] = x.x; v[1] = x.y; v[2] = x.z; v[3] = x.w;
            }
        } else {
            const int col = 64 * c + (tid & 63);
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const long long row = x_row(tile, (tid >> 6) + 8 * j);
                xpre[j >> 3][j & 7] = (row >= 0 && col < O) ? __ldg(p.obs + row * O + col) : 0.f;
            }
        }
    };
    auto store_x = [&]() {
        if constexpr (X3) {
#pragma unroll
            for (int c8 = 0; c8 < 4; ++c8) x3::store8_x3(sX, T::SUB, tid >> 1, ((tid & 1) << 5) + 8 * c8, xpre[c8]);
        } else if (vec) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float* v = &xpre[j >> 1][4 * (j & 1)];
                asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(tile_addr(sX, (tid >> 4) + 32 * j, (tid & 15) << 2, TC_ROWS)),
                             "f"(tf32r(v[0])), "f"(tf32r(v[1])), "f"(tf32r(v[2])), "f"(tf32r(v[3]))
                             : "memory");
            }
        } else {
#pragma unroll
            for (int j = 0; j < 16; ++j) sts(tile_addr(sX, (tid >> 6) + 8 * j, tid & 63, TC_ROWS), tf32r(xpre[j >> 3][j & 7]));
        }
    };
    // H = f(Z + b) into `dst`, dH = f'(H) (T + bv) into the tangent buffer; the layer's MMAs have completed
    const Hidden<ACT, TcTanh<X3>> af(spec, 0);
    auto epilogue = [&](const float* sBz, const float* sBt, int width, uint32_t dst) {
#pragma unroll
        for (int c8 = 0; c8 < EC / 8; ++c8) {
            const int c0 = EC * h + 8 * c8;
            float z[8], t[8];
            acc_ld<8>(tm, lane_base + FVP_C_Z + (uint32_t)c0, z);
            acc_ld<8>(tm, lane_base + FVP_C_T + (uint32_t)c0, t);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float hh = af(z[i] + sBz[c0 + i], c0 + i, width);
                z[i] = hh;
                t[i] = af.d(hh) * (t[i] + sBt[c0 + i]);
            }
            fvp_store8<X3>(dst, s_row, c0, z);
            fvp_store8<X3>(sD, s_row, c0, t);
        }
        fence_async_smem();
        __syncthreads();
    };

    gather(blockIdx.x, 0);
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        // ---- layer 1: Z1 = X W1^T, T1 = X V1^T --------------------------------------------------------------------
#pragma unroll 1
        for (int c = 0; c < nchunks; ++c) {
            if constexpr (CHUNKED) {     // the previous chunk's MMAs have completed: X, W1 and V1 are free
                if (tid < NTHREADS) tc_stage_w1_chunk(sW1, p.theta, L, O, c);               // W1 and V1 side by side
                else tc_stage_w1_chunk(sW1 + F::V, p.vec, L, O, c, tid - NTHREADS);
            }
            store_x();
            fence_async_smem();
            __syncthreads();
            // the loads of the next chunk or tile: tf32 K chunks issue them ahead of the MMAs in every warp; otherwise
            // warpgroup 0 issues them once its MMAs have completed (measured faster, and no spills there)
            auto gather_next = [&] {
                if (c + 1 < nchunks) gather(tile, c + 1);
                else if constexpr (!X3) gather(tile + gridDim.x, 0);
            };
            if constexpr (CHUNKED) gather_next();
            if (mma_wg) {
                fvp_gemm<X3, 64>(tm, FVP_C_Z, sX, sW1, CHUNKED && c > 0);
                fvp_gemm<X3, 64>(tm, FVP_C_T, sX, sW1 + F::V, CHUNKED && c > 0);
                mma_commit(&bar);
            }
            if constexpr (!CHUNKED) gather_next();
            mbar_wait(&bar, phase); phase ^= 1;
        }
        epilogue(sB, sBv, af.w1, sH1);                                // H1, dH1
        // ---- layer 2: Z2 = H1 W2^T, T2 = dH1 W2^T + H1 V2^T ---------------------------------------------------------
        if (mma_wg) {
            fvp_gemm<X3, 64>(tm, FVP_C_Z, sH1, sW2, false);
            fvp_gemm<X3, 64>(tm, FVP_C_T, sD, sW2, false);
            fvp_gemm<X3, 64>(tm, FVP_C_T, sH1, sW2 + F::V, true);
            mma_commit(&bar);
        }
        if constexpr (X3) gather(tile + gridDim.x, 0);
        mbar_wait(&bar, phase); phase ^= 1;
        epilogue(sB + 64, sBv + 64, af.w2, sX);                       // H2 over X, dH2 over dH1
        // ---- layer 3: dmu = dH2 W3^T + H2 V3^T + bv3 ----------------------------------------------------------------
        if (mma_wg) {
            fvp_gemm<X3, 16>(tm, FVP_C_OUT, sD, sW3, false);
            fvp_gemm<X3, 16>(tm, FVP_C_OUT, sX, sW3 + F::V, true);
            mma_commit(&bar);
        }
        mbar_wait(&bar, phase); phase ^= 1;
        const long long k = tile * TC_ROWS + s_row;
        if (h == 0 && k < nrows) {
            float o16[16];
            acc_ld16(tm, lane_base + FVP_C_OUT, o16);
#pragma unroll
            for (int a = 0; a < 16; ++a)
                if (a < A) p.dmu[k * p.stride * A + a] = o16[a] + sBv[128 + a];
        }
        __syncthreads();          // the layer-3 MMAs (readers of both buffers) have completed
    }
}

// Fisher-vector product partials of one precision: the tangent pass into the dmu scratch, then the backward half.
// 1024: the alignment pad in front of the tiles.
template <bool X3>
static int fvp_partials(const float* theta_actor, const float* vec, int O, int A, const float* obs, long long total,
                        int stride, float* dmu, float* gpart, float* stats_scratch, cudaStream_t stream) {
    OSB_CHECK_ARG(theta_actor && vec && obs && dmu && gpart && stats_scratch && total > 0 && stride > 0, "bad argument");
    if (X3) OSB_CHECK_ARG(O > 0 && O <= 64 && A > 0 && A <= 16, "bf16x3 path needs O <= 64, A <= 16");
    else OSB_CHECK_ARG(O > 0 && O <= 512 && A > 0 && A <= 16, "tensor-core path needs O <= 512, A <= 16");
    const long long nrows = (total + stride - 1) / stride;
    OSB_CHECK_ARG(nrows < (1ll << 31), "too many rows");
    const int nb = osb_tc_grid_blocks(nrows, 1);
    FvpTanArgs t{obs, total, stride, theta_actor, vec, dmu, O, A, nullptr};
    t.acc = acc_scratch(ACC_FVP, (size_t)nb * 128 * FVP_COLS * sizeof(float));
    if (!t.acc) return OSB_ERR_CUDA;
    const size_t smem = 1024 + FvpTiles<X3>::FLOATS + FVP_WORDS * sizeof(float);
    const NetSpec spec = net_spec();
    const int rc = with_act<false>(spec.act[0], [&](auto a) {
        static bool attr = false;
        if (!attr) {
            OSB_CUDA(cudaFuncSetAttribute(fvp_tangent_kernel<X3, false, a.value>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            if constexpr (!X3)
                OSB_CUDA(cudaFuncSetAttribute(fvp_tangent_kernel<false, true, a.value>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            attr = true;
        }
        void (*kernel)(FvpTanArgs, NetSpec) = fvp_tangent_kernel<X3, false, a.value>;
        if constexpr (!X3)
            if (O > 64) kernel = fvp_tangent_kernel<false, true, a.value>;
        kernel<<<nb, FVP_NT<X3>, smem, stream>>>(t, spec);
        OSB_LAUNCH_CHECK();
        return OSB_OK;
    });
    if (rc) return rc;
    return X3 ? fvp_backward_x3(theta_actor, vec, O, A, obs, total, stride, dmu, gpart, stats_scratch, stream)
              : fvp_backward_tc(theta_actor, vec, O, A, obs, total, stride, dmu, gpart, stats_scratch, stream);
}

}  // namespace osb

using namespace osb;

extern "C" {

// tf32 Fisher-vector product partials (O <= 512): see the header.
int osb_fvp_partials_tc(const float* theta_actor, const float* vec, int O, int A, const float* obs, long long total,
                        int stride, float* dmu, float* gpart, float* stats_scratch, void* stream) {
    return fvp_partials<false>(theta_actor, vec, O, A, obs, total, stride, dmu, gpart, stats_scratch, (cudaStream_t)stream);
}

// Split-bf16 Fisher-vector product partials (O <= 64): see the header.
int osb_fvp_partials_x3(const float* theta_actor, const float* vec, int O, int A, const float* obs, long long total,
                        int stride, float* dmu, float* gpart, float* stats_scratch, void* stream) {
    return fvp_partials<true>(theta_actor, vec, O, A, obs, total, stride, dmu, gpart, stats_scratch, (cudaStream_t)stream);
}

}  // extern "C"
