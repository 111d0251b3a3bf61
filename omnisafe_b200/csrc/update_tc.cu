// Tensor-core (wgmma, tf32 wgmma, accumulator images) variant of the fused minibatch
// forward + loss + backward kernel -- the "fast" arithmetic mode of csrc/update.cu (which stays as
// the exact-fp32 parity path).  Same interface, same per-CTA partial-gradient outputs.
//
// All GEMM operands are fp32 tiles in shared memory in the K-major 128B-swizzled canonical layout
// (csrc/umma.cuh).  TF32 has no usable MN-major view of such a tile, so every activation that is
// needed with the sample index as the contraction dimension (weight gradients) is produced a second
// time in transposed form by a role-swapped MMA (D^T = W * X^T) instead of a transposed copy:
//
//   per 128-sample tile and network (O <= 64; for 64 < O <= 512, MMA1 / MMA2 and MMA9 loop over 64-column chunks of X):
//     MMA1  Z1    [s][n] = X  * W1^T      -> H1    = f(.+b1)               (A operand of layer 2)
//     MMA2  Z1^T  [n][s] = W1 * X^T       -> H1^T                          (B operand of dW2)
//     MMA3  Z2    [s][n] = H1 * W2^T      -> H2
//     MMA4  OUT   [s][o] = H2 * W3^T      -> per-sample loss, dOUT
//     MMA5  dZ2   [s][k] = dOUT * W3      -> * f'(H2)                      (B operand of dZ1^T)
//     MMA6  dZ2^T [k][s] = W3^T * dOUT^T  -> * f'(H2)                      (A operand of dW2)
//     MMA7  dW2   [j][k] += dZ2^T * H1    (accumulator images kept across tiles)
//     MMA8  dZ1^T [k][s] = W2^T * dZ2^T   -> * f'(H1)                      (A operand of dW1)
//     MMA9  dW1   [j][o] += dZ1^T * X     (accumulator images kept across tiles)
//   dW3, the bias gradients and d log_std stay on the CUDA cores (tiny).
#include "common.cuh"
#include "loss.cuh"
#include "mlp.cuh"
#include "umma.cuh"

namespace osb {

using namespace umma;

constexpr int TT = 128;                 // samples per tile
constexpr uint32_t BUF = TT * 64 * 4;   // 32 KB activation buffer ([128][64] or [64][128] fp32)

struct TcArgs {
    Batch b;
    LossParams lc;
    const float* theta;
    float* gpart;
    float* stats_part;
    const int* stop_flag;
    int O, A, P, net_mask;
    const float* fvp_dmu;    // LOSS_FVP: tangent of mu per row [total][A] (fvp_tangent_kernel, csrc/fvp_tc.cu)
    const float* fvp_vec;    // LOSS_FVP: direction v (log_std block of F v)
    float fvp_scale;         // LOSS_FVP: 1 / (rows * A)
    int forward_only;        // pass 1 of FOCOPS / P3O: statistics only, no backward
    float* acc;              // accumulator images, one [128][TC_COLS] per CTA
    float* value_out;        // LOSS_DMU on a critic (DMU instantiation only), or null: V per row as this launch computes it
};

// accumulator column map (csrc/umma.cuh)
constexpr uint32_t C_Z = 0, C_ZT = 64, C_ZT2 = 192, C_OUT = 320, C_DW2 = 336, C_DW1 = 400, C_DW3 = 464, TC_COLS = 480;
constexpr int NTC = 512;   // 16 warps: lane quarter q = warp % 4, column group h = warp / 4 (0..3)

// 16-column variants of the row accessors (c0 % 16 == 0)
__device__ __forceinline__ void store_row16(uint32_t base, int r, int c0, int R, const float (&v)[16]) {
    const uint32_t row = base + (uint32_t)((c0 >> 5) * R * 128 + r * 128);
    const int ch0 = (c0 & 31) >> 2;
#pragma unroll
    for (int i = 0; i < 4; ++i)
        asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(row + (uint32_t)(((ch0 + i) ^ (r & 7)) << 4)),
                     "f"(tf32r(v[4 * i])), "f"(tf32r(v[4 * i + 1])), "f"(tf32r(v[4 * i + 2])), "f"(tf32r(v[4 * i + 3]))
                     : "memory");
}
__device__ __forceinline__ void load_row16(uint32_t base, int r, int c0, int R, float (&v)[16]) {
    const uint32_t row = base + (uint32_t)((c0 >> 5) * R * 128 + r * 128);
    const int ch0 = (c0 & 31) >> 2;
#pragma unroll
    for (int i = 0; i < 4; ++i)
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                     : "=f"(v[4 * i]), "=f"(v[4 * i + 1]), "=f"(v[4 * i + 2]), "=f"(v[4 * i + 3])
                     : "r"(row + (uint32_t)(((ch0 + i) ^ (r & 7)) << 4)));
}

// CHUNKED = obs dim > 64: layer 1 runs as a K loop over 64-column chunks of X / W1 (forward: Z1 and Z1^T
// accumulate over chunks; backward: one dW1 chunk per MMA, flushed from accumulator image into this CTA's partial gradient).
// EXT = the two-pass / supplied-dOUT loss kinds (FOCOPS, P3O, FVP); the plain instantiation (PPO-clip, ratio,
// cost surrogate: the headline path) carries none of their registers or branches.
// DMU = LOSS_DMU only: the supplied dL/dmu (fvp_dmu, per row) or, for a critic, dL/dV (tv_r / tv_c) is dOUT as it
// stands, no loss, no log_std term.
template <bool CHUNKED, bool EXT, bool DMU, int ACT>
__global__ void __launch_bounds__(NTC, 1) minibatch_grad_tc_kernel(TcArgs p, NetSpec spec) {
    if (p.stop_flag && *p.stop_flag) return;
    // one network selected: grid.y == 1 and all of grid.x (up to one CTA per SM) works on that network
    const int net = (gridDim.y == 1) ? (__ffs(p.net_mask) - 1) : (int)blockIdx.y;
    if (!((p.net_mask >> net) & 1)) return;
    const Hidden<ACT, umma::TanhFast> af(spec, net);

    extern __shared__ __align__(16) uint8_t smem_raw[];
    const uint32_t pad = (1024u - (smem_u32(smem_raw) & 1023u)) & 1023u;   // tiles need 1024 B alignment
    const uint32_t B0 = smem_u32(smem_raw) + pad;   // X -> H2 -> dZ1^T
    const uint32_t B1 = B0 + BUF;                   // X^T
    const uint32_t B2 = B1 + BUF;                   // H1 -> dZ2
    const uint32_t B3 = B2 + BUF;                   // H1^T
    const uint32_t B4 = B3 + BUF;                   // dOUT (first 16 KB) -> dZ2^T
    const uint32_t sW1 = B4 + BUF;                  // [64][64]
    const uint32_t sW2 = sW1 + 16384;               // [64][64]
    const uint32_t sW2T = sW2 + 16384;              // [64][64]
    const uint32_t sW3 = sW2T + 16384;              // [16][64]   (2 atoms x 16 rows)
    const uint32_t sW3T = sW3 + 4096;               // [64][32]   (cols >= out zero)
    float* sB1 = reinterpret_cast<float*>(smem_raw + pad + 5 * BUF + 3 * 16384 + 4096 + 8192);
    float* sB2 = sB1 + 64;
    float* sB3 = sB2 + 64;            // [16]
    float* sPol = sB3 + 16;           // [48] policy constants of csrc/loss.cuh
    float* sStat = sPol + 48;         // [8]
    float* sRed = sStat + 8;          // [4 * 8 + 4 * 16 + 4 * 16]
    float* sB3acc = sRed + 160;       // [16]
    float* sOld = sB3acc + 16;        // [32] old-policy constants of csrc/loss.cuh
    float* sDls = sOld + 32;          // [16] accumulated d log_std
    long long* sRowBuf = reinterpret_cast<long long*>(sDls + 16);   // [2][128] rows of this / the next tile
    __shared__ uint64_t bar;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int q = warp & 3, h = warp >> 2;           // h in [0, 4)
    const int O = p.O, A = p.A;
    const NetLayout L = net_layout(net, O, A);
    const int noff = net_offset(net, O, A);
    const float* theta = p.theta + noff;
    float* gout = p.gpart + (size_t)blockIdx.x * p.P + noff;
    const int ntiles = (p.b.mb_count + TT - 1) / TT;
    const float inv_b = 1.0f / (float)p.b.mb_count;

    // ---- weights -> swizzled K-major tiles (loads batched so they are all in flight together) ----
    {
        float w1v[8], w2v[8], w3v[2];
        const int k = tid & 63;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int n = (tid >> 6) + 8 * j;
            w1v[j] = (!CHUNKED && k < O) ? __ldg(theta + L.off_w1 + n * O + k) : 0.f;
            w2v[j] = __ldg(theta + L.off_w2 + n * 64 + k);
        }
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int o = (tid >> 6) + 8 * j;
            w3v[j] = (o < L.out) ? __ldg(theta + L.off_w3 + o * 64 + k) : 0.f;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int n = (tid >> 6) + 8 * j;
            sts(tile_addr(sW1, n, k, 64), tf32r(w1v[j]));
            const float w2 = tf32r(w2v[j]);
            sts(tile_addr(sW2, n, k, 64), w2);
            sts(tile_addr(sW2T, k, n, 64), w2);
        }
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int o = (tid >> 6) + 8 * j;
            const float w = tf32r(w3v[j]);
            sts(tile_addr(sW3, o, k, 16), w);
            sts(tile_addr(sW3T, k, o, 64), w);
        }
    }
    for (int i = tid; i < 64 * 16; i += NTC) sts(tile_addr(sW3T, i >> 4, 16 + (i & 15), 64), 0.f);
    if (tid < 64) { sB1[tid] = __ldg(theta + L.off_b1 + tid); sB2[tid] = __ldg(theta + L.off_b2 + tid); }
    if (tid < 16) {
        sB3[tid] = (tid < L.out) ? __ldg(theta + L.off_b3 + tid) : 0.f;
        const bool act = net == 0 && tid < A;
        stage_policy(sPol, tid, act ? __ldg(theta + L.off_logstd + tid) : 0.f);
        stage_policy_old(sOld, tid, (act && p.lc.logstd_old) ? __ldg(p.lc.logstd_old + tid) : 0.f);
        sDls[tid] = 0.f;
    }
    if (tid < 8) sStat[tid] = 0.f;
    if (tid < 16) sB3acc[tid] = 0.f;
    if (tid == 0) { mbar_init(&bar, 1); mbar_init_fence(); }
    __syncthreads();
    const Acc tm = acc_cta(p.acc, TC_COLS);
    const uint32_t lane_base = (uint32_t)(q * 32) << 16;
    uint32_t phase = 0;

    const AdvNorm an = adv_norm(p.b.moments, p.lc.lagrange);
    const bool is_fvp = EXT && p.lc.kind == LOSS_FVP, is_focops = EXT && p.lc.kind == LOSS_FOCOPS;
    float ab1 = 0.f, ab2 = 0.f;
    bool first_tile = true;
    const int s_row = 32 * q + lane;       // sample row of this thread in [s][.] accumulators
    const int t_row = 16 * q + lane;       // row (valid for lane < 16) in [64][.] accumulators
    const int c16 = 16 * h;                // 16-column group of the plain epilogues
    const int c32 = 32 * h;                // 32-column group of the transposed epilogues

    const bool vec = (O & 3) == 0;            // rows 16 B aligned: 128-bit gathers, prefetched one tile ahead
    auto tile_rows = [&](int tile, long long* dst) {
        if (tid < TT) {
            const int local = tile * TT + tid;
            dst[tid] = (local < p.b.mb_count) ? sample_row(p.b, p.b.mb_start + local) : -1;
        }
    };
    float4 xpre[4];
    auto prefetch_x = [&](const long long* rows) {
        const int k4 = (tid & 15) << 2;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const long long row = rows[(tid >> 4) + 32 * j];
            xpre[j] = (row >= 0 && k4 < O) ? __ldg(reinterpret_cast<const float4*>(p.b.obs + row * O + k4))
                                            : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    };
    // CHUNKED: one 64-column chunk of this thread's X elements in flight (global -> registers -> tile)
    const int nchunks = (O + 63) >> 6;
    float xr[16];
    auto load_chunk = [&](const long long* rows, int c) {
        if (vec) {
            const int col = c * 64 + ((tid & 15) << 2);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const long long row = rows[(tid >> 4) + 32 * j];
                const float4 v = (row >= 0 && col < O) ? __ldg(reinterpret_cast<const float4*>(p.b.obs + row * O + col))
                                                        : make_float4(0.f, 0.f, 0.f, 0.f);
                xr[4 * j] = v.x; xr[4 * j + 1] = v.y; xr[4 * j + 2] = v.z; xr[4 * j + 3] = v.w;
            }
        } else {
            const int col = c * 64 + (tid & 63);
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const long long row = rows[(tid >> 6) + 8 * j];
                xr[j] = (row >= 0 && col < O) ? __ldg(p.b.obs + row * O + col) : 0.f;
            }
        }
    };
    auto store_chunk = [&](uint32_t dst, bool transposed) {     // dst: [128 s][64 k] K-major, or its transpose [64 k][128 s]
        if (vec) {
            const int k4 = (tid & 15) << 2;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int m = (tid >> 4) + 32 * j;
                const float a = tf32r(xr[4 * j]), b = tf32r(xr[4 * j + 1]), c = tf32r(xr[4 * j + 2]), d = tf32r(xr[4 * j + 3]);
                if (!transposed) {
                    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(tile_addr(dst, m, k4, TT)), "f"(a), "f"(b),
                                 "f"(c), "f"(d)
                                 : "memory");
                } else {
                    sts(tile_addr(dst, k4 + 0, m, 64), a); sts(tile_addr(dst, k4 + 1, m, 64), b);
                    sts(tile_addr(dst, k4 + 2, m, 64), c); sts(tile_addr(dst, k4 + 3, m, 64), d);
                }
            }
        } else {
            const int k = tid & 63;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int m = (tid >> 6) + 8 * j;
                const float v = tf32r(xr[j]);
                if (!transposed) sts(tile_addr(dst, m, k, TT), v);
                else sts(tile_addr(dst, k, m, 64), v);
            }
        }
    };
    auto load_w1_chunk = [&](int c) {                            // W1[:, 64c : 64c+64] -> sW1 (zero padded)
        const int k = tid & 63, col = c * 64 + k;
        float w[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) w[j] = (col < O) ? __ldg(theta + L.off_w1 + ((tid >> 6) + 8 * j) * O + col) : 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) sts(tile_addr(sW1, (tid >> 6) + 8 * j, k, 64), tf32r(w[j]));
    };
    int rpar = 0;
    tile_rows(blockIdx.x, sRowBuf);
    __syncthreads();
    if (CHUNKED) load_chunk(sRowBuf, 0);
    else if (vec) prefetch_x(sRowBuf);

    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        // ---- P0: X and X^T tiles (data of this tile was prefetched into registers) ---------------
        long long* sRow = sRowBuf + rpar * TT;
        long long* sRowNext = sRowBuf + (rpar ^ 1) * TT;
        const bool has_next = tile + (int)gridDim.x < ntiles;
        if (has_next) tile_rows(tile + gridDim.x, sRowNext);     // visible after the next barrier
        if (CHUNKED) {
            // X is staged chunk by chunk inside P1 (and again, transposed, inside P6)
        } else if (vec) {
            const int k4 = (tid & 15) << 2;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int m = (tid >> 4) + 32 * j;
                const float4 v = make_float4(tf32r(xpre[j].x), tf32r(xpre[j].y), tf32r(xpre[j].z), tf32r(xpre[j].w));
                asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(tile_addr(B0, m, k4, TT)), "f"(v.x),
                             "f"(v.y), "f"(v.z), "f"(v.w)
                             : "memory");
                sts(tile_addr(B1, k4 + 0, m, 64), v.x);
                sts(tile_addr(B1, k4 + 1, m, 64), v.y);
                sts(tile_addr(B1, k4 + 2, m, 64), v.z);
                sts(tile_addr(B1, k4 + 3, m, 64), v.w);
            }
        } else {
            const int k = tid & 63;
            float xv[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const long long row = sRow[(tid >> 6) + 8 * j];
                xv[j] = (row >= 0 && k < O) ? __ldg(p.b.obs + row * O + k) : 0.f;
            }
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int m = (tid >> 6) + 8 * j;
                const float v = tf32r(xv[j]);
                sts(tile_addr(B0, m, k, TT), v);
                sts(tile_addr(B1, k, m, 64), v);
            }
        }
        fence_async_smem();
        __syncthreads();
        // ---- P1: Z1 and Z1^T ---------------------------------------------------------------------
        if (CHUNKED) {
            for (int c = 0; c < nchunks; ++c) {
                load_w1_chunk(c);                     // the previous chunk's MMAs completed: B0 / sW1 are free
                store_chunk(B0, false);
                fence_async_smem();
                __syncthreads();
                if (c + 1 < nchunks) load_chunk(sRow, c + 1);      // next chunk's rows fly during the MMAs
                if (warpgroup_index() == 0) {
                    tc_gemm(tm, C_Z, B0, TT, sW1, 64, 128, 64, 64, c > 0);
                    tc_gemm(tm, C_ZT, sW1, 64, B0, TT, 64, 128, 64, c > 0);
                    mma_commit(&bar);
                }
                mbar_wait(&bar, phase); phase ^= 1;
            }
        } else {
            if (warpgroup_index() == 0) {
                tc_gemm(tm, C_Z, B0, TT, sW1, 64, 128, 64, 64, false);
                tc_gemm(tm, C_ZT, sW1, 64, B0, TT, 64, 128, 64, false);
                mma_commit(&bar);
            }
            mbar_wait(&bar, phase); phase ^= 1;
        }
        {   // plain epilogue only: H1 is all that layer 2 needs
            float v[16];
            acc_ld16(tm, lane_base + C_Z + c16, v);
#pragma unroll
            for (int i = 0; i < 16; ++i) v[i] = af(v[i] + sB1[c16 + i], c16 + i, af.w1);
            store_row16(B2, s_row, c16, TT, v);
        }
        fence_async_smem();
        __syncthreads();
        // ---- P2: Z2 (-> C_Z) and Z2^T (-> C_ZT2); warps 4-15 run the H1^T epilogue while warpgroup 0 computes them ----
        if (warpgroup_index() == 0) {
            tc_gemm(tm, C_Z, B2, TT, sW2, 64, 128, 64, 64, false);
            tc_gemm(tm, C_ZT2, sW2, 64, B2, TT, 64, 128, 64, false);
            mma_commit(&bar);
        }
        {   // deferred: H1^T = f(Z1^T + b1) -> B3 (B operand of dW2, needed only in P5)
            float w[32];
            acc_ld32(tm, lane_base + C_ZT + c32, w);
            if (lane < 16) {
                const float bb = sB1[t_row];
#pragma unroll
                for (int i = 0; i < 32; ++i) w[i] = af(w[i] + bb, t_row, af.w1);
                store_row32(B3, t_row, c32, 64, w);
            }
        }
        mbar_wait(&bar, phase); phase ^= 1;
        {
            float v[16];
            acc_ld16(tm, lane_base + C_Z + c16, v);
#pragma unroll
            for (int i = 0; i < 16; ++i) v[i] = af(v[i] + sB2[c16 + i], c16 + i, af.w2);
            store_row16(B0, s_row, c16, TT, v);                  // H2 (X is dead)
        }
        fence_async_smem();
        __syncthreads();
        // ---- P3: OUT -> loss -> dOUT (B4, cols 0..31) --------------------------------------------
        if (warpgroup_index() == 0) {
            tc_gemm(tm, C_OUT, B0, TT, sW3, 16, 128, 16, 64, false);
            mma_commit(&bar);
        }
        {   // deferred: H2^T = f(Z2^T + b2) -> B2 (H1 is dead: MMA3 / MMA3T completed)
            float w[32];
            acc_ld32(tm, lane_base + C_ZT2 + c32, w);
            if (lane < 16) {
                const float bb = sB2[t_row];
#pragma unroll
                for (int i = 0; i < 32; ++i) w[i] = af(w[i] + bb, t_row, af.w2);
                store_row32(B2, t_row, c32, 64, w);
            }
        }
        // per-sample scalars: issue the global loads before blocking on the MMA
        float pf_act[16], pf_logp = 0.f, pf_advr = 0.f, pf_advc = 0.f, pf_tv = 0.f;
        const long long prow = (h == 0) ? sRow[s_row] : -1;
        {
#pragma unroll
            for (int a = 0; a < 16; ++a) pf_act[a] = 0.f;
            if (prow >= 0) {
                if (net == 0) {
                    const float* src = (DMU || is_fvp) ? p.fvp_dmu : p.b.act;
#pragma unroll
                    for (int a = 0; a < 16; ++a)
                        if (a < A) pf_act[a] = __ldg(src + prow * A + a);
                    if (!DMU && !is_fvp) {
                        pf_logp = __ldg(p.b.logp + prow);
                        pf_advr = __ldg(p.b.adv_r + prow);
                        pf_advc = __ldg(p.b.adv_c + prow);
                    }
                } else {
                    pf_tv = __ldg((net == 1 ? p.b.tv_r : p.b.tv_c) + prow);
                }
            }
        }
        mbar_wait(&bar, phase); phase ^= 1;
        if (h == 0) {
            float st[5] = {0.f, 0.f, 0.f, 0.f, 0.f};   // loss, ratio, kl, count, focops mask
            float dls[16];
#pragma unroll
            for (int a = 0; a < 16; ++a) dls[a] = 0.f;
            float o16[16], d32[32];
            acc_ld16(tm, lane_base + C_OUT, o16);
#pragma unroll
            for (int i = 0; i < 32; ++i) d32[i] = 0.f;
            if (prow >= 0) {
                if (DMU && net != 0) {       // critic: the supplied dL/dV (tv_r / tv_c)
                    if (p.value_out) p.value_out[prow] = o16[0] + sB3[0];
                    d32[0] = pf_tv;
                    st[3] = 1.f;
                } else if (net != 0) {
                    const float d = o16[0] + sB3[0] - pf_tv;
                    st[0] = d * d; st[3] = 1.f;
                    d32[0] = 2.f * d * inv_b;
                } else if (DMU) {
#pragma unroll
                    for (int a = 0; a < 16; ++a)
                        if (a < A) d32[a] = pf_act[a];
                    st[3] = 1.f;
                } else if (is_fvp) {
                    // dOUT = diag(sigma^-2) J v / (rows * A): the backward below then yields J^T of it
#pragma unroll
                    for (int a = 0; a < 16; ++a)
                        if (a < A) {
                            const float sd = sPol[16 + a];
                            d32[a] = pf_act[a] / (sd * sd) * p.fvp_scale;
                        }
                    st[3] = 1.f;
                } else {
                    float mu[16];
#pragma unroll
                    for (int a = 0; a < 16; ++a) mu[a] = o16[a] + sB3[a];
                    actor_sample_loss<EXT, 16>(p.lc, an, A, inv_b, mu, pf_act,
                                                                    [&](int a) { return __ldg(p.lc.mu_old + prow * A + a); }, pf_logp, pf_advr,
                                                                    pf_advc, sPol, sOld, st,
                                                                    [&](int a, float dm, float dl) { d32[a] = dm; dls[a] = dl; });
                }
            }
            store_row32(B4, s_row, 0, TT, d32);
#pragma unroll
            for (int o = 0; o < 16; ++o) sts(tile_addr(B4 + 16384u, o, s_row, 16), tf32r(d32[o]));   // dOUT^T [o][s]
            // deterministic reductions over the 128 sample threads (warps with h == 0)
#pragma unroll
            for (int i = 0; i < 5; ++i) st[i] = warp_sum(st[i]);
            if (net == 0) {
#pragma unroll
                for (int a = 0; a < 16; ++a) dls[a] = warp_sum(dls[a]);
            }
            float db[16];   // db3[o] = sum_s dOUT[s][o]
#pragma unroll
            for (int a = 0; a < 16; ++a) db[a] = (a < L.out) ? warp_sum(d32[a]) : 0.f;
            if (lane == 0) {
#pragma unroll
                for (int i = 0; i < 5; ++i) sRed[q * 8 + i] = st[i];
#pragma unroll
                for (int a = 0; a < 16; ++a) { sRed[32 + q * 16 + a] = dls[a]; sRed[96 + q * 16 + a] = db[a]; }
            }
        }
        fence_async_smem();
        __syncthreads();
        if (tid < 5) sStat[tid] += sRed[tid] + sRed[8 + tid] + sRed[16 + tid] + sRed[24 + tid];
        if (net == 0 && tid >= 32 && tid < 48) {
            const int a = tid - 32;
            sDls[a] += sRed[32 + a] + sRed[48 + a] + sRed[64 + a] + sRed[80 + a];
        }
        if (tid >= 64 && tid < 64 + L.out) {
            const int a = tid - 64;
            sB3acc[a] += sRed[96 + a] + sRed[112 + a] + sRed[128 + a] + sRed[144 + a];
        }
        if (EXT && p.forward_only) {   // pass 1: statistics only
            if (CHUNKED) { if (has_next) load_chunk(sRowNext, 0); }
            else if (vec && has_next) prefetch_x(sRowNext);
            first_tile = false;
            rpar ^= 1;
            __syncthreads();
            continue;
        }
        // ---- P4: dZ2, dZ2^T and dW3^T += H2^T dOUT ------------------------------------------------
        if (warpgroup_index() == 0) {
            tc_gemm(tm, C_Z, B4, TT, sW3T, 64, 128, 64, 16, false);
            tc_gemm(tm, C_ZT, sW3T, 64, B4, TT, 64, 128, 16, false);
            tc_gemm(tm, C_DW3, B2, 64, B4 + 16384u, 16, 64, 16, 128, !first_tile);
            mma_commit(&bar);
        }
        mbar_wait(&bar, phase); phase ^= 1;
        {
            float w[32], hh[32];
            acc_ld32(tm, lane_base + C_ZT + c32, w);
            if (lane < 16) {
                load_row32(B2, t_row, c32, 64, hh);              // H2^T
#pragma unroll
                for (int i = 0; i < 32; ++i) w[i] *= af.d(hh[i]);
                store_row32(B4, t_row, c32, 64, w);              // dZ2^T [k][s]
            }
        }
        __syncthreads();           // every read of H2^T (B2) is done before dZ2 overwrites it
        {
            float v[16], hh[16];
            acc_ld16(tm, lane_base + C_Z + c16, v);
            load_row16(B0, s_row, c16, TT, hh);
#pragma unroll
            for (int i = 0; i < 16; ++i) v[i] *= af.d(hh[i]);
            store_row16(B2, s_row, c16, TT, v);                  // dZ2 [s][k]
        }
        fence_async_smem();
        __syncthreads();
        // ---- P5: dW2 += dZ2^T H1 ; dZ1^T = W2^T dZ2^T --------------------------------------------
        if (CHUNKED) load_chunk(sRow, 0);             // chunk 0 of THIS tile again: P6 needs X^T chunk by chunk
        else if (vec && has_next) prefetch_x(sRowNext);    // global loads of the next tile fly during P5 / P6
        if (warpgroup_index() == 0) {
            tc_gemm(tm, C_DW2, B4, 64, B3, 64, 64, 64, 128, !first_tile);
            tc_gemm(tm, C_ZT, sW2T, 64, B2, TT, 64, 128, 64, false);
            mma_commit(&bar);
        }
        if (tid < 64) {   // db2[j] = sum_s dZ2^T[j][s]
            float c = 0.f, v[32];
#pragma unroll 1
            for (int a4 = 0; a4 < 4; ++a4) {
                load_row32(B4, tid, 32 * a4, 64, v);
#pragma unroll
                for (int i = 0; i < 32; ++i) c += v[i];
            }
            ab2 += c;
        }
        mbar_wait(&bar, phase); phase ^= 1;
        {
            float w[32], hh[32];
            acc_ld32(tm, lane_base + C_ZT + c32, w);
            if (lane < 16) {
                load_row32(B3, t_row, c32, 64, hh);
#pragma unroll
                for (int i = 0; i < 32; ++i) w[i] *= af.d(hh[i]);
                store_row32(B0, t_row, c32, 64, w);              // dZ1^T [k][s] (H2 is dead)
            }
        }
        fence_async_smem();
        __syncthreads();
        // ---- P6: dW1 += dZ1^T X --------------------------------------------------------------------
        if (CHUNKED) {
            for (int c = 0; c < nchunks; ++c) {
                store_chunk(B1, true);               // X^T chunk [64 k][128 s]
                fence_async_smem();
                __syncthreads();                     // (c > 0) every read of the previous chunk's accumulator is done
                if (c + 1 < nchunks) load_chunk(sRow, c + 1);
                if (warpgroup_index() == 0) {
                    tc_gemm(tm, C_DW1, B0, 64, B1, 64, 64, 64, 128, false);
                    mma_commit(&bar);
                }
                if (c == 0 && tid < 64) {   // db1[j] = sum_s dZ1^T[j][s]
                    float cs = 0.f, v[32];
#pragma unroll 1
                    for (int a4 = 0; a4 < 4; ++a4) {
                        load_row32(B0, tid, 32 * a4, 64, v);
#pragma unroll
                        for (int i = 0; i < 32; ++i) cs += v[i];
                    }
                    ab1 += cs;
                }
                mbar_wait(&bar, phase); phase ^= 1;
                {   // flush this chunk of dW1 into the CTA's partial gradient (each element owned by one thread)
                    float v[16];
                    acc_ld16(tm, lane_base + C_DW1 + c16, v);
                    if (lane < 16) {
                        float* qrow = gout + L.off_w1 + t_row * O + c * 64 + c16;
                        const int nvalid = O - (c * 64 + c16);          // columns of this 16-group inside [0, O)
                        if (!first_tile) {                              // all loads first (independent), then the stores
                            float old[16];
#pragma unroll
                            for (int i = 0; i < 16; ++i) old[i] = (i < nvalid) ? __ldcg(qrow + i) : 0.f;
#pragma unroll
                            for (int i = 0; i < 16; ++i) v[i] += old[i];
                        }
#pragma unroll
                        for (int i = 0; i < 16; ++i)
                            if (i < nvalid) __stcg(qrow + i, v[i]);
                    }
                }
            }
            if (has_next) load_chunk(sRowNext, 0);
        } else {
        if (warpgroup_index() == 0) {
            tc_gemm(tm, C_DW1, B0, 64, B1, 64, 64, 64, 128, !first_tile);
            mma_commit(&bar);
        }
        if (tid < 64) {   // db1[j] = sum_s dZ1^T[j][s]
            float c = 0.f, v[32];
#pragma unroll 1
            for (int a4 = 0; a4 < 4; ++a4) {
                load_row32(B0, tid, 32 * a4, 64, v);
#pragma unroll
                for (int i = 0; i < 32; ++i) c += v[i];
            }
            ab1 += c;
        }
        mbar_wait(&bar, phase); phase ^= 1;      // B0 / B1 are rewritten by the next tile's gather
        }
        first_tile = false;
        rpar ^= 1;
        __syncthreads();
    }

    // ---- write this CTA's partial gradient segment (staged through smem so that stores coalesce) ----
    if (EXT && p.forward_only) {
        if (tid < 8) p.stats_part[((size_t)blockIdx.x * 3 + net) * 8 + tid] = sStat[tid];
    } else {
        float v[16];
        float* stage = reinterpret_cast<float*>(smem_raw + pad);            // B0 region: [2][64][65]
        acc_ld16(tm, lane_base + C_DW2 + c16, v);
        if (lane < 16)
#pragma unroll
            for (int i = 0; i < 16; ++i) stage[t_row * 65 + c16 + i] = v[i];
        if (!CHUNKED) {
            acc_ld16(tm, lane_base + C_DW1 + c16, v);
            if (lane < 16)
#pragma unroll
                for (int i = 0; i < 16; ++i) stage[64 * 65 + t_row * 65 + c16 + i] = v[i];
        }
        if (h == 0) {   // dW3^T [k][o] accumulator (M = 64 layout)
            acc_ld16(tm, lane_base + C_DW3, v);
            if (lane < 16)
#pragma unroll
                for (int o = 0; o < 16; ++o) stage[2 * 64 * 65 + o * 65 + t_row] = v[o];
        }
        __syncthreads();
        for (int i = tid; i < 64 * 64; i += NTC) gout[L.off_w2 + i] = stage[(i >> 6) * 65 + (i & 63)];
        if (!CHUNKED)
            for (int i = tid; i < 64 * O; i += NTC) gout[L.off_w1 + i] = stage[64 * 65 + (i / O) * 65 + (i % O)];
        for (int i = tid; i < L.out * 64; i += NTC) gout[L.off_w3 + i] = stage[2 * 64 * 65 + (i >> 6) * 65 + (i & 63)];
        if (tid < 64) { gout[L.off_b1 + tid] = ab1; gout[L.off_b2 + tid] = ab2; }
        if (tid < L.out) gout[L.off_b3 + tid] = sB3acc[tid];
        if (net == 0 && tid < A) {
            float g = sDls[tid];
            if (blockIdx.x == 0 && loss_has_entropy<EXT>(p.lc.kind)) g -= p.lc.entropy_coef / (float)A;
            // log_std block of the Fisher matrix: (2/A) v, counted once (natural_pg.py:L74-119, analytic form)
            if (is_fvp) g = (blockIdx.x == 0) ? 2.f / (float)A * __ldg(p.fvp_vec + L.off_logstd + tid) : 0.f;
            gout[L.off_logstd + tid] = g;
        }
        if (tid < 8)
            p.stats_part[((size_t)blockIdx.x * 3 + net) * 8 + tid] =
                (tid == 5 && net == 0) ? entropy_bonus_sum<EXT>(p.lc, A, sPol, sStat[3]) : sStat[tid];
    }
    __syncthreads();
}

}  // namespace osb

using namespace osb;

static size_t tc_smem_bytes() {
    return 1024 + 5 * (size_t)BUF + 3 * 16384 + 4096 + 8192 + (64 + 64 + 16 + 48 + 8 + 160 + 16 + 32 + 16) * 4 + 2 * 128 * 8 + 64;
}

static int launch_grad_tc(TcArgs& p, int nblocks, cudaStream_t stream) {
    const size_t smem = tc_smem_bytes();
    const bool single = (p.net_mask & (p.net_mask - 1)) == 0;     // one network: it gets every CTA
    dim3 grid(nblocks, single ? 1 : 3);
    p.acc = acc_scratch(ACC_UPDATE_TC, (size_t)grid.x * grid.y * 128 * TC_COLS * sizeof(float));
    if (!p.acc) return OSB_ERR_CUDA;
    const bool ext = loss_two_pass(p.lc.kind) || p.lc.kind == LOSS_FVP;
    const NetSpec spec = net_spec();
    return with_act<true>(launch_act(spec, p.net_mask), [&](auto a) {
        static bool attr = false;
        if (!attr) {
            OSB_CUDA(cudaFuncSetAttribute(minibatch_grad_tc_kernel<false, false, false, a.value>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            OSB_CUDA(cudaFuncSetAttribute(minibatch_grad_tc_kernel<false, true, false, a.value>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            OSB_CUDA(cudaFuncSetAttribute(minibatch_grad_tc_kernel<true, false, false, a.value>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            OSB_CUDA(cudaFuncSetAttribute(minibatch_grad_tc_kernel<true, true, false, a.value>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            attr = true;
        }
        if (p.O > 64) {
            if (ext) minibatch_grad_tc_kernel<true, true, false, a.value><<<grid, NTC, smem, stream>>>(p, spec);
            else minibatch_grad_tc_kernel<true, false, false, a.value><<<grid, NTC, smem, stream>>>(p, spec);
        } else {
            if (ext) minibatch_grad_tc_kernel<false, true, false, a.value><<<grid, NTC, smem, stream>>>(p, spec);
            else minibatch_grad_tc_kernel<false, false, false, a.value><<<grid, NTC, smem, stream>>>(p, spec);
        }
        OSB_LAUNCH_CHECK();
        return OSB_OK;
    });
}

extern "C" {

// CTAs along x of the tensor-core kernel: three networks share the SMs (a third each); a single
// network (full-batch actor passes of the natural-gradient family) spreads over all of them.
int osb_tc_grid_blocks(long long rows, int net_mask) {
    const long long tiles = (rows + TT - 1) / TT;
    const int cap = ((net_mask & (net_mask - 1)) == 0) ? grid_sms() : grid_sms() / 3;
    return (int)(tiles < cap ? tiles : cap);
}

// Tensor-core (TF32 wgmma) variant of osb_minibatch_grad: same arguments, O <= 512, A <= 16.
// gpart holds osb_tc_grid_blocks(mb_count, net_mask) rows of P floats.
int osb_minibatch_grad_tc(const float* theta, int O, int A, const float* obs, const float* act,
                          const float* logp, const float* adv_r, const float* adv_c,
                          const float* tv_r, const float* tv_c, const float* mu_old,
                          const float* moments, const int* perm, long long total, unsigned perm_seed,
                          long long mb_start, int mb_count, int loss_kind, float clip,
                          float entropy_coef, float focops_lam, float focops_eta,
                          const float* lagrange, const float* logstd_old, int net_mask, float* gpart,
                          float* stats_part, const int* stop_flag, void* stream) {
    OSB_CHECK_ARG(theta && obs && act && logp && adv_r && adv_c && tv_r && tv_c && moments, "null input");
    OSB_CHECK_ARG(O > 0 && O <= 512 && A > 0 && A <= 16 && mb_count > 0 && total > 0, "tensor-core path needs O <= 512, A <= 16");
    OSB_CHECK_ARG(mb_start >= 0 && mb_start + mb_count <= total, "minibatch window out of range");
    OSB_CHECK_ARG((loss_kind >= 0 && loss_kind <= 3) || loss_kind == LOSS_P3O, "loss kind");
    OSB_CHECK_ARG(loss_kind != LOSS_FOCOPS || (mu_old && logstd_old), "FOCOPS needs mu_old/logstd_old");
    OSB_CHECK_ARG(net_mask > 0 && net_mask < 8, "net_mask");
    TcArgs p;
    p.b = Batch{obs, act, logp, adv_r, adv_c, tv_r, tv_c, moments, perm, total, perm_seed, mb_start, mb_count, 0};
    p.lc = LossParams{loss_kind, clip, entropy_coef, focops_lam, focops_eta, lagrange, mu_old, logstd_old, nullptr};
    p.theta = theta; p.gpart = gpart; p.stats_part = stats_part; p.stop_flag = stop_flag;
    p.O = O; p.A = A; p.P = actor_layout(O, A).size + 2 * critic_layout(O, A).size; p.net_mask = net_mask;
    p.fvp_dmu = nullptr; p.fvp_vec = nullptr; p.fvp_scale = 0.f;
    p.forward_only = 0;
    const int nb = osb_tc_grid_blocks(mb_count, net_mask);
    if (loss_two_pass(loss_kind) && (net_mask & 1)) {   // pass 1: actor forward only
        TcArgs q = p;
        q.forward_only = 1; q.net_mask = 1;
        const int nb1 = osb_tc_grid_blocks(mb_count, 1);
        int rc = launch_grad_tc(q, nb1, (cudaStream_t)stream);
        if (rc) return rc;
        if ((rc = pass1_gate(stats_part, nb1, stop_flag, p.lc, (cudaStream_t)stream))) return rc;
    }
    return launch_grad_tc(p, nb, (cudaStream_t)stream);
}

}  // extern "C"

// LOSS_DMU launch of the DMU instantiations (one network, grid.y == 1) on nb CTAs
static int launch_dmu_tc(TcArgs& p, int nb, cudaStream_t stream) {
    p.lc = LossParams{LOSS_DMU, 0.f, 0.f, 1.f, 0.f, nullptr, nullptr, nullptr, nullptr};
    p.stop_flag = nullptr; p.fvp_vec = nullptr; p.fvp_scale = 1.f;
    p.forward_only = 0;
    const size_t smem = tc_smem_bytes();
    p.acc = acc_scratch(ACC_UPDATE_TC, (size_t)nb * 128 * TC_COLS * sizeof(float));
    if (!p.acc) return OSB_ERR_CUDA;
    const NetSpec spec = net_spec();
    return with_act<false>(launch_act(spec, p.net_mask), [&](auto a) {
        static bool attr = false;
        if (!attr) {
            OSB_CUDA(cudaFuncSetAttribute(minibatch_grad_tc_kernel<false, false, true, a.value>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            OSB_CUDA(cudaFuncSetAttribute(minibatch_grad_tc_kernel<true, false, true, a.value>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            attr = true;
        }
        if (p.O > 64) minibatch_grad_tc_kernel<true, false, true, a.value><<<dim3(nb, 1), NTC, smem, stream>>>(p, spec);
        else minibatch_grad_tc_kernel<false, false, true, a.value><<<dim3(nb, 1), NTC, smem, stream>>>(p, spec);
        OSB_LAUNCH_CHECK();
        return OSB_OK;
    });
}

int osb::dmu_backward_tc(const float* theta_actor, int O, int A, const float* obs, const float* dmu, int rows, float* gpart,
                         float* stats_scratch, cudaStream_t stream) {
    OSB_CHECK_ARG(O <= 512 && A <= 16, "tensor-core path needs O <= 512, A <= 16");
    TcArgs p;
    p.b = Batch{obs, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, rows, 0u, 0, rows, 1};
    p.theta = theta_actor; p.gpart = gpart; p.stats_part = stats_scratch;
    p.O = O; p.A = A; p.P = actor_layout(O, A).size; p.net_mask = 1;
    p.fvp_dmu = dmu; p.value_out = nullptr;
    return launch_dmu_tc(p, osb_tc_grid_blocks(rows, 1), stream);
}

int osb::fvp_backward_tc(const float* theta_actor, const float* vec, int O, int A, const float* obs, long long total,
                         int stride, const float* dmu, float* gpart, float* stats_scratch, cudaStream_t stream) {
    const long long nrows = (total + stride - 1) / stride;
    TcArgs p;
    p.b = Batch{obs, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, total, 0u, 0, (int)nrows, stride};
    p.lc = LossParams{LOSS_FVP, 0.f, 0.f, 1.f, 0.f, nullptr, nullptr, nullptr, nullptr};
    p.theta = theta_actor; p.gpart = gpart; p.stats_part = stats_scratch; p.stop_flag = nullptr;
    p.O = O; p.A = A; p.P = actor_layout(O, A).size; p.net_mask = 1;
    p.fvp_dmu = dmu; p.fvp_vec = vec; p.fvp_scale = 1.0f / ((float)nrows * (float)A);
    p.forward_only = 0;
    return launch_grad_tc(p, osb_tc_grid_blocks(nrows, 1), stream);
}

int osb::dv_backward_tc(const float* theta, int O, int A, int net, const float* obs, const float* dv, float* value, int rows,
                        float* gpart, float* stats_scratch, cudaStream_t stream) {
    OSB_CHECK_ARG(O <= 512 && A <= 16, "tensor-core path needs O <= 512, A <= 16");
    TcArgs p;
    p.b = Batch{obs, nullptr, nullptr, nullptr, nullptr, dv, dv, nullptr, nullptr, rows, 0u, 0, rows, 1};
    p.theta = theta; p.gpart = gpart; p.stats_part = stats_scratch;
    p.O = O; p.A = A; p.P = actor_layout(O, A).size + 2 * critic_layout(O, A).size; p.net_mask = 1 << net;
    p.fvp_dmu = nullptr; p.value_out = value;
    return launch_dmu_tc(p, osb_tc_grid_blocks(rows, 1 << net), stream);
}
