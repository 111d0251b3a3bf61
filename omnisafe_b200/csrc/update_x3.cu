// Parity-grade tensor-core variant of the fused minibatch forward + loss + backward kernel
// (PolicyGradient._update, algorithms/on_policy/base/policy_gradient.py:L345-524; PPO._loss_pi base/ppo.py:L35-87;
// PPOLag._compute_adv_surrogate naive_lagrange/ppo_lag.py:L82-102): split-bf16 arithmetic (csrc/x3.cuh), i.e.
// every GEMM is six bf16 wgmma MMAs over the three bf16 pieces of its fp32 operands with fp32
// accumulation in the accumulator image -- fp32-level results on the tensor cores (the reference computes fp32 Linear layers,
// omnisafe/utils/model.py:L105-111).
//
// One CTA = one network x a strided set of 128-sample tiles (same grid / per-CTA partial-gradient contract as
// minibatch_grad_tc_kernel).  Warp-specialised: 16 epilogue warps + 1 MMA-issue warp, linked by mbarriers only:
//
//   per tile (activations stored ONCE as [sample][feature] bf16x3 tiles; the weight-gradient GEMMs read the
//   same tiles MN-major, so there are no transposed copies):
//     Z1   = X  W1^T            -> H1 = tanh(. + b1)
//     Z2   = H1 W2^T            -> H2 = tanh(. + b2)
//     OUT  = H2 W3^T            -> per-sample loss, dOUT
//     dZ2' = dOUT W3            -> dZ2 = dZ2' (1 - H2^2)   (stored over H2)     | dW3^T += H2^T dOUT
//     dZ1' = dZ2 W2             -> dZ1 = dZ1' (1 - H1^2)   (stored over H1)     | dW2 += dZ2^T H1, db2 += dZ2^T 1
//                                                                               | dW1 += dZ1^T X,  db1 += dZ1^T 1
//   Every epilogue writes its activation in two column halves, each announced by its own mbarrier, so the
//   next layer's MMAs start on k-steps 0-1 while the epilogue still produces k-steps 2-3; weight / bias
//   gradient MMAs run behind the dependent chain while the epilogue warps work.  The loss warps' per-sample inputs
//   are copied asynchronously into shared memory (cp.async) at the start of the tile.
//
// FUSED instantiation = the persistent cooperative kernel of one update iteration: after each minibatch the partial
// gradients are reduced slice-wise behind a software grid barrier, clipped per network, (multi-rank) exchanged over
// NVLink as 8-byte {step tag, value} words, stepped with torch-Adam arithmetic -- speculatively before the norm barrier
// on one rank -- and the weight tiles come back with one TMA bulk copy of a pre-split bf16x3 image maintained by the
// Adam owners.  Loss kinds: PPO-clip, ratio, cost surrogate (fused or stepwise), FOCOPS and P3O (stepwise, with a
// forward-only statistics pass), supplied dOUT (Fisher-vector product backward).
#include "common.cuh"
#include "loss.cuh"
#include "mlp.cuh"
#include "x3.cuh"

namespace osb {

using namespace x3;

__device__ __forceinline__ void epi_bar_sync() { asm volatile("bar.sync 1, 512;\n" ::: "memory"); }      // epilogue warps only
__device__ __forceinline__ void loss_bar_sync() { asm volatile("bar.sync 2, 128;\n" ::: "memory"); }     // loss warps (h == 0)

struct X3Args {
    Batch b;
    LossParams lc;
    const float* theta;
    float* gpart;            // [gridDim.x][P]
    float* stats_part;       // [gridDim.x][3][8]
    const int* stop_flag;
    int O, A, P, net_mask;
    // ---- fused optimiser (persistent mode: one launch = one pass over [mb_start, mb_start + mb_count) in
    //      minibatches of batch_size, each followed by reduce + clip + (all-reduce) + Adam inside the kernel) ----
    int batch_size;
    float* theta_rw; float* grad; float* adam_m; float* adam_v; int* adam_step;
    float critic_norm_coef, max_grad_norm, lr[3];
    float* sumsq_part;           // [3][2][gridDim.x]
    float* train_stats;          // [3][8]
    unsigned int* bar_ctr;       // [3] per-network grid barrier counters, zero at launch
    float* const* peer_buf;      // [world] receive buffers, each [2][world][P] 8-byte words {step tag, value} (pushed over NVLink), or null
    unsigned int* const* peer_flag;   // [world] flag arrays, each [2 * world + 2 * world * 160]
    int world, rank;
    unsigned int step_base;      // exchange step id of this launch's first minibatch (identical on all ranks)
    int* error_flag;
    uint8_t* wimg;               // FUSED: [3 nets][W_IMG] bf16x3 images of the weight tiles (W1 | W2 | W3), written by the Adam owners,
                                 // pulled into shared memory with one bulk copy (TMA) after every optimiser step
    int forward_only;            // pass 1 of FOCOPS / P3O (stepwise launches only): statistics only
    const float* fvp_dmu;        // LOSS_FVP: tangent of mu per slab row [total][A] (fvp_tangent_x3_kernel)
    const float* fvp_vec;        // LOSS_FVP: direction v (its log_std block gives the log_std block of F v)
    float fvp_scale;             // LOSS_FVP: 1 / (rows * A)
    long long* dbg;              // optional clock64 stamps of CTA (0, 0): [0] = count, then (id, clock) pairs (tools/x3_stage_times.py)
    float* acc;                  // accumulator images, one [128][T_COLS] per CTA
};

constexpr int XT = 128;                      // samples per tile
constexpr int NEPI = 512;                    // 16 epilogue warps: lane quarter q = warp % 4, column group h = warp / 4
constexpr int NTX3 = NEPI + 128;             // + the MMA-issue warpgroup (warps 16..19)
constexpr uint32_t ACT_SUB = XT * 128, ACT_X3 = 3 * ACT_SUB;        // [128][64] bf16 sub-tile, x3 tile
constexpr uint32_t D_SUB = XT * 32, D_X3 = 3 * D_SUB;               // [128][16] bf16 (SW32)
constexpr uint32_t W_SUB = 64 * 128, W_X3 = 3 * W_SUB;              // [64][64]
constexpr uint32_t W3_SUB = 16 * 128, W3_X3 = 3 * W3_SUB;           // [16][64]
constexpr uint32_t W_IMG = 2 * W_X3 + W3_X3;                         // 55 296 B: the weight tiles W1 | W2 | W3 as they sit in shared memory
constexpr uint32_t OFF_X = 0, OFF_H1 = OFF_X + ACT_X3, OFF_H2 = OFF_H1 + ACT_X3, OFF_D = OFF_H2 + ACT_X3,
                   OFF_W1 = OFF_D + D_X3, OFF_W2 = OFF_W1 + W_X3, OFF_W3 = OFF_W2 + W_X3, OFF_ONES = OFF_W3 + W3_X3,
                   OFF_MISC = OFF_ONES + 512;
// misc region (floats unless noted)
constexpr int MF_B1 = 0, MF_B2 = 64, MF_B3 = 128, MF_LS = 144 /* logstd[16] sigma[16] dlogstd acc[16] */, MF_STAT = 192,
              MF_RED = 200 /* [4*8 + 4*16 + 4*16] */, MF_B3ACC = 360, MF_PART = 376 /* [2][256] */, MF_SCAL = 888 /* [16] */, MF_OLD = 904 /* log sigma_old[16], 1 / sigma_old^2 [16] */, MF_END = 936;
constexpr uint32_t OFF_ROWS = OFF_MISC + MF_END * 4;                 // long long [2][128]
constexpr uint32_t OFF_BARS = OFF_ROWS + 2 * XT * 8;                 // uint64 [NBAR]
enum Bar { RDY_X0 = 0, RDY_X1, RDY_H1_0, RDY_H1_1, RDY_H2_0, RDY_H2_1, RDY_D, RDY_DZ2_0, RDY_DZ2_1, RDY_DZ1,
           DONE_C1, DONE_C2, DONE_C3, DONE_C4A, DONE_C4B, DONE_C5A, DONE_C5B, DONE_C6, RDY_W, NBAR };
constexpr uint32_t OFF_PF = OFF_BARS + NBAR * 8 + 16;                       // float [128][12]: per-sample loss inputs (AP == 8), copied asynchronously
constexpr int PF_LD = 12;
constexpr uint32_t X3_SMEM = OFF_PF + XT * PF_LD * 4;
// accumulator columns
constexpr uint32_t T_ZA = 0, T_ZB = 64, T_OUT = 128, T_DW1 = 144, T_DW2 = 208, T_DW3 = 272, T_DB1 = 288, T_DB2 = 304, T_COLS = 320;

// fp32 parameters of one network -> bf16x3 weight tiles + fp32 biases in shared memory (all NEPI epilogue threads).
// All global loads are issued before the first store (one L2 round trip instead of one per loop iteration).
// O < 64 ("ones column"): column 63 of the X tile holds 1.0 and column 63 of the W1 tile holds b1, so the layer-1
// bias rides in the GEMM and db1 falls out of the dW1 accumulator (column 63) -- no bias add, no db1 MMAs.
__device__ __forceinline__ void stage_weights_x3(uint32_t sbase, float* misc, const float* __restrict__ theta,
                                                 const NetLayout& L, int net, int O, int A, int tid) {
    const bool ones_col = O < 64;
    float a1[4], b1[4], a2[4], b2[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {                          // W1 / W2: [64 n][64 k], two columns per thread
        const int i = tid + j * NEPI;
        const int n = i >> 5, k = (i & 31) << 1;
        a1[j] = (k < O) ? __ldcg(theta + L.off_w1 + n * O + k) : 0.f;
        b1[j] = (k + 1 < O) ? __ldcg(theta + L.off_w1 + n * O + k + 1) : ((ones_col && k == 62) ? __ldcg(theta + L.off_b1 + n) : 0.f);
        a2[j] = __ldcg(theta + L.off_w2 + n * 64 + k); b2[j] = __ldcg(theta + L.off_w2 + n * 64 + k + 1);
    }
    const int o3 = tid >> 5, k3 = (tid & 31) << 1;         // W3: [16 o][64 k], rows >= out zero
    const float a3 = (o3 < L.out) ? __ldcg(theta + L.off_w3 + o3 * 64 + k3) : 0.f;
    const float b3 = (o3 < L.out) ? __ldcg(theta + L.off_w3 + o3 * 64 + k3 + 1) : 0.f;
    float bb1 = 0.f, bb2 = 0.f, bb3 = 0.f, ls = 0.f;
    if (tid < 64) { bb1 = ones_col ? 0.f : __ldcg(theta + L.off_b1 + tid); bb2 = __ldcg(theta + L.off_b2 + tid); }
    if (tid < 16) {
        bb3 = (tid < L.out) ? __ldcg(theta + L.off_b3 + tid) : 0.f;
        ls = (net == 0 && tid < A) ? __ldcg(theta + L.off_logstd + tid) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int i = tid + j * NEPI;
        const int n = i >> 5, k = (i & 31) << 1;
        uint32_t w0, w1, w2;
        const uint32_t off = off128(n, k);
        split2(a1[j], b1[j], w0, w1, w2);
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sbase + OFF_W1 + off), "r"(w0) : "memory");
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sbase + OFF_W1 + W_SUB + off), "r"(w1) : "memory");
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sbase + OFF_W1 + 2 * W_SUB + off), "r"(w2) : "memory");
        split2(a2[j], b2[j], w0, w1, w2);
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sbase + OFF_W2 + off), "r"(w0) : "memory");
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sbase + OFF_W2 + W_SUB + off), "r"(w1) : "memory");
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sbase + OFF_W2 + 2 * W_SUB + off), "r"(w2) : "memory");
    }
    {
        uint32_t w0, w1, w2;
        split2(a3, b3, w0, w1, w2);
        const uint32_t off = off128(o3, k3);
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sbase + OFF_W3 + off), "r"(w0) : "memory");
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sbase + OFF_W3 + W3_SUB + off), "r"(w1) : "memory");
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sbase + OFF_W3 + 2 * W3_SUB + off), "r"(w2) : "memory");
    }
    if (tid < 64) { misc[MF_B1 + tid] = bb1; misc[MF_B2 + tid] = bb2; }
    if (tid < 16) {
        misc[MF_B3 + tid] = bb3;
        stage_policy(misc + MF_LS, tid, ls);
    }
}

__device__ __forceinline__ unsigned int ld_acquire_gpu_u32(const unsigned int* p) {
    unsigned int v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned int ld_acquire_sys_u32(const unsigned int* p) {
    unsigned int v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys_u32(unsigned int* p, unsigned int v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

constexpr int PSTR = 9472;          // FUSED: row stride of the private partial-gradient layout [3][G][PSTR] (16 B aligned rows)

// FUSED = false: one minibatch, per-CTA partial gradients out (the contract of minibatch_grad_tc_kernel).
// FUSED = true : persistent cooperative kernel -- the CTA loops over all minibatches of one update iteration
//   (policy_gradient.py:L369-381); after each minibatch the CTAs of a network meet at a software grid barrier,
//   reduce the partial gradients slice-wise in a fixed order, clip per network (clip_grad_norm_), exchange the
//   clipped slice with the peer ranks over NVLink (clip -> average -> step, policy_gradient.py:L437-443,
//   distributed.py:L193-198), apply torch-Adam and re-stage the new weights: no relaunch, no separate
//   optimiser kernel.
// AP = padded action width of the loss epilogue (8 or 16).
// (20 warps = 640 threads: 96 registers each, the register file divided in units of 8 per thread)
template <bool FUSED, int AP>
__global__ void __launch_bounds__(NTX3, 1) minibatch_grad_x3_kernel(X3Args p) {
    if (p.stop_flag && *p.stop_flag) return;
    const int net = (gridDim.y == 1) ? (__ffs(p.net_mask) - 1) : (int)blockIdx.y;
    if (!((p.net_mask >> net) & 1)) return;

    extern __shared__ __align__(16) uint8_t smem_raw[];
    const uint32_t pad = (1024u - (smem_u32(smem_raw) & 1023u)) & 1023u;
    const uint32_t sbase = smem_u32(smem_raw) + pad;
    uint8_t* gbase = smem_raw + pad;
    float* misc = reinterpret_cast<float*>(gbase + OFF_MISC);
    long long* sRowBuf = reinterpret_cast<long long*>(gbase + OFF_ROWS);
    const uint32_t bars = sbase + OFF_BARS;
    auto bar = [&](int i) { return bars + (uint32_t)i * 8u; };

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int O = p.O, A = p.A;
    const int G = (int)gridDim.x;
    const NetLayout L = net_layout(net, O, A);
    const int noff = net_offset(net, O, A);
    const float* theta = (FUSED ? p.theta_rw : p.theta) + noff;
    // partial gradients of this CTA: FUSED -> private aligned layout, else the [CTA][P] layout optim_fused reads
    float* gout = FUSED ? p.gpart + ((size_t)((gridDim.y == 1 ? 0 : net) * G + (int)blockIdx.x)) * PSTR
                        : p.gpart + (size_t)blockIdx.x * p.P + noff;
    const bool is_mma_warp = warp >= NEPI / 32;        // the four warps of the MMA-issue warpgroup
    const int batch = FUSED ? p.batch_size : p.b.mb_count;
    const int n_mb = (p.b.mb_count + batch - 1) / batch;
    const bool ones_col = O < 64;          // bias of layer 1 / db1 ride in the GEMMs (see stage_weights_x3)

    // ---- one-time setup -------------------------------------------------------------------------------
    if (!is_mma_warp) {
        stage_weights_x3(sbase, misc, theta, L, net, O, A, tid);
        if (tid < 128) reinterpret_cast<uint32_t*>(gbase + OFF_ONES)[tid] = 0x3F803F80u;       // bf16 1.0 x 256
        if (tid < 16 && (!FUSED && p.lc.kind == LOSS_FOCOPS))
            stage_policy_old(misc + MF_OLD, tid, (tid < A) ? __ldg(p.lc.logstd_old + tid) : 0.f);
    } else {
        if (tid == NEPI) {
            for (int i = 0; i < NBAR; ++i) {
                const uint32_t cnt = (i >= DONE_C1) ? 1u : (i == RDY_D ? 4u : 16u);      // (RDY_W: one expect_tx arrival)
                asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(bar(i)), "r"(cnt) : "memory");
            }
            mbar_init_fence();
        }
    }
    fence_async_smem();
    __syncthreads();
    const Acc tm = acc_cta(p.acc, T_COLS);

    if (is_mma_warp) {
        // ======================= MMA-issue warpgroup: uniform control flow ====================================
        const uint64_t dX = desc128(sbase + OFF_X), dH1 = desc128(sbase + OFF_H1), dH2 = desc128(sbase + OFF_H2);
        const uint64_t dD = desc32(sbase + OFF_D), dW1 = desc128(sbase + OFF_W1), dW2 = desc128(sbase + OFF_W2);
        const uint64_t dW3 = desc128(sbase + OFF_W3), dOnes = desc32(sbase + OFF_ONES);
        const uint32_t id_fwd = idesc_bf16(128, 64, 0, 0), id_out = idesc_bf16(128, 16, 0, 0), id_bwd = idesc_bf16(128, 64, 0, 1);
        const uint32_t id_dw = idesc_bf16(64, 64, 1, 1), id_dw16 = idesc_bf16(64, 16, 1, 1);
        int it = 0;
#pragma unroll 1
        for (int mb = 0; mb < n_mb; ++mb) {
            const int count = min(batch, p.b.mb_count - mb * batch);
            const int ntiles = (count + XT - 1) / XT;
#pragma unroll 1
            for (int tile = blockIdx.x; tile < ntiles; tile += G, ++it) {
                const uint32_t par = (uint32_t)(it & 1);
                const bool first = tile == (int)blockIdx.x;         // the first tile of a minibatch overwrites the accumulators
                const bool last = tile + G >= ntiles;
                // Z1 = X W1^T  (k-steps 0-1 after the first column half of X, 2-3 after the second)
#pragma unroll 1
                for (int ph = 0; ph < 2; ++ph) {
                    mbar_wait_a(bar(RDY_X0 + ph), par);
                    gemm_x3(tm, T_ZA, desc_add(dX, 64u * ph), ACT_SUB, 32u, desc_add(dW1, 64u * ph), W_SUB, 32u, id_fwd, 2, ph > 0);
                }
                mma_commit_a(bar(DONE_C1));
                // db2 of the PREVIOUS tile (dZ2 still sits in the H2 buffer until this tile's E2): runs under E1,
                // completes before Z2 (in-order pipe), so DONE_C2 covers it
                if (!first && !(!FUSED && p.forward_only)) gemm_x3(tm, T_DB2, dH2, ACT_SUB, 2048u, dOnes, 0u, 0u, id_dw16, 8, tile != (int)blockIdx.x + G);
                // Z2 = H1 W2^T
#pragma unroll 1
                for (int ph = 0; ph < 2; ++ph) {
                    mbar_wait_a(bar(RDY_H1_0 + ph), par);
                    gemm_x3(tm, T_ZB, desc_add(dH1, 64u * ph), ACT_SUB, 32u, desc_add(dW2, 64u * ph), W_SUB, 32u, id_fwd, 2, ph > 0);
                }
                mma_commit_a(bar(DONE_C2));
                // OUT = H2 W3^T
#pragma unroll 1
                for (int ph = 0; ph < 2; ++ph) {
                    mbar_wait_a(bar(RDY_H2_0 + ph), par);
                    gemm_x3(tm, T_OUT, desc_add(dH2, 64u * ph), ACT_SUB, 32u, desc_add(dW3, 64u * ph), W3_SUB, 32u, id_out, 2, ph > 0);
                }
                mma_commit_a(bar(DONE_C3));
                if (!FUSED && p.forward_only) continue;              // statistics pass (FOCOPS mask mean): no backward
                // dZ2' = dOUT W3 ; dW3^T += H2^T dOUT
                mbar_wait_a(bar(RDY_D), par);
                gemm_x3(tm, T_ZA, dD, D_SUB, 32u, dW3, W3_SUB, 2048u, id_bwd, 1, false);
                mma_commit_a(bar(DONE_C4A));
                gemm_x3(tm, T_DW3, dH2, ACT_SUB, 2048u, dD, D_SUB, 512u, id_dw16, 8, !first);
                mma_commit_a(bar(DONE_C4B));
                // dZ1' = dZ2 W2 ; dW2 += dZ2^T H1
#pragma unroll 1
                for (int ph = 0; ph < 2; ++ph) {
                    mbar_wait_a(bar(RDY_DZ2_0 + ph), par);
                    gemm_x3(tm, T_ZB, desc_add(dH2, 64u * ph), ACT_SUB, 32u, desc_add(dW2, 4096u * ph), W_SUB, 2048u, id_bwd, 2, ph > 0);
                }
                mma_commit_a(bar(DONE_C5A));
                gemm_x3(tm, T_DW2, dH2, ACT_SUB, 2048u, dH1, ACT_SUB, 2048u, id_dw, 8, !first);
                mma_commit_a(bar(DONE_C5B));
                // dW1 += dZ1^T X (column 63 = db1 with the ones column) ; last tile of the minibatch: its own db2
                mbar_wait_a(bar(RDY_DZ1), par);
                gemm_x3(tm, T_DW1, dH1, ACT_SUB, 2048u, dX, ACT_SUB, 2048u, id_dw, 8, !first);
                if (!ones_col) gemm_x3(tm, T_DB1, dH1, ACT_SUB, 2048u, dOnes, 0u, 0u, id_dw16, 8, !first);
                if (last) gemm_x3(tm, T_DB2, dH2, ACT_SUB, 2048u, dOnes, 0u, 0u, id_dw16, 8, !first);
                mma_commit_a(bar(DONE_C6));
            }
        }
    } else {
        // ======================= epilogue warps ===============================================================
        const int q = warp & 3, h = warp >> 2;
        const uint32_t lane_base = (uint32_t)(q * 32) << 16;
        const int s_row = 32 * q + lane;                 // sample row of this thread in the [s][.] accumulators
        const AdvNorm an = adv_norm(p.b.moments, p.lc.lagrange);
        float* sB1 = misc + MF_B1; float* sB2 = misc + MF_B2; float* sB3 = misc + MF_B3; float* sLs = misc + MF_LS;
        float* sRed = misc + MF_RED; float* sPart = misc + MF_PART; float* sScal = misc + MF_SCAL;

        // X gather: thread -> row xm = tid / 4, columns 32 ph + 8 (tid % 4) .. + 7 in column half ph
        const int xm = tid >> 2, xc = (tid & 3) << 3;
        const bool vec = (O & 3) == 0;
        float xpre[16];
        auto prefetch_x = [&](const long long* rows) {
            const long long row = rows[xm];
#pragma unroll
            for (int ph = 0; ph < 2; ++ph) {
                const int c0 = 32 * ph + xc;
                if (vec) {
#pragma unroll
                    for (int v4 = 0; v4 < 2; ++v4) {
                        const int c = c0 + 4 * v4;
                        const float4 v = (row >= 0 && c < O) ? __ldg(reinterpret_cast<const float4*>(p.b.obs + row * O + c))
                                                             : make_float4(0.f, 0.f, 0.f, 0.f);
                        xpre[8 * ph + 4 * v4] = v.x; xpre[8 * ph + 4 * v4 + 1] = v.y; xpre[8 * ph + 4 * v4 + 2] = v.z; xpre[8 * ph + 4 * v4 + 3] = v.w;
                    }
                } else {
#pragma unroll
                    for (int i = 0; i < 8; ++i) xpre[8 * ph + i] = (row >= 0 && c0 + i < O) ? __ldg(p.b.obs + row * O + c0 + i) : 0.f;
                }
            }
            if (ones_col && xc == 24) xpre[15] = 1.0f;     // column 63: the ones column (every row: padding rows have dZ1 = 0)
        };
        auto announce = [&](int b) {        // this warp's stores of one column half are visible to the tensor core
            fence_async_smem();
            __syncwarp();
            if (lane == 0) mbar_arrive(bar(b));
        };
        const bool dbg_on = p.dbg != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && (tid == 0 || tid == 256);
        int dbg_n = 0;
        auto stamp = [&](int id) {
            if (dbg_on && dbg_n < 400) {
                long long* d = p.dbg + (tid == 0 ? 0 : 1024);
                d[1 + 2 * dbg_n] = id; d[2 + 2 * dbg_n] = clock64(); ++dbg_n; d[0] = dbg_n;
            }
        };
        unsigned int nbar = 0;              // software grid barriers passed so far (FUSED)
        auto net_barrier = [&]() {          // all CTAs of this network: writes before it are visible after it (via L2)
            epi_bar_sync();                  // the CTA's writes happen-before thread 0's release (cumulative at gpu scope)
            if (tid == 0) {
                asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p.bar_ctr + net), "r"(1u) : "memory");
                const unsigned int target = (unsigned int)G * (nbar + 1u);
                while (ld_acquire_gpu_u32(p.bar_ctr + net) < target) {}
            }
            ++nbar;
            epi_bar_sync();
        };
        auto mb_geom = [&](int mb, long long& start, int& count) {
            start = p.b.mb_start + (long long)mb * batch;
            count = min(batch, p.b.mb_count - mb * batch);
        };
        auto tile_rows = [&](int mb, int tile, long long* dst) {
            if (tid < XT) {
                long long start; int count;
                mb_geom(mb, start, count);
                const int local = tile * XT + tid;
                dst[tid] = (local < count) ? sample_row(p.b, start + local) : -1;
            }
        };
        int step_t0 = 0;
        if (FUSED) step_t0 = p.adam_step[net];
        // FUSED: where this thread's parameter (the first of its slice chunk) lives inside the weight-tile image, or -1
        // (log_std, b2, b3, and b1 when it is not folded into W1): byte offset of the hi piece, stride between pieces
        int img_off = -1; uint32_t img_sub = 0;
        if (FUSED) {
            const int Sx = (L.size + G - 1) / G, px = (int)blockIdx.x * Sx + tid;
            if (tid < Sx && px < L.size) {
                if (px >= L.off_w1 && px < L.off_b1) { const int e = px - L.off_w1; img_off = (int)off128(e / O, e % O); img_sub = W_SUB; }
                else if (px >= L.off_b1 && px < L.off_w2) { if (ones_col) { img_off = (int)off128(px - L.off_b1, 63); img_sub = W_SUB; } }
                else if (px >= L.off_w2 && px < L.off_b2) { const int e = px - L.off_w2; img_off = (int)(W_X3 + off128(e >> 6, e & 63)); img_sub = W_SUB; }
                else if (px >= L.off_w3 && px < L.off_b3) { const int e = px - L.off_w3; img_off = (int)(2 * W_X3 + off128(e >> 6, e & 63)); img_sub = W3_SUB; }
            }
        }
        uint8_t* wimg = FUSED ? p.wimg + (size_t)net * W_IMG : nullptr;
        // per-thread partial sums of the loss warps over the tiles of one minibatch (reduced once per minibatch)
        float acc_st[5] = {0.f, 0.f, 0.f, 0.f, 0.f}, acc_dls[AP], acc_db[AP];      // loss, ratio, kl, count, FOCOPS mask
#pragma unroll
        for (int a = 0; a < AP; ++a) { acc_dls[a] = 0.f; acc_db[a] = 0.f; }

        int rpar = 0, it = 0;
        if ((int)blockIdx.x < (min(batch, p.b.mb_count) + XT - 1) / XT) {     // rows + X of the first tile
            tile_rows(0, blockIdx.x, sRowBuf);
            epi_bar_sync();
            prefetch_x(sRowBuf);
        }
#pragma unroll 1
        for (int mb = 0; mb < n_mb; ++mb) {
            long long mb_start; int count;
            mb_geom(mb, mb_start, count);
            const int ntiles = (count + XT - 1) / XT;
            const float inv_b = 1.0f / (float)count;
            const bool have_tiles = (int)blockIdx.x < ntiles;
            if (FUSED && tid == NEPI - 1) {        // Adam bias corrections of this minibatch's step, off the critical path
                const int step_t = step_t0 + mb + 1;
                const double bc1 = 1.0 - pow(0.9, (double)step_t), bc2 = 1.0 - pow(0.999, (double)step_t);
                sScal[8] = (float)((double)p.lr[net] / bc1);
                sScal[9] = (float)sqrt(bc2);
            }
#pragma unroll 1
            for (int tile = blockIdx.x; tile < ntiles; tile += G, ++it) {
                const uint32_t par = (uint32_t)(it & 1);
                long long* sRow = sRowBuf + rpar * XT;
                long long* sRowNext = sRowBuf + (rpar ^ 1) * XT;
                const bool has_next = tile + G < ntiles;
                // ---- E0: X tile (prefetched registers -> bf16x3) ------------------------------------------------
                stamp(0);
                if (has_next) tile_rows(mb, tile + G, sRowNext);
                if (it > 0 && !(!FUSED && p.forward_only)) mbar_wait_a(bar(DONE_C6), par ^ 1u);   // previous tile's dW1 / db1 read X and dZ1
                stamp(1);
#pragma unroll
                for (int ph = 0; ph < 2; ++ph) {
                    float v[8];
#pragma unroll
                    for (int i = 0; i < 8; ++i) v[i] = xpre[8 * ph + i];
                    store8_x3(sbase + OFF_X, ACT_SUB, xm, 32 * ph + xc, v);
                    announce(RDY_X0 + ph);
                }
                epi_bar_sync();                                            // next tile's row list is complete
                stamp(2);
                // loss warps: this tile's per-sample inputs (used in E3) fly under the forward phases -- asynchronously into
                // shared memory when they fit (AP == 8), so that no register has to wait for them
                float pf_act[AP], pf_logp = 0.f, pf_advr = 0.f, pf_advc = 0.f, pf_tv = 0.f;
                long long prow = -1;
                if (h == 0) {
                    prow = sRow[s_row];
#pragma unroll
                    for (int a = 0; a < AP; ++a) pf_act[a] = 0.f;
                    if (prow >= 0) {
                        const float* asrc = (p.lc.kind == LOSS_FVP) ? p.fvp_dmu : p.b.act;
                        if (AP == 8) {
                            const uint32_t dst = sbase + OFF_PF + (uint32_t)(s_row * PF_LD) * 4u;
                            auto cp4 = [&](uint32_t d, const float* src) {
                                asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(d), "l"(src) : "memory");
                            };
                            if (net == 0) {
#pragma unroll
                                for (int a = 0; a < AP; ++a)
                                    if (a < A) cp4(dst + 4u * a, asrc + prow * A + a);
                                if (p.lc.kind != LOSS_FVP) { cp4(dst + 32u, p.b.logp + prow); cp4(dst + 36u, p.b.adv_r + prow); cp4(dst + 40u, p.b.adv_c + prow); }
                            } else {
                                cp4(dst + 32u, (net == 1 ? p.b.tv_r : p.b.tv_c) + prow);
                            }
                        } else if (net == 0) {
#pragma unroll
                            for (int a = 0; a < AP; ++a)
                                if (a < A) pf_act[a] = __ldg(asrc + prow * A + a);
                            if (p.lc.kind != LOSS_FVP) { pf_logp = __ldg(p.b.logp + prow); pf_advr = __ldg(p.b.adv_r + prow); pf_advc = __ldg(p.b.adv_c + prow); }
                        } else {
                            pf_tv = __ldg((net == 1 ? p.b.tv_r : p.b.tv_c) + prow);
                        }
                    }
                }
                // ---- E1: H1 = tanh(Z1 + b1) -------------------------------------------------------------------
                mbar_wait_a(bar(DONE_C1), par);
                stamp(3);
#pragma unroll
                for (int ph = 0; ph < 2; ++ph) {
                    const int c0 = 32 * ph + 8 * h;
                    float v[8];
                    acc_ld8(tm, lane_base + T_ZA + (uint32_t)c0, v);
#pragma unroll
                    for (int i = 0; i < 8; ++i) v[i] = tanh_acc(v[i] + sB1[c0 + i]);
                    store8_x3(sbase + OFF_H1, ACT_SUB, s_row, c0, v);
                    announce(RDY_H1_0 + ph);
                }
                // ---- E2: H2 = tanh(Z2 + b2) -------------------------------------------------------------------
                stamp(4);
                mbar_wait_a(bar(DONE_C2), par);
                stamp(5);
#pragma unroll
                for (int ph = 0; ph < 2; ++ph) {
                    const int c0 = 32 * ph + 8 * h;
                    float v[8];
                    acc_ld8(tm, lane_base + T_ZB + (uint32_t)c0, v);
#pragma unroll
                    for (int i = 0; i < 8; ++i) v[i] = tanh_acc(v[i] + sB2[c0 + i]);
                    store8_x3(sbase + OFF_H2, ACT_SUB, s_row, c0, v);
                    announce(RDY_H2_0 + ph);
                }
                stamp(6);
                // ---- E3: OUT -> loss -> dOUT (warps with h == 0: one thread per sample) -------------------------
                if (h == 0) {
                    if (AP == 8) {
                        asm volatile("cp.async.wait_all;\n" ::: "memory");
                        const float* pf = reinterpret_cast<const float*>(gbase + OFF_PF) + s_row * PF_LD;
                        if (prow >= 0) {
                            if (net == 0) {
#pragma unroll
                                for (int a = 0; a < AP; ++a)
                                    if (a < A) pf_act[a] = pf[a];
                                pf_logp = pf[8]; pf_advr = pf[9]; pf_advc = pf[10];
                            } else {
                                pf_tv = pf[8];
                            }
                        }
                    }
                    mbar_wait_a(bar(DONE_C3), par);
                    stamp(7);
                    float o[AP], d16[16];
#pragma unroll
                    for (int a = 0; a < 16; ++a) d16[a] = 0.f;
                    if (AP == 8) {
                        float t8[8];
                        acc_ld8(tm, lane_base + T_OUT, t8);
#pragma unroll
                        for (int a = 0; a < AP; ++a) o[a] = t8[a];
                    } else {
                        float t16[16];
                        acc_ld16(tm, lane_base + T_OUT, t16);
#pragma unroll
                        for (int a = 0; a < AP; ++a) o[a] = t16[a];
                    }
                    if (prow >= 0) {
                        if (net != 0) {
                            const float d = o[0] + sB3[0] - pf_tv;
                            acc_st[0] += d * d; acc_st[3] += 1.f;
                            d16[0] = 2.f * d * inv_b;
                            acc_db[0] += d16[0];
                        } else if (p.lc.kind == LOSS_FVP) {
                            // J^T diag(sigma^-2) dmu / (B A): the supplied tangent is the output gradient
                            acc_st[3] += 1.f;
#pragma unroll
                            for (int a = 0; a < AP; ++a)
                                if (a < A) {
                                    const float dm = pf_act[a] * sLs[32 + a] * p.fvp_scale;
                                    d16[a] = dm;
                                    acc_db[a] += dm;
                                }
                        } else {
                            float mu[AP];
#pragma unroll
                            for (int a = 0; a < AP; ++a) mu[a] = o[a] + sB3[a];
                            actor_sample_loss<!FUSED, AP>(p.lc, an, A, inv_b, mu, pf_act,
                                                                               [&](int a) { return __ldg(p.lc.mu_old + prow * A + a); },
                                                                               pf_logp, pf_advr, pf_advc, sLs, misc + MF_OLD, acc_st,
                                                                               [&](int a, float dm, float dl) {
                                                                                   d16[a] = dm; acc_db[a] += dm; acc_dls[a] += dl;
                                                                               });
                        }
                    }
                    store16_x3_sw32(sbase + OFF_D, D_SUB, s_row, d16);
                    announce(RDY_D);
                    stamp(8);
                }
                stamp(9);
                if (!FUSED && p.forward_only) {                                      // statistics pass: no backward; H2 is free once OUT is done
                    if (has_next) prefetch_x(sRowNext);
                    if (h != 0) { mbar_wait_a(bar(DONE_C3), par); }
                    rpar ^= 1;
                    continue;
                }
                // ---- E4: dZ2 = (dOUT W3) (1 - H2^2), stored over H2 once dW3 has read it --------------------------
                if (has_next) prefetch_x(sRowNext);                        // next tile's rows fly during the backward half
                mbar_wait_a(bar(DONE_C4A), par);
                stamp(10);
                float dz[16];
#pragma unroll
                for (int ph = 0; ph < 2; ++ph) {
                    const int c0 = 32 * ph + 8 * h;
                    float v[8], hh[8];
                    acc_ld8(tm, lane_base + T_ZA + (uint32_t)c0, v);
                    load8_x3(sbase + OFF_H2, ACT_SUB, s_row, c0, hh);
#pragma unroll
                    for (int i = 0; i < 8; ++i) dz[8 * ph + i] = v[i] * (1.f - hh[i] * hh[i]);
                }
                stamp(11);
                mbar_wait_a(bar(DONE_C4B), par);
                stamp(12);
#pragma unroll
                for (int ph = 0; ph < 2; ++ph) {
                    float v[8];
#pragma unroll
                    for (int i = 0; i < 8; ++i) v[i] = dz[8 * ph + i];
                    store8_x3(sbase + OFF_H2, ACT_SUB, s_row, 32 * ph + 8 * h, v);
                    announce(RDY_DZ2_0 + ph);
                }
                // ---- E5: dZ1 = (dZ2 W2) (1 - H1^2), stored over H1 once dW2 has read it --------------------------
                stamp(13);
                mbar_wait_a(bar(DONE_C5A), par);
                stamp(14);
#pragma unroll
                for (int ph = 0; ph < 2; ++ph) {
                    const int c0 = 32 * ph + 8 * h;
                    float v[8], hh[8];
                    acc_ld8(tm, lane_base + T_ZB + (uint32_t)c0, v);
                    load8_x3(sbase + OFF_H1, ACT_SUB, s_row, c0, hh);
#pragma unroll
                    for (int i = 0; i < 8; ++i) dz[8 * ph + i] = v[i] * (1.f - hh[i] * hh[i]);
                }
                stamp(15);
                mbar_wait_a(bar(DONE_C5B), par);
                stamp(16);
#pragma unroll
                for (int ph = 0; ph < 2; ++ph) {
                    float v[8];
#pragma unroll
                    for (int i = 0; i < 8; ++i) v[i] = dz[8 * ph + i];
                    store8_x3(sbase + OFF_H1, ACT_SUB, s_row, 32 * ph + 8 * h, v);
                }
                announce(RDY_DZ1);
                stamp(17);
                rpar ^= 1;
            }
            stamp(20);
            // ---- rows + X of the first tile of the NEXT minibatch: the gather flies under the optimiser phases ------
            if (FUSED && mb + 1 < n_mb) {
                long long s2; int c2;
                mb_geom(mb + 1, s2, c2);
                if ((int)blockIdx.x < (c2 + XT - 1) / XT) {
                    tile_rows(mb + 1, blockIdx.x, sRowBuf + rpar * XT);
                    epi_bar_sync();
                    prefetch_x(sRowBuf + rpar * XT);
                }
            }
            // ---- this CTA's partial gradient of the minibatch: accumulator images -> global ------------------------
            if (have_tiles) {
                // loss-warp sums: lanes -> warp (butterfly) -> the four loss warps (fixed order)
                if (h == 0) {
#pragma unroll
                    for (int i = 0; i < 5; ++i) acc_st[i] = warp_sum(acc_st[i]);
#pragma unroll
                    for (int a = 0; a < AP; ++a) { acc_dls[a] = warp_sum(acc_dls[a]); acc_db[a] = warp_sum(acc_db[a]); }
                    if (lane == 0) {
#pragma unroll
                        for (int i = 0; i < 5; ++i) sRed[q * 8 + i] = acc_st[i];
#pragma unroll
                        for (int a = 0; a < AP; ++a) { sRed[32 + q * 16 + a] = acc_dls[a]; sRed[96 + q * 16 + a] = acc_db[a]; }
                    }
#pragma unroll
                    for (int i = 0; i < 5; ++i) acc_st[i] = 0.f;
#pragma unroll
                    for (int a = 0; a < AP; ++a) { acc_dls[a] = 0.f; acc_db[a] = 0.f; }
                }
                if (!FUSED && p.forward_only) {
                    epi_bar_sync();                    // sRed of the four loss warps
                    if (tid >= 64 && tid < 72) {
                        const int i = tid - 64;
                        __stcg(p.stats_part + ((size_t)blockIdx.x * 3 + net) * 8 + i, (i < 5) ? (sRed[i] + sRed[8 + i]) + (sRed[16 + i] + sRed[24 + i]) : 0.f);
                    }
                    break;
                }
                mbar_wait_a(bar(DONE_C6), (uint32_t)((it - 1) & 1));
                stamp(21);
                const int t_row = 16 * q + lane;       // row (lane < 16) of the M = 64 accumulators
                const int c16 = 16 * h;
                float v[16];
                acc_ld16(tm, lane_base + T_DW2 + (uint32_t)c16, v);
                if (lane < 16) {
                    float* dst = gout + L.off_w2 + t_row * 64 + c16;
                    if (FUSED && (L.off_w2 & 3) == 0) {
#pragma unroll
                        for (int i = 0; i < 16; i += 4) __stcg(reinterpret_cast<float4*>(dst + i), make_float4(v[i], v[i + 1], v[i + 2], v[i + 3]));
                    } else {
#pragma unroll
                        for (int i = 0; i < 16; ++i) __stcg(dst + i, v[i]);
                    }
                }
                acc_ld16(tm, lane_base + T_DW1 + (uint32_t)c16, v);
                if (lane < 16) {
                    float* dst = gout + L.off_w1 + t_row * O + c16;
                    if (FUSED && ((L.off_w1 | O) & 3) == 0) {
#pragma unroll
                        for (int i = 0; i < 16; i += 4)
                            if (c16 + i < O) __stcg(reinterpret_cast<float4*>(dst + i), make_float4(v[i], v[i + 1], v[i + 2], v[i + 3]));
                    } else {
#pragma unroll
                        for (int i = 0; i < 16; ++i)
                            if (c16 + i < O) __stcg(dst + i, v[i]);
                    }
                    if (ones_col && h == 3) __stcg(gout + L.off_b1 + t_row, v[15]);        // column 63 of dW1 = db1
                }
                if (h == 0) {      // dW3^T [k][o]
                    acc_ld16(tm, lane_base + T_DW3, v);
                    if (lane < 16)
#pragma unroll
                        for (int o = 0; o < 16; ++o)
                            if (o < L.out) __stcg(gout + L.off_w3 + o * 64 + t_row, v[o]);
                } else if (h == 1) {
                    if (!ones_col) {
                        acc_ld16(tm, lane_base + T_DB1, v);
                        if (lane < 16) __stcg(gout + L.off_b1 + t_row, v[0]);
                    }
                } else if (h == 2) {
                    acc_ld16(tm, lane_base + T_DB2, v);
                    if (lane < 16) __stcg(gout + L.off_b2 + t_row, v[0]);
                }
                epi_bar_sync();                        // sRed of the four loss warps
                if (tid < L.out) __stcg(gout + L.off_b3 + tid, (sRed[96 + tid] + sRed[112 + tid]) + (sRed[128 + tid] + sRed[144 + tid]));
                if (net == 0 && tid >= 32 && tid < 32 + A) {
                    const int a = tid - 32;
                    float g = (sRed[32 + a] + sRed[48 + a]) + (sRed[64 + a] + sRed[80 + a]);
                    if (blockIdx.x == 0 && loss_has_entropy<!FUSED>(p.lc.kind)) g -= p.lc.entropy_coef / (float)A;
                    if (p.lc.kind == LOSS_FVP) g = (blockIdx.x == 0) ? 2.f / (float)A * __ldg(p.fvp_vec + L.off_logstd + a) : 0.f;
                    __stcg(gout + L.off_logstd + a, g);
                }
                if (tid >= 64 && tid < 72) {
                    const int i = tid - 64;
                    __stcg(p.stats_part + ((size_t)blockIdx.x * 3 + net) * 8 + i, (i < 5) ? (sRed[i] + sRed[8 + i]) + (sRed[16 + i] + sRed[24 + i]) : 0.f);
                }
            } else {
                for (int i = tid; i < L.size; i += NEPI) __stcg(gout + i, 0.f);      // no tile of this (short) minibatch
                if (tid < 8) __stcg(p.stats_part + ((size_t)blockIdx.x * 3 + net) * 8 + tid, 0.f);
            }
            stamp(22);
            if (!FUSED) break;

            // ================= in-kernel optimiser step =========================================================
            net_barrier();                                             // every partial gradient of this network is in L2
            stamp(23);
            const int S = (L.size + G - 1) / G;                        // parameters owned by this CTA: [p0, p0 + S)
            const int p0 = (int)blockIdx.x * S;
            const int Gh = (G + 1) >> 1;
            const float* gnet = p.gpart + (size_t)((gridDim.y == 1 ? 0 : net) * G) * PSTR;
            float ssq = 0.f, st2 = 0.f;
            for (int base = 0; base < S; base += 256) {
                const int pi = base + (tid & 255), part = tid >> 8;
                const bool valid = pi < S && p0 + pi < L.size;
                float sacc = 0.f;
                if (valid) {
                    const float* src = gnet + p0 + pi;
                    const int b1 = min(G, (part + 1) * Gh);
                    for (int b = part * Gh; b < b1; b += 32) {       // 32 partial rows in flight per thread
                        float t[32];
#pragma unroll
                        for (int u = 0; u < 32; ++u) t[u] = (b + u < b1) ? __ldcg(src + (size_t)(b + u) * PSTR) : 0.f;
#pragma unroll
                        for (int w = 16; w > 0; w >>= 1)
#pragma unroll
                            for (int u = 0; u < w; ++u) t[u] += t[u + w];
                        sacc += t[0];
                    }
                }
                sPart[tid] = sacc;
                epi_bar_sync();
                if (part == 0 && valid) {
                    const int qg = noff + p0 + pi;
                    float g = sPart[tid] + sPart[256 + tid];
                    if (net != 0 && p.critic_norm_coef > 0.f) {
                        const float th = __ldcg(p.theta_rw + qg);
                        g += 2.f * p.critic_norm_coef * th; st2 += th * th;
                    }
                    __stcg(p.grad + qg, g);
                    ssq += g * g;
                }
                epi_bar_sync();
            }
            ssq = warp_sum(ssq); st2 = warp_sum(st2);
            if (lane == 0) { sPart[warp] = ssq; sPart[16 + warp] = st2; }
            epi_bar_sync();
            if (tid == 0) {
                float a = 0.f, b = 0.f;
                for (int w = 0; w < 16; ++w) { a += sPart[w]; b += sPart[16 + w]; }
                __stcg(p.sumsq_part + (net * 2 + 0) * G + blockIdx.x, a);
                __stcg(p.sumsq_part + (net * 2 + 1) * G + blockIdx.x, b);
            }
            // Adam state of this thread's parameter: loaded before the barrier, consumed after it
            const bool own = tid < S && p0 + tid < L.size;
            float pre_th = 0.f, pre_m = 0.f, pre_v = 0.f;
            if (own) { pre_th = __ldcg(p.theta_rw + noff + p0 + tid); pre_m = __ldcg(p.adam_m + noff + p0 + tid); pre_v = __ldcg(p.adam_v + noff + p0 + tid); }
            // torch-Adam step of one parameter (+ its three bf16 pieces in the weight-tile image)
            auto adam_store = [&](int qg, float g, float th, float m, float v, bool img) {
                const float step_size = sScal[8], bc2_sqrt = sScal[9];
                m = __fadd_rn(m, __fmul_rn(0.1f, __fadd_rn(g, -m)));                       // exp_avg.lerp_(grad, 1 - beta1)
                v = __fadd_rn(__fmul_rn(v, 0.999f), __fmul_rn(__fmul_rn(0.001f, g), g));   // mul_(beta2).addcmul_(g, g, 1 - beta2)
                const float denom = __fadd_rn(__fdiv_rn(sqrtf(v), bc2_sqrt), 1e-8f);
                const float th_new = __fadd_rn(th, __fmul_rn(-step_size, __fdiv_rn(m, denom)));
                __stcg(p.theta_rw + qg, th_new);
                __stcg(p.adam_m + qg, m); __stcg(p.adam_v + qg, v);
                if (img && img_off >= 0) {           // where the weight tiles expect them
                    uint32_t w0, w1, w2;
                    split2(th_new, 0.f, w0, w1, w2);
                    __stcg(reinterpret_cast<unsigned short*>(wimg + img_off), (unsigned short)w0);
                    __stcg(reinterpret_cast<unsigned short*>(wimg + img_off + img_sub), (unsigned short)w1);
                    __stcg(reinterpret_cast<unsigned short*>(wimg + img_off + 2 * img_sub), (unsigned short)w2);
                }
            };
            // One rank: clip_grad_norm_ almost never clips (max_grad_norm 40), so Adam runs SPECULATIVELY with coefficient 1
            // before the slice norms are known; the barrier that publishes the norms is then also the one that publishes the
            // new parameters, and only a step that does clip redoes Adam from the saved state (one more barrier).
            const bool spec = p.world == 1 && S <= NEPI;
            float g_raw = 0.f;
            if (spec && own) { g_raw = __ldcg(p.grad + noff + p0 + tid); adam_store(noff + p0 + tid, g_raw, pre_th, pre_m, pre_v, true); }
            stamp(24);
            net_barrier();                                             // every slice norm of this network is in L2
            stamp(25);
            if (warp == 0) {
                float tot = 0.f, t2 = 0.f;
                for (int b = lane; b < G; b += 32) { tot += __ldcg(p.sumsq_part + (net * 2 + 0) * G + b); t2 += __ldcg(p.sumsq_part + (net * 2 + 1) * G + b); }
                tot = warp_sum(tot); t2 = warp_sum(t2);
                if (lane == 0) {
                    sScal[0] = (p.max_grad_norm > 0.f) ? fminf(p.max_grad_norm / (sqrtf(tot) + 1e-6f), 1.0f) : 1.0f;
                    sScal[3] = t2;
                }
            } else if (warp == 1 && blockIdx.x == 0) {               // loss statistics of this minibatch (logger means)
                float acc[4] = {0.f, 0.f, 0.f, 0.f};
                for (int b = lane; b < G; b += 32)
#pragma unroll
                    for (int i = 0; i < 4; ++i) acc[i] += __ldcg(p.stats_part + ((size_t)b * 3 + net) * 8 + i);
#pragma unroll
                for (int i = 0; i < 4; ++i) acc[i] = warp_sum(acc[i]);
                if (lane == 0) { sScal[4] = acc[0]; sScal[5] = acc[1]; sScal[6] = acc[2]; sScal[7] = acc[3]; }
            }
            epi_bar_sync();
            if (blockIdx.x == 0 && tid == 0) {
                const float inv = sScal[7] > 0.f ? 1.f / sScal[7] : 0.f;
                float* ts = p.train_stats + net * 8;
                ts[0] += sScal[4] * inv + ((net != 0) ? p.critic_norm_coef * sScal[3] : 0.f);
                ts[1] += sScal[5] * inv;
                ts[2] += sScal[6] * inv;
                ts[3] += 1.f;
            }
            const float clipc = sScal[0];
            const unsigned int xstep = p.step_base + (unsigned int)mb;
            const int xpar = (int)(xstep & 1u);
            if (spec) {
                if (clipc != 1.0f) {                                   // (uniform over the network: same partial norms, same order)
                    if (own) {
                        const float g = g_raw * clipc;
                        __stcg(p.grad + noff + p0 + tid, g);
                        adam_store(noff + p0 + tid, g, pre_th, pre_m, pre_v, true);
                    }
                    stamp(26);
                    net_barrier();
                }
            } else {
                    // clip -> average over ranks -> Adam (policy_gradient.py:L437-443, distributed.py:L193-198).  world > 1: every
            // parameter of the slice travels as ONE 8-byte word {step tag, clipped gradient} stored straight into every peer's
            // receive buffer [parity][source rank][P] over NVLink; the receiver spins on the tag of each word -- data and
            // flag arrive together, so there is no fence, no flag round and no barrier in the exchange.
            for (int base = 0; base < S; base += NEPI) {
                const int pi = base + tid;
                if (pi < S && p0 + pi < L.size) {
                    const int qg = noff + p0 + pi;
                    float g = __ldcg(p.grad + qg) * clipc;
                    bool fail = false;
                    if (p.world > 1) {
                        const unsigned long long word = ((unsigned long long)xstep << 32) | (unsigned long long)__float_as_uint(g);
                        const size_t slot = ((size_t)(xpar * p.world + p.rank)) * p.P + qg;
                        for (int r = 0; r < p.world; ++r)
                            if (r != p.rank)
                                asm volatile("st.relaxed.sys.global.b64 [%0], %1;" ::"l"(reinterpret_cast<unsigned long long*>(p.peer_buf[r]) + slot), "l"(word) : "memory");
                        const unsigned long long* mine = reinterpret_cast<const unsigned long long*>(p.peer_buf[p.rank]);
                        float sum = 0.f;
                        const long long t0 = clock64();
                        for (int r = 0; r < p.world; ++r) {
                            float v = g;
                            if (r != p.rank) {
                                const unsigned long long* src = mine + ((size_t)(xpar * p.world + r)) * p.P + qg;
                                unsigned long long w64;
                                for (;;) {
                                    asm volatile("ld.relaxed.sys.global.b64 %0, [%1];" : "=l"(w64) : "l"(src) : "memory");
                                    if ((unsigned int)(w64 >> 32) == xstep) break;
                                    if (clock64() - t0 > 20000000000LL) { *p.error_flag = 1; fail = true; break; }   // ~10 s: fail loudly, never hang the GPU
                                }
                                v = __uint_as_float((unsigned int)w64);
                            }
                            sum += v;
                        }
                        g = sum / (float)p.world;
                    }
                    if (!fail) {
                        __stcg(p.grad + qg, g);
                        const bool pre = base == 0;                     // first chunk: state prefetched before the barrier
                        adam_store(qg, g, pre ? pre_th : __ldcg(p.theta_rw + qg), pre ? pre_m : __ldcg(p.adam_m + qg),
                                   pre ? pre_v : __ldcg(p.adam_v + qg), pre);
                    }
                }
            }
            stamp(26);
            net_barrier();                                             // the new parameters of this network are in L2
            }
            stamp(27);
            if (S <= NEPI) {
                // weights: ONE bulk copy (TMA) of the image the Adam owners just wrote; biases / log_std: a few scalar loads
                if (tid == 0) {
                    asm volatile("fence.proxy.async.global;\n" ::: "memory");       // generic-proxy writes (other SMs, acquired above) -> async-proxy read
                    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(bar(RDY_W)), "r"(W_IMG) : "memory");
                    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
                                 ::"r"(sbase + OFF_W1), "l"(wimg), "r"(W_IMG), "r"(bar(RDY_W)) : "memory");
                }
                if (tid >= 64 && tid < 128) { const int i = tid - 64; if (!ones_col) misc[MF_B1 + i] = __ldcg(theta + L.off_b1 + i); misc[MF_B2 + i] = __ldcg(theta + L.off_b2 + i); }
                if (tid >= 128 && tid < 144) {
                    const int i = tid - 128;
                    misc[MF_B3 + i] = (i < L.out) ? __ldcg(theta + L.off_b3 + i) : 0.f;
                    stage_policy(misc + MF_LS, i, (net == 0 && i < A) ? __ldcg(theta + L.off_logstd + i) : 0.f);
                }
                mbar_wait_a(bar(RDY_W), (uint32_t)(mb & 1));
            } else {
                stage_weights_x3(sbase, misc, theta, L, net, O, A, tid);   // slices longer than the block: the image is incomplete
            }
            epi_bar_sync();
            stamp(28);
        }
        if (FUSED && blockIdx.x == 0 && tid == 0) p.adam_step[net] = step_t0 + n_mb;     // every CTA read it before the first barrier
    }
    __syncthreads();
}

}  // namespace osb

using namespace osb;

extern "C" {

int osb_tc_grid_blocks(long long rows, int net_mask);

static long long* g_x3_dbg = nullptr;
// development aid: clock64 stamps of CTA (0, 0) of the next launches go to buf (2048 long long), NULL turns it off
int osb_x3_debug_buffer(long long* buf) { g_x3_dbg = buf; return OSB_OK; }

static int x3_set_attr() {
    static bool attr = false;
    if (!attr) {
        const size_t smem = 1024 + X3_SMEM;
        OSB_CUDA(cudaFuncSetAttribute(minibatch_grad_x3_kernel<false, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        OSB_CUDA(cudaFuncSetAttribute(minibatch_grad_x3_kernel<false, 16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        OSB_CUDA(cudaFuncSetAttribute(minibatch_grad_x3_kernel<true, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        OSB_CUDA(cudaFuncSetAttribute(minibatch_grad_x3_kernel<true, 16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr = true;
    }
    return OSB_OK;
}

// accumulator images for a grid of nb x (up to) 3 CTAs
static int x3_bind_acc(X3Args& p, int nb) {
    p.acc = acc_scratch(ACC_UPDATE_X3, (size_t)nb * 3 * 128 * T_COLS * sizeof(float));
    return p.acc ? OSB_OK : OSB_ERR_CUDA;
}

// Split-bf16 (parity-grade tensor-core) variant of osb_minibatch_grad: same arguments, O <= 64, A <= 16,
// loss kinds PPO-clip / ratio / FOCOPS / cost surrogate / P3O.  gpart holds osb_tc_grid_blocks(mb_count, net_mask) rows of P floats.
int osb_minibatch_grad_x3(const float* theta, int O, int A, const float* obs, const float* act,
                          const float* logp, const float* adv_r, const float* adv_c,
                          const float* tv_r, const float* tv_c, const float* mu_old,
                          const float* moments, const int* perm, long long total, unsigned perm_seed,
                          long long mb_start, int mb_count, int loss_kind, float clip,
                          float entropy_coef, float focops_lam, float focops_eta,
                          const float* lagrange, const float* logstd_old, int net_mask, float* gpart,
                          float* stats_part, const int* stop_flag, void* stream) {
    OSB_CHECK_ARG(theta && obs && act && logp && adv_r && adv_c && tv_r && tv_c && moments, "null input");
    OSB_CHECK_ARG(O > 0 && O <= 64 && A > 0 && A <= 16 && mb_count > 0 && total > 0, "bf16x3 path needs O <= 64, A <= 16");
    OSB_CHECK_ARG(mb_start >= 0 && mb_start + mb_count <= total, "minibatch window out of range");
    OSB_CHECK_ARG((loss_kind >= 0 && loss_kind <= 3) || loss_kind == LOSS_P3O, "loss kind not on the bf16x3 path");
    OSB_CHECK_ARG(loss_kind != LOSS_FOCOPS || (mu_old && logstd_old), "FOCOPS needs mu_old / logstd_old");
    OSB_CHECK_ARG(net_mask > 0 && net_mask < 8, "net_mask");
    X3Args p = {};
    p.b = Batch{obs, act, logp, adv_r, adv_c, tv_r, tv_c, moments, perm, total, perm_seed, mb_start, mb_count, 0};
    p.lc = LossParams{loss_kind, clip, entropy_coef, focops_lam, focops_eta, lagrange, mu_old, logstd_old, nullptr};
    p.theta = theta; p.gpart = gpart; p.stats_part = stats_part; p.stop_flag = stop_flag;
    p.O = O; p.A = A; p.P = actor_layout(O, A).size + 2 * critic_layout(O, A).size; p.net_mask = net_mask;
    p.batch_size = mb_count; p.world = 1; p.dbg = g_x3_dbg;
    const int nb = osb_tc_grid_blocks(mb_count, net_mask);
    int rc = x3_set_attr();
    if (rc) return rc;
    if ((rc = x3_bind_acc(p, nb))) return rc;
    const bool single = (net_mask & (net_mask - 1)) == 0;
    if (loss_two_pass(loss_kind) && (net_mask & 1)) {   // pass 1: actor forward only
        X3Args q = p;
        q.forward_only = 1; q.net_mask = 1;
        const int nb1 = osb_tc_grid_blocks(mb_count, 1);
        if (A <= 8) minibatch_grad_x3_kernel<false, 8><<<dim3(nb1, 1), NTX3, 1024 + X3_SMEM, (cudaStream_t)stream>>>(q);
        else minibatch_grad_x3_kernel<false, 16><<<dim3(nb1, 1), NTX3, 1024 + X3_SMEM, (cudaStream_t)stream>>>(q);
        OSB_LAUNCH_CHECK();
        if ((rc = pass1_gate(stats_part, nb1, stop_flag, p.lc, (cudaStream_t)stream))) return rc;
    }
    if (A <= 8) minibatch_grad_x3_kernel<false, 8><<<dim3(nb, single ? 1 : 3), NTX3, 1024 + X3_SMEM, (cudaStream_t)stream>>>(p);
    else minibatch_grad_x3_kernel<false, 16><<<dim3(nb, single ? 1 : 3), NTX3, 1024 + X3_SMEM, (cudaStream_t)stream>>>(p);
    OSB_LAUNCH_CHECK();
    return OSB_OK;
}

// backward half of the bf16x3 Fisher-vector product (called by osb_fvp_partials_x3, csrc/fvp_x3.cu)
int osb_x3_fvp_backward(const float* theta_actor, const float* vec, int O, int A, const float* obs, long long total, int stride,
                        const float* dmu, float* gpart, float* stats_scratch, void* stream) {
    const long long nrows = (total + stride - 1) / stride;
    X3Args p = {};
    p.b = Batch{obs, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, total, 0u, 0, (int)nrows, stride};
    p.lc.kind = LOSS_FVP; p.theta = theta_actor; p.gpart = gpart; p.stats_part = stats_scratch;
    p.O = O; p.A = A; p.P = actor_layout(O, A).size; p.net_mask = 1;
    p.batch_size = (int)nrows; p.world = 1; p.dbg = nullptr;
    p.fvp_dmu = dmu; p.fvp_vec = vec; p.fvp_scale = 1.0f / ((float)nrows * (float)A);
    const int nb = osb_tc_grid_blocks(nrows, 1);
    int rc = x3_set_attr();
    if (rc) return rc;
    if ((rc = x3_bind_acc(p, nb))) return rc;
    if (A <= 8) minibatch_grad_x3_kernel<false, 8><<<dim3(nb, 1), NTX3, 1024 + X3_SMEM, (cudaStream_t)stream>>>(p);
    else minibatch_grad_x3_kernel<false, 16><<<dim3(nb, 1), NTX3, 1024 + X3_SMEM, (cudaStream_t)stream>>>(p);
    OSB_LAUNCH_CHECK();
    return OSB_OK;
}

// One update iteration of PolicyGradient._update (policy_gradient.py:L369-381) as ONE persistent cooperative
// kernel on bf16x3 tiles: all minibatches of [0, total) in steps of batch_size, each = fused forward + loss +
// backward, fixed-order partial reduction, per-network clip_grad_norm_, (world > 1: clipped-gradient exchange
// over NVLink peer memory, policy_gradient.py:L437-443 / distributed.py:L193-198) and torch-Adam, with the
// parameters re-staged in shared memory between minibatches.  perm: [total] slab rows of this iteration or NULL
// (Feistel order keyed by perm_seed).  gpart: osb_tc_grid_blocks(batch_size, net_mask) rows of P floats.
// peer_buf / peer_flag: device arrays of `world` pointers ([2][world][P] floats, [2*world + 2*world*160] flags)
// or NULL for one rank.
int osb_ppo_update_iter_x3(float* theta, float* grad, float* adam_m, float* adam_v, int* adam_step, int O, int A,
                           const float* obs, const float* act, const float* logp, const float* adv_r,
                           const float* adv_c, const float* tv_r, const float* tv_c, const float* moments,
                           const int* perm, long long total, unsigned perm_seed, int batch_size, int loss_kind,
                           float clip, float entropy_coef, const float* lagrange, int net_mask,
                           float critic_norm_coef, float max_grad_norm, float lr_actor, float lr_critic_r,
                           float lr_critic_c, float* gpart, float* stats_part, float* train_stats,
                           const int* stop_flag, void* peer_buf, void* peer_flag, int world, int rank,
                           int* p2p_error, void* stream) {
    OSB_CHECK_ARG(theta && grad && adam_m && adam_v && adam_step && obs && act && logp && adv_r && adv_c && tv_r && tv_c && moments, "null input");
    OSB_CHECK_ARG(O > 0 && O <= 64 && A > 0 && A <= 16 && batch_size > 0 && total > 0 && total < (1ll << 31), "bf16x3 path needs O <= 64, A <= 16");
    OSB_CHECK_ARG(loss_kind == LOSS_PPO_CLIP || loss_kind == LOSS_RATIO || loss_kind == LOSS_COST, "loss kind not on the fused bf16x3 path");
    OSB_CHECK_ARG(net_mask > 0 && net_mask < 8 && gpart && stats_part && train_stats, "bad argument");
    OSB_CHECK_ARG(world >= 1 && (world == 1 || (peer_buf && peer_flag && p2p_error && rank >= 0 && rank < world && world <= 64)), "bad p2p argument");
    static float* d_ws = nullptr;            // [0, 4): barrier counters (u32); [64, 64 + 6 * 148): slice norms
    static unsigned int step_base = 0;       // identical on every rank: same call sequence
    cudaStream_t s = (cudaStream_t)stream;
    if (!d_ws) OSB_CUDA(cudaMalloc(&d_ws, (64 + 6 * 148) * sizeof(float)));
    OSB_CUDA(cudaMemsetAsync(d_ws, 0, 4 * sizeof(unsigned int), s));
    X3Args p = {};
    p.b = Batch{obs, act, logp, adv_r, adv_c, tv_r, tv_c, moments, perm, total, perm_seed, 0, (int)total, 0};
    p.lc.kind = loss_kind; p.lc.clip = clip; p.lc.entropy_coef = entropy_coef; p.lc.lagrange = lagrange;
    p.theta = theta; p.gpart = gpart; p.stats_part = stats_part; p.stop_flag = stop_flag;
    p.O = O; p.A = A; p.P = actor_layout(O, A).size + 2 * critic_layout(O, A).size; p.net_mask = net_mask;
    p.batch_size = batch_size; p.theta_rw = theta; p.grad = grad; p.adam_m = adam_m; p.adam_v = adam_v; p.adam_step = adam_step;
    p.critic_norm_coef = critic_norm_coef; p.max_grad_norm = max_grad_norm;
    p.lr[0] = lr_actor; p.lr[1] = lr_critic_r; p.lr[2] = lr_critic_c;
    p.sumsq_part = d_ws + 64; p.train_stats = train_stats; p.bar_ctr = reinterpret_cast<unsigned int*>(d_ws);
    p.peer_buf = (float* const*)peer_buf; p.peer_flag = (unsigned int* const*)peer_flag;
    p.world = world; p.rank = rank; p.error_flag = p2p_error; p.dbg = g_x3_dbg;
    {   // weight-tile images: padding positions stay zero, so a change of the layout clears them
        static uint8_t* d_wimg = nullptr;
        static int img_O = -1, img_A = -1;
        if (!d_wimg) OSB_CUDA(cudaMalloc(&d_wimg, 3 * W_IMG));
        if (img_O != O || img_A != A) { OSB_CUDA(cudaMemsetAsync(d_wimg, 0, 3 * W_IMG, s)); img_O = O; img_A = A; }
        p.wimg = d_wimg;
    }
    const int n_mb = (int)((total + batch_size - 1) / batch_size);
    p.step_base = step_base + 1u;
    step_base += (unsigned int)n_mb;
    const int first = (int)(total < batch_size ? total : batch_size);
    const int nb = osb_tc_grid_blocks(first, net_mask);
    int rc = x3_set_attr();
    if (rc) return rc;
    if ((rc = x3_bind_acc(p, nb))) return rc;
    const bool single = (net_mask & (net_mask - 1)) == 0;
    void* args[] = {&p};
    osb_count_launch();
    OSB_CUDA(cudaLaunchCooperativeKernel(A <= 8 ? (void*)minibatch_grad_x3_kernel<true, 8> : (void*)minibatch_grad_x3_kernel<true, 16>,
                                         dim3(nb, single ? 1 : 3), dim3(NTX3), args, 1024 + X3_SMEM, s));
    return OSB_OK;
}

}  // extern "C"
