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
//     Z1   = X  W1^T            -> H1 = f(. + b1)          (f: csrc/activation.cuh)
//     Z2   = H1 W2^T            -> H2 = f(. + b2)
//     OUT  = H2 W3^T            -> per-sample loss, dOUT
//     dZ2' = dOUT W3            -> dZ2 = dZ2' f'(H2)       (stored over H2)     | dW3^T += H2^T dOUT
//     dZ1' = dZ2 W2             -> dZ1 = dZ1' f'(H1)       (stored over H1)     | dW2 += dZ2^T H1, db2 += dZ2^T 1
//                                                                               | dW1 += dZ1^T X,  db1 += dZ1^T 1
//   Rows 0-63 and rows 64-127 of a tile never meet in the forward and backward chain (only the weight-gradient
//   products contract over samples), so the tile runs as a pipeline of its two row halves: every product of the chain
//   is one m64 block per half over the whole K, stored once and committed on that half's mbarrier, and every epilogue
//   warp waits for and announces its own half only -- the epilogue of rows 0-63 runs under the MMAs of rows 64-127 and
//   the next product of rows 0-63 under the epilogue of rows 64-127.  Weight / bias gradient MMAs run behind the
//   dependent chain and release their operands as soon as they have read them.  The per-sample loss inputs are copied
//   asynchronously into shared memory (cp.async) at the start of the tile; all four warps of a sample's rows compute
//   its loss, each the gradient of a quarter of the actions.  The MMA-issue warpgroup runs on 160 registers per
//   thread, the epilogue warps on 80 (setmaxnreg).
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
#include "optim.cuh"
#include "x3.cuh"

namespace osb {

using namespace x3;

__device__ __forceinline__ void epi_bar_sync() { asm volatile("bar.sync 1, 512;\n" ::: "memory"); }      // epilogue warps only
__device__ __forceinline__ void loss_bar_sync() { asm volatile("bar.sync 2, 128;\n" ::: "memory"); }     // loss warps (h == 0)
// the four epilogue warps of rows 32 q .. 32 q + 31 (named barriers 4 .. 7)
__device__ __forceinline__ void rows_bar_sync(int q) { asm volatile("bar.sync %0, 128;\n" ::"r"(4 + q) : "memory"); }

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
    const float* fvp_dmu;        // LOSS_FVP: tangent of mu per slab row [total][A] (fvp_tangent_kernel, csrc/fvp_tc.cu)
    const float* fvp_vec;        // LOSS_FVP: direction v (its log_std block gives the log_std block of F v)
    float fvp_scale;             // LOSS_FVP: 1 / (rows * A)
    long long* dbg;              // optional clock64 stamps of one CTA (x3_dbg_cta): three regions of X3_DBG_REGION, each [0] = count,
                                 // then (id, clock) pairs (tools/x3_stage_times.py)
    float* acc;                  // accumulator images, one [128][T_COLS] per CTA
    float* value_out;            // LOSS_DMU on a critic (DMU instantiation only), or null: V per row as this launch computes it
    NetSpec spec;          // hidden activations and widths (csrc/activation.cuh)
};

constexpr int XT = 128;                      // samples per tile
constexpr int NEPI = 512;                    // 16 epilogue warps: lane quarter q = warp % 4, column group h = warp / 4
constexpr int NTX3 = NEPI + 128;             // + the MMA-issue warpgroup (warps 16..19)
// Registers per thread after the one-time setup (setmaxnreg; the launch gives every warp 96).  The MMA-issue warpgroup
// holds an N = 64 fragment and the 32 image values it adds to in dW2 and dW1 (at 128 it still spills there); the
// epilogue warps give up 16 each for it.
constexpr int X3_REGS_MMA = 160, X3_REGS_EPI = 80;
static_assert(4 * 128 * X3_REGS_EPI + 128 * X3_REGS_MMA <= NTX3 * 96, "register budgets exceed the launch allocation");
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
// mbarriers.  Each completes exactly one phase per tile (waiters use the parity of the CTA's tile counter).  _0 / _1 =
// rows 0-63 / 64-127 of the tile; an epilogue warp (q = warp % 4 owns rows 32 q .. 32 q + 31) belongs to half q / 2.
enum Bar {
    // epilogue warps -> MMA-issue warpgroup, one arrival per warp: the operand's rows of that half are stored
    RDY_X0 = 0, RDY_X1,            // 8: X is staged by row tid / 4, warps 0-7 rows 0-63, warps 8-15 rows 64-127
    RDY_H1_0, RDY_H1_1,            // 8
    RDY_H2_0, RDY_H2_1,            // 8
    RDY_D0, RDY_D1,                // 8: each warp stores the dOUT columns of its own actions
    RDY_DZ2_0, RDY_DZ2_1,          // 8
    RDY_DZ1_0, RDY_DZ1_1,          // 8
    // MMA-issue warpgroup -> epilogue warps, one arrival: the product's rows of that half are in the image
    DONE_C1_0, DONE_C1_1, DONE_C2_0, DONE_C2_1, DONE_C3_0, DONE_C3_1, DONE_C4A_0, DONE_C4A_1, DONE_C5A_0, DONE_C5A_1,
    // one arrival, all 16 warps wait: the MMAs of dW3 have read H2, of dW2 H2 and H1, of dW1 X -- dZ2, dZ1 and the
    // next tile's X may be stored over them
    DONE_C4B, DONE_C5B, FREE_X,
    DONE_C6,                       // 1: the tile's last gradient product is in the image
    RDY_W,                         // 1: the expect_tx arrival of the weight-image bulk copy
    NBAR };
__host__ __device__ constexpr uint32_t bar_arrivals(int b) { return b >= DONE_C1_0 ? 1u : 8u; }
// float [128][AP + 3]: per-sample loss inputs (actions or supplied dmu, then logp, adv_r, adv_c; a critic's target at
// column AP), copied asynchronously by the warps with h == 0 and read by all four warps of the rows
constexpr uint32_t OFF_PF = OFF_BARS + NBAR * 8 + 16;
__host__ __device__ constexpr int pf_ld(int AP) { return AP + 3; }
constexpr uint32_t X3_SMEM = OFF_PF + XT * pf_ld(16) * 4;
static_assert(1024 + X3_SMEM <= 232448, "more shared memory than an H100 block can have");
// The forward products Z1, Z2 and OUT are staged as fp32 in the footprints of H1, H2 and D (x3::Staged), which they
// become: each row quarter's values stay inside its own rows of the tile, so no other warps' bytes are overwritten.
static_assert(staged_in_own_rows<64>(ACT_SUB) && staged_in_own_rows<16>(D_SUB), "a staged row leaves its own bytes of the tile");
// accumulator columns: dZ2' and dZ1' (T_ZA, T_ZB), the weight and bias gradients; [128, 144) is not written
constexpr uint32_t T_ZA = 0, T_ZB = 64, T_DW1 = 144, T_DW2 = 208, T_DW3 = 272, T_DB1 = 288, T_DB2 = 304, T_COLS = 320;

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

// stage-time stamps (development aid): regions of thread 0, thread 320 and thread 512 (the MMA-issue warpgroup), then the
// selected CTA as x | y << 16 at X3_DBG_SEL, written by the host before the launch
constexpr int X3_DBG_REGION = 4096, X3_DBG_MAX = 2000, X3_DBG_SEL = 3 * X3_DBG_REGION;
__device__ __forceinline__ bool x3_dbg_cta(const long long* dbg) {
    if (dbg == nullptr) return false;
    const long long sel = dbg[X3_DBG_SEL];
    return blockIdx.x == (unsigned)(sel & 0xffff) && blockIdx.y == (unsigned)(sel >> 16);
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
constexpr int X3_ACT_STRIDE = 32;
constexpr int x3_apv(int AP, int ACT) { return AP + X3_ACT_STRIDE * ACT; }
// DMU = LOSS_DMU only (FUSED = false): the supplied dL/dmu (fvp_dmu, per row) or, for a critic, dL/dV (tv_r / tv_c)
// is dOUT as it stands, no loss, no log_std term.
// (20 warps = 640 threads: 96 registers each, the register file divided in units of 8 per thread)
// APV = x3_apv(AP, ACT): the action width and the hidden activation in one template argument, so that the tanh
// instantiations (APV = AP) keep the symbols minibatch_grad_x3_kernel<FUSED, AP, DMU> that profiles and the SASS tests
// name; the activations' widths come in p.spec.
template <bool FUSED, int APV, bool DMU = false>
__global__ void __launch_bounds__(NTX3, 1) minibatch_grad_x3_kernel(X3Args p) {
    constexpr int AP = APV % X3_ACT_STRIDE, ACT = APV / X3_ACT_STRIDE;
    if (p.stop_flag && *p.stop_flag) return;
    const int net = (gridDim.y == 1) ? (__ffs(p.net_mask) - 1) : (int)blockIdx.y;
    if (!((p.net_mask >> net) & 1)) return;
    const Hidden<ACT, TanhAcc> af(p.spec, net);

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
    const bool is_mma_warp = warpgroup_index() == NEPI / 128;     // the four warps of the MMA-issue warpgroup
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
            for (int i = 0; i < NBAR; ++i) mbar_init_a(bar(i), bar_arrivals(i));
            mbar_init_fence();
        }
    }
    fence_async_smem();
    __syncthreads();
    const Acc tm = acc_cta(p.acc, T_COLS);
    const Staged sZ1{sbase + OFF_H1, ACT_SUB}, sZ2{sbase + OFF_H2, ACT_SUB}, sOut{sbase + OFF_D, D_SUB};

    if (is_mma_warp) {
        // ======================= MMA-issue warpgroup: uniform control flow ====================================
        wg_regs_inc<X3_REGS_MMA>();
        const uint64_t dX = desc128(sbase + OFF_X), dH1 = desc128(sbase + OFF_H1), dH2 = desc128(sbase + OFF_H2);
        const uint64_t dD = desc32(sbase + OFF_D), dW1 = desc128(sbase + OFF_W1), dW2 = desc128(sbase + OFF_W2);
        const uint64_t dW3 = desc128(sbase + OFF_W3), dOnes = desc32(sbase + OFF_ONES);
        // stage-time stamps of this warpgroup (third region of p.dbg).  Ids: 100 + 20 k for product k of Z1, Z2, OUT, dZ2',
        // dZ1', plus 4 r + {0: operands ready, 1: MMAs complete, 2: image stored, 3: committed} for row half r;
        // 200 / 201 / 202: dW3, dW2 and dW1 have read their operands; 203: the last gradient product committed; 204: dW2
        // stored, 205: dZ1 ready, 206: dW1 stored, 207: the last tile's db2 stored.
        const bool mdbg_on = tid == NEPI && x3_dbg_cta(p.dbg);
        int mdbg_n = 0;
        auto mstamp = [&](int id) {
            if (mdbg_on && mdbg_n < X3_DBG_MAX) {
                long long* d = p.dbg + 2 * X3_DBG_REGION;
                d[1 + 2 * mdbg_n] = id; d[2 + 2 * mdbg_n] = clock64(); ++mdbg_n; d[0] = mdbg_n;
            }
        };
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
                // Z1 = X W1^T, one row half after the other: each half is stored and committed on its own, and the epilogue
                // of rows 0-63 runs under the MMAs of rows 64-127.
                // Z1, Z2 and OUT are staged in shared memory, over the tile each becomes, by generic stores after this
                // warpgroup's wgmma wait; the commit's fence + bar.sync 3 + mbarrier arrival (release) orders them before
                // the epilogue's loads (acquire by its DONE wait), and `announce` fences the epilogue's bf16x3 stores
                // over them for the next MMAs.  Every earlier reader of a destination has completed by then:
                //   H1 <- Z1(t): the wgmma readers Z2(t-1), dW2(t-1), dW1(t-1) and db1(t-1) were waited on by this
                //   in-order warpgroup before DONE_C6(t-1); the epilogue's E5(t-1) loads precede its RDY_DZ1 arrivals.
                //   H2 <- Z2(t): OUT(t-1), dW3(t-1), dZ1'(t-1), dW2(t-1) likewise, and db2 of tile t-1 -- issued after
                //   Z1(t), or before DONE_C6(t-1) on a minibatch's last tile -- is a gemm_x3 that returns only after its
                //   wg_wait<0>; E4(t-1)'s loads precede RDY_DZ2.
                //   D <- OUT(t): dZ2'(t-1) and dW3(t-1) were waited on; every dOUT store of rows of half r precedes the
                //   RDY_D arrivals (and, in a statistics pass, which skips the backward, the RDY_H2 arrivals) of half r.
#pragma unroll 1
                for (int r = 0; r < 2; ++r) {
                    mbar_wait_a(bar(RDY_X0 + r), par);
                    mstamp(100 + 4 * r);
                    gemm_x3_rows<64, 2, 2, 0>(sZ1, r, dX, ACT_SUB, 32u, dW1, W_SUB, 32u, [&](int) { mstamp(101 + 4 * r); });
                    mstamp(102 + 4 * r);
                    mma_commit_a(bar(DONE_C1_0 + r));
                    mstamp(103 + 4 * r);
                }
                // db2 of the PREVIOUS tile (dZ2 still sits in the H2 buffer until this tile's Z2 is staged there): runs
                // under E1 and is waited on before Z2 is issued
                if (!first && !(!FUSED && p.forward_only)) gemm_x3<64, 16, 8, 1, 1, true>(tm, T_DB2, dH2, ACT_SUB, 2048u, dOnes, 0u, 0u, tile != (int)blockIdx.x + G);
                // Z2 = H1 W2^T
#pragma unroll 1
                for (int r = 0; r < 2; ++r) {
                    mbar_wait_a(bar(RDY_H1_0 + r), par);
                    mstamp(120 + 4 * r);
                    gemm_x3_rows<64, 2, 2, 0>(sZ2, r, dH1, ACT_SUB, 32u, dW2, W_SUB, 32u, [&](int) { mstamp(121 + 4 * r); });
                    mstamp(122 + 4 * r);
                    mma_commit_a(bar(DONE_C2_0 + r));
                    mstamp(123 + 4 * r);
                }
                // OUT = H2 W3^T
#pragma unroll 1
                for (int r = 0; r < 2; ++r) {
                    mbar_wait_a(bar(RDY_H2_0 + r), par);
                    mstamp(140 + 4 * r);
                    gemm_x3_rows<16, 2, 2, 0>(sOut, r, dH2, ACT_SUB, 32u, dW3, W3_SUB, 32u, [&](int) { mstamp(141 + 4 * r); });
                    mstamp(142 + 4 * r);
                    mma_commit_a(bar(DONE_C3_0 + r));
                    mstamp(143 + 4 * r);
                }
                if (!FUSED && p.forward_only) continue;              // statistics pass (FOCOPS mask mean): no backward
                // dZ2' = dOUT W3 ; dW3^T += H2^T dOUT (all 128 samples: behind both halves)
#pragma unroll 1
                for (int r = 0; r < 2; ++r) {
                    mbar_wait_a(bar(RDY_D0 + r), par);
                    mstamp(160 + 4 * r);
                    gemm_x3_rows<64, 1, 1, 1>(tm, T_ZA, r, dD, D_SUB, 32u, dW3, W3_SUB, 2048u, [&](int) { mstamp(161 + 4 * r); });
                    mstamp(162 + 4 * r);
                    mma_commit_a(bar(DONE_C4A_0 + r));
                    mstamp(163 + 4 * r);
                }
                // H2 is free for dZ2 once dW3's MMAs have read it; the gradient images are read only after DONE_C6
                gemm_x3<64, 16, 8, 1, 1>(tm, T_DW3, dH2, ACT_SUB, 2048u, dD, D_SUB, 512u, !first, [&](int) { mma_release_a(bar(DONE_C4B)); mstamp(200); });
                // dZ1' = dZ2 W2 ; dW2 += dZ2^T H1
#pragma unroll 1
                for (int r = 0; r < 2; ++r) {
                    mbar_wait_a(bar(RDY_DZ2_0 + r), par);
                    mstamp(180 + 4 * r);
                    gemm_x3_rows<64, 2, 2, 1>(tm, T_ZB, r, dH2, ACT_SUB, 32u, dW2, W_SUB, 2048u, [&](int) { mstamp(181 + 4 * r); });
                    mstamp(182 + 4 * r);
                    mma_commit_a(bar(DONE_C5A_0 + r));
                    mstamp(183 + 4 * r);
                }
                gemm_x3<64, 64, 8, 1, 1>(tm, T_DW2, dH2, ACT_SUB, 2048u, dH1, ACT_SUB, 2048u, !first, [&](int) { mma_release_a(bar(DONE_C5B)); mstamp(201); });
                mstamp(204);
                // last tile of the minibatch: its own db2 (dZ2 has been in H2 since RDY_DZ2), issued while the epilogue
                // stores dZ1, so that the minibatch's last commit follows dW1 directly
                if (last) { gemm_x3<64, 16, 8, 1, 1, true>(tm, T_DB2, dH2, ACT_SUB, 2048u, dOnes, 0u, 0u, !first); mstamp(207); }
                // dW1 += dZ1^T X (column 63 = db1 with the ones column).  Only dW1 reads X, and dZ1 / dZ2 are overwritten no
                // earlier than the next tile's E1 / E2, behind its Z1 / Z2.
                mbar_wait_a(bar(RDY_DZ1_0), par);
                mbar_wait_a(bar(RDY_DZ1_1), par);
                mstamp(205);
                gemm_x3<64, 64, 8, 1, 1>(tm, T_DW1, dH1, ACT_SUB, 2048u, dX, ACT_SUB, 2048u, !first, [&](int) { mma_release_a(bar(FREE_X)); mstamp(202); });
                mstamp(206);
                if (!ones_col) gemm_x3<64, 16, 8, 1, 1, true>(tm, T_DB1, dH1, ACT_SUB, 2048u, dOnes, 0u, 0u, !first);
                mma_commit_a(bar(DONE_C6));
                mstamp(203);
            }
        }
    } else {
        // ======================= epilogue warps ===============================================================
        wg_regs_dec<X3_REGS_EPI>();
        const int q = warp & 3, h = warp >> 2, rh = q >> 1;      // rh: the row half of this warp's rows (all but the X staging)
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
        auto announce = [&](int b) {        // this warp's stores are visible to the tensor core
            fence_async_smem();
            __syncwarp();
            if (lane == 0) mbar_arrive(bar(b));
        };
        const bool dbg_on = (tid == 0 || tid == 320) && x3_dbg_cta(p.dbg);      // rows 0-63 with h == 0, rows 64-127 with h == 2
        int dbg_n = 0;
        auto stamp = [&](int id) {
            if (dbg_on && dbg_n < X3_DBG_MAX) {
                long long* d = p.dbg + (tid == 0 ? 0 : X3_DBG_REGION);
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
        const int S = (L.size + G - 1) / G;                        // FUSED: parameters owned by this CTA: [p0, p0 + S)
        const int p0 = (int)blockIdx.x * S;
        const bool own = tid < S && p0 + tid < L.size;             // FUSED: this thread owns parameter p0 + tid
        // FUSED: where this thread's parameter (the first of its slice chunk) lives inside the weight-tile image, or -1
        // (log_std, b2, b3, and b1 when it is not folded into W1): byte offset of the hi piece, stride between pieces
        int img_off = -1; uint32_t img_sub = 0;
        if (FUSED) {
            const int px = p0 + tid;
            if (own) {
                if (px >= L.off_w1 && px < L.off_b1) { const int e = px - L.off_w1; img_off = (int)off128(e / O, e % O); img_sub = W_SUB; }
                else if (px >= L.off_b1 && px < L.off_w2) { if (ones_col) { img_off = (int)off128(px - L.off_b1, 63); img_sub = W_SUB; } }
                else if (px >= L.off_w2 && px < L.off_b2) { const int e = px - L.off_w2; img_off = (int)(W_X3 + off128(e >> 6, e & 63)); img_sub = W_SUB; }
                else if (px >= L.off_w3 && px < L.off_b3) { const int e = px - L.off_w3; img_off = (int)(2 * W_X3 + off128(e >> 6, e & 63)); img_sub = W3_SUB; }
            }
        }
        // FUSED: where a CTA's partial gradient of parameter px sits in its accumulator image (float offset; row m of an M = 64
        // product is lane 32 (m / 16) + m % 16), or -1: W1 [n][k] and W2 [n][k] lie along the image's columns, so a warp
        // reading 32 consecutive parameters touches one or two lines; b1, b2 and W3^T lie along its rows (1280 B apart, a
        // line per parameter), so their partials, with b3 and log_std, go to the CTA's row of gpart
        auto grad_src = [&](int px) -> int {
            int row, col;
            if (px >= L.off_w1 && px < L.off_b1) { const int e = px - L.off_w1; row = e / O; col = (int)T_DW1 + e % O; }
            else if (px >= L.off_w2 && px < L.off_b2) { const int e = px - L.off_w2; row = e >> 6; col = (int)T_DW2 + (e & 63); }
            else return -1;
            return (32 * (row >> 4) + (row & 15)) * (int)T_COLS + col;
        };
        uint8_t* wimg = FUSED ? p.wimg + (size_t)net * W_IMG : nullptr;
        // per-thread partial sums over the tiles of one minibatch (reduced once per minibatch): the statistics of the warps
        // with h == 0, and every warp's gradients of its own actions a = NA h + j in slot j
        constexpr int NA = AP / 4;
        const int a_lo = NA * h;
        float acc_st[5] = {0.f, 0.f, 0.f, 0.f, 0.f}, acc_dls[NA], acc_db[NA];      // loss, ratio, kl, count, FOCOPS mask
#pragma unroll
        for (int j = 0; j < NA; ++j) { acc_dls[j] = 0.f; acc_db[j] = 0.f; }

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
                const AdamScalars s = adam_scalars(p.lr[net], step_t0 + mb + 1);
                sScal[8] = s.step_size;
                sScal[9] = s.bc2_sqrt;
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
                if (it > 0 && !(!FUSED && p.forward_only)) mbar_wait_a(bar(FREE_X), par ^ 1u);    // previous tile's dW1 has read X
                stamp(1);
#pragma unroll
                for (int ph = 0; ph < 2; ++ph) {
                    float v[8];
#pragma unroll
                    for (int i = 0; i < 8; ++i) v[i] = xpre[8 * ph + i];
                    store8_x3(sbase + OFF_X, ACT_SUB, xm, 32 * ph + xc, v);
                }
                announce(RDY_X0 + (warp >> 3));                            // rows xm = tid / 4: warps 0-7 hold rows 0-63
                epi_bar_sync();                                            // next tile's row list is complete
                stamp(2);
                // this tile's per-sample loss inputs (used in E3) fly under the forward phases, asynchronously into shared
                // memory (the PF rows), so that no register has to wait for them
                if (h == 0) {
                    const long long prow = sRow[s_row];
                    if (prow >= 0) {
                        const float* asrc = (DMU || p.lc.kind == LOSS_FVP) ? p.fvp_dmu : p.b.act;
                        const uint32_t dst = sbase + OFF_PF + (uint32_t)(s_row * pf_ld(AP)) * 4u;
                        auto cp4 = [&](uint32_t d, const float* src) {
                            asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(d), "l"(src) : "memory");
                        };
                        if (net == 0) {
#pragma unroll
                            for (int a = 0; a < AP; ++a)
                                if (a < A) cp4(dst + 4u * a, asrc + prow * A + a);
                            if (!DMU && p.lc.kind != LOSS_FVP) { cp4(dst + 4u * AP, p.b.logp + prow); cp4(dst + 4u * AP + 4u, p.b.adv_r + prow); cp4(dst + 4u * AP + 8u, p.b.adv_c + prow); }
                        } else {
                            cp4(dst + 4u * AP, (net == 1 ? p.b.tv_r : p.b.tv_c) + prow);
                        }
                    }
                }
                // ---- E1: H1 = f(Z1 + b1) ----------------------------------------------------------------------
                // Z1 is staged over H1 (see the MMA-issue loop): the four warps of the rows read their values of it, meet,
                // and only then store the pieces of H1 over them
                mbar_wait_a(bar(DONE_C1_0 + rh), par);
                stamp(3);
                float hv[2][8];
#pragma unroll
                for (int ph = 0; ph < 2; ++ph) {
                    const int c0 = 32 * ph + 8 * h;
                    staged_load<64>(sZ1, s_row, c0, hv[ph]);
#pragma unroll
                    for (int i = 0; i < 8; ++i) hv[ph][i] = af(hv[ph][i] + sB1[c0 + i], c0 + i, af.w1);
                }
                rows_bar_sync(q);
#pragma unroll
                for (int ph = 0; ph < 2; ++ph) store8_x3(sbase + OFF_H1, ACT_SUB, s_row, 32 * ph + 8 * h, hv[ph]);
                announce(RDY_H1_0 + rh);
                // ---- E2: H2 = f(Z2 + b2), from Z2 staged over H2 -----------------------------------------------
                stamp(4);
                mbar_wait_a(bar(DONE_C2_0 + rh), par);
                stamp(5);
#pragma unroll
                for (int ph = 0; ph < 2; ++ph) {
                    const int c0 = 32 * ph + 8 * h;
                    staged_load<64>(sZ2, s_row, c0, hv[ph]);
#pragma unroll
                    for (int i = 0; i < 8; ++i) hv[ph][i] = af(hv[ph][i] + sB2[c0 + i], c0 + i, af.w2);
                }
                rows_bar_sync(q);
#pragma unroll
                for (int ph = 0; ph < 2; ++ph) store8_x3(sbase + OFF_H2, ACT_SUB, s_row, 32 * ph + 8 * h, hv[ph]);
                announce(RDY_H2_0 + rh);
                stamp(6);
                // ---- E3: OUT -> loss -> dOUT (one thread per sample in each of the four warps of the rows) -----------
                // Every warp computes the sample's scalar part of the loss (the same bits in each) and the gradient of
                // its own actions a_lo .. a_lo + NA - 1; the statistics are those of the warps with h == 0.
                mbar_wait_a(bar(DONE_C3_0 + rh), par);
                stamp(7);
                {
                    // every warp reads the whole OUT row, staged over D, before the four meet: behind the barrier they
                    // store dOUT over it
                    float o[AP];
                    staged_load<16>(sOut, s_row, 0, o);
                    if (h == 0) asm volatile("cp.async.wait_all;\n" ::: "memory");
                    rows_bar_sync(q);                                      // and the PF rows of the four warps' samples
                    const long long prow = sRow[s_row];
                    const float* pf = reinterpret_cast<const float*>(gbase + OFF_PF) + s_row * pf_ld(AP);
                    float dq[NA];
#pragma unroll
                    for (int j = 0; j < NA; ++j) dq[j] = 0.f;
                    auto own = [&](int a) { return a < A && a >= a_lo && a < a_lo + NA; };
                    if (prow >= 0) {
                        if (net != 0) {              // critic: one output, action 0 of the warps with h == 0
                            if (h == 0) {
                                const float tv = pf[AP];
                                if (DMU) {           // the supplied dL/dV (tv_r / tv_c)
                                    if (p.value_out) p.value_out[prow] = o[0] + sB3[0];
                                    acc_st[3] += 1.f;
                                    dq[0] = tv;
                                    acc_db[0] += tv;
                                } else {
                                    const float d = o[0] + sB3[0] - tv;
                                    acc_st[0] += d * d; acc_st[3] += 1.f;
                                    dq[0] = 2.f * d * inv_b;
                                    acc_db[0] += dq[0];
                                }
                            }
                        } else if (DMU) {
                            if (h == 0) acc_st[3] += 1.f;
#pragma unroll
                            for (int a = 0; a < AP; ++a)
                                if (own(a)) { const float dm = pf[a]; dq[a % NA] = dm; acc_db[a % NA] += dm; }
                        } else if (p.lc.kind == LOSS_FVP) {
                            // J^T diag(sigma^-2) dmu / (B A): the supplied tangent is the output gradient
                            if (h == 0) acc_st[3] += 1.f;
#pragma unroll
                            for (int a = 0; a < AP; ++a)
                                if (own(a)) {
                                    const float dm = pf[a] * sLs[32 + a] * p.fvp_scale;
                                    dq[a % NA] = dm;
                                    acc_db[a % NA] += dm;
                                }
                        } else {
                            float mu[AP], act[AP];
#pragma unroll
                            for (int a = 0; a < AP; ++a) { mu[a] = o[a] + sB3[a]; act[a] = (a < A) ? pf[a] : 0.f; }
                            actor_sample_loss<!FUSED, AP>(p.lc, an, A, inv_b, mu, act,
                                                          [&](int a) { return __ldg(p.lc.mu_old + prow * A + a); },
                                                          pf[AP], pf[AP + 1], pf[AP + 2], sLs, misc + MF_OLD, acc_st,
                                                          [&](int a, float dm, float dl) {
                                                              dq[a % NA] = dm; acc_db[a % NA] += dm; acc_dls[a % NA] += dl;
                                                          },
                                                          a_lo, a_lo + NA, h == 0);
                        }
                    }
                    // this warp's columns of the dOUT row: its actions, and (AP == 8) as many of the zero columns 8 .. 15
#pragma unroll
                    for (int k = 0; k < 2; ++k) {
                        const int c = (AP == 8) ? 2 * h + 8 * k : 4 * h + 2 * k;
                        const bool mine = AP == 16 || k == 0;
                        store2_x3_sw32(sbase + OFF_D, D_SUB, s_row, c, mine ? dq[(2 * k) % NA] : 0.f, mine ? dq[(2 * k + 1) % NA] : 0.f);
                    }
                    announce(RDY_D0 + rh);
                    stamp(8);
                }
                stamp(9);
                if (!FUSED && p.forward_only) {                                      // statistics pass: no backward; H2 is free once OUT is done
                    if (has_next) prefetch_x(sRowNext);
                    rpar ^= 1;
                    continue;
                }
                // ---- E4: dZ2 = (dOUT W3) f'(H2), stored over H2 once dW3 has read it -----------------------------
                if (has_next) prefetch_x(sRowNext);                        // next tile's rows fly during the backward half
                mbar_wait_a(bar(DONE_C4A_0 + rh), par);
                stamp(10);
                float dz[16];
#pragma unroll
                for (int ph = 0; ph < 2; ++ph) {
                    const int c0 = 32 * ph + 8 * h;
                    float v[8], hh[8];
                    acc_ld8(tm, lane_base + T_ZA + (uint32_t)c0, v);
                    load8_x3(sbase + OFF_H2, ACT_SUB, s_row, c0, hh);
#pragma unroll
                    for (int i = 0; i < 8; ++i) dz[8 * ph + i] = v[i] * af.d(hh[i]);
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
                }
                announce(RDY_DZ2_0 + rh);
                // ---- E5: dZ1 = (dZ2 W2) f'(H1), stored over H1 once dW2 has read it -----------------------------
                stamp(13);
                mbar_wait_a(bar(DONE_C5A_0 + rh), par);
                stamp(14);
#pragma unroll
                for (int ph = 0; ph < 2; ++ph) {
                    const int c0 = 32 * ph + 8 * h;
                    float v[8], hh[8];
                    acc_ld8(tm, lane_base + T_ZB + (uint32_t)c0, v);
                    load8_x3(sbase + OFF_H1, ACT_SUB, s_row, c0, hh);
#pragma unroll
                    for (int i = 0; i < 8; ++i) dz[8 * ph + i] = v[i] * af.d(hh[i]);
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
                announce(RDY_DZ1_0 + rh);
                stamp(17);
                rpar ^= 1;
            }
            stamp(20);
            // ---- rows of the first tile of the NEXT minibatch (its X is gathered behind the slice reduction) ------
            bool next_x = false;
            if (FUSED && mb + 1 < n_mb) {
                long long s2; int c2;
                mb_geom(mb + 1, s2, c2);
                next_x = (int)blockIdx.x < (c2 + XT - 1) / XT;
                if (next_x) tile_rows(mb + 1, blockIdx.x, sRowBuf + rpar * XT);
            }
            stamp(35);
            // FUSED: the owner's Adam state does not depend on the gradient (only this thread writes it), so its loads fly
            // under the wait for the last gradient product and the first grid barrier
            float pre_th = 0.f, pre_m = 0.f, pre_v = 0.f;
            if (FUSED && own) { pre_th = __ldcg(p.theta_rw + noff + p0 + tid); pre_m = __ldcg(p.adam_m + noff + p0 + tid); pre_v = __ldcg(p.adam_v + noff + p0 + tid); }
            // ---- this CTA's partial gradient of the minibatch: stepwise, accumulator images -> gpart; FUSED, the slice
            //      reduction reads dW1 / dW2 in the images themselves and gpart holds b1, b2, W3, b3 and log_std -------
            if (have_tiles) {
                // statistics: lanes -> warp (butterfly) -> the four warps with h == 0 (fixed order)
                if (h == 0) {
#pragma unroll
                    for (int i = 0; i < 5; ++i) acc_st[i] = warp_sum(acc_st[i]);
                    if (lane == 0) {
#pragma unroll
                        for (int i = 0; i < 5; ++i) sRed[q * 8 + i] = acc_st[i];
                    }
#pragma unroll
                    for (int i = 0; i < 5; ++i) acc_st[i] = 0.f;
                }
                // gradient sums of every warp's own actions: lanes -> warp (butterfly), per action
#pragma unroll
                for (int j = 0; j < NA; ++j) { acc_dls[j] = warp_sum(acc_dls[j]); acc_db[j] = warp_sum(acc_db[j]); }
                if (lane == 0) {
#pragma unroll
                    for (int j = 0; j < NA; ++j) { sRed[32 + q * 16 + a_lo + j] = acc_dls[j]; sRed[96 + q * 16 + a_lo + j] = acc_db[j]; }
                }
#pragma unroll
                for (int j = 0; j < NA; ++j) { acc_dls[j] = 0.f; acc_db[j] = 0.f; }
                if (!FUSED && p.forward_only) {
                    epi_bar_sync();                    // sRed of the sixteen epilogue warps
                    if (tid >= 64 && tid < 72) {
                        const int i = tid - 64;
                        __stcg(p.stats_part + ((size_t)blockIdx.x * 3 + net) * 8 + i, (i < 5) ? (sRed[i] + sRed[8 + i]) + (sRed[16 + i] + sRed[24 + i]) : 0.f);
                    }
                    break;
                }
                epi_bar_sync();                        // sRed of the sixteen epilogue warps
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
                    float s = (i < 5) ? (sRed[i] + sRed[8 + i]) + (sRed[16 + i] + sRed[24 + i]) : 0.f;
                    if (i == 5 && net == 0) s = entropy_bonus_sum<!FUSED>(p.lc, A, sLs, (sRed[3] + sRed[11]) + (sRed[19] + sRed[27]));
                    __stcg(p.stats_part + ((size_t)blockIdx.x * 3 + net) * 8 + i, s);
                }
                stamp(32);
                mbar_wait_a(bar(DONE_C6), (uint32_t)((it - 1) & 1));
                stamp(21);
                const int t_row = 16 * q + lane;       // row (lane < 16) of the M = 64 accumulators
                const int c16 = 16 * h;
                float v[16];
                if (FUSED) {                           // db1 = column 63 of dW1 (the slice reduction reads W1, W2 in the images)
                    if (ones_col && h == 3 && lane < 16) __stcg(gout + L.off_b1 + t_row, __ldcg(tm.p + (size_t)(32 * q + lane) * T_COLS + T_DW1 + 63));
                } else {
                    acc_ld16(tm, lane_base + T_DW2 + (uint32_t)c16, v);
                    if (lane < 16) {
                        float* dst = gout + L.off_w2 + t_row * 64 + c16;
#pragma unroll
                        for (int i = 0; i < 16; ++i) __stcg(dst + i, v[i]);
                    }
                    acc_ld16(tm, lane_base + T_DW1 + (uint32_t)c16, v);
                    if (lane < 16) {
                        float* dst = gout + L.off_w1 + t_row * O + c16;
#pragma unroll
                        for (int i = 0; i < 16; ++i)
                            if (c16 + i < O) __stcg(dst + i, v[i]);
                        if (ones_col && h == 3) __stcg(gout + L.off_b1 + t_row, v[15]);        // column 63 of dW1 = db1
                    }
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
            } else {
                // no tile of this (short) minibatch; FUSED: the slice reduction adds 0.f for this CTA without reading it
                if (!FUSED) for (int i = tid; i < L.size; i += NEPI) __stcg(gout + i, 0.f);
                if (tid < 8) __stcg(p.stats_part + ((size_t)blockIdx.x * 3 + net) * 8 + tid, 0.f);
            }
            stamp(22);
            if (!FUSED) break;

            // ================= in-kernel optimiser step =========================================================
            net_barrier();                                             // every partial gradient of this network is in L2
            stamp(23);
            // One rank: clip_grad_norm_ almost never clips (max_grad_norm 40), so Adam runs SPECULATIVELY with coefficient 1
            // before the slice norms are known; the barrier that publishes the norms is then also the one that publishes the
            // new parameters, and only a step that does clip redoes Adam from the saved state (one more barrier).
            const bool spec = p.world == 1 && S <= NEPI;
            const int Gh = (G + 1) >> 1;
            // The W1 / W2 partials of CTA b are read straight from its accumulator image: the MMA-issue warpgroup's image stores
            // precede its DONE_C6 arrival (fence + bar.sync 3 + mbarrier.arrive, release at CTA scope), the epilogue warps
            // acquire them by their DONE_C6 wait, and epi_bar_sync orders that before thread 0's red.release.gpu in
            // net_barrier: causality order is transitive across scopes, so the stores happen-before every read behind the
            // barrier's acquire, and the reads bypass L1 (ld.cg).  No CTA writes its dW / db columns again before the next
            // minibatch's first tile, which follows the barrier after this reduction.
            const float* anet = p.acc + (size_t)blockIdx.y * G * 128 * T_COLS;
            const float* gnet = p.gpart + (size_t)((gridDim.y == 1 ? 0 : net) * G) * PSTR;      // b3 / log_std partials
            float ssq = 0.f, st2 = 0.f, g_raw = 0.f;       // g_raw: the reduced gradient of the parameter this thread owns
            for (int base = 0; base < S; base += 256) {
                const int pi = base + (tid & 255), part = tid >> 8;
                const bool valid = pi < S && p0 + pi < L.size;
                float sacc = 0.f;
                if (valid) {
                    const int off = grad_src(p0 + pi);
                    const float* src = off >= 0 ? anet + off : gnet + p0 + pi;
                    const size_t stride = off >= 0 ? (size_t)128 * T_COLS : (size_t)PSTR;
                    const int b1 = min(G, (part + 1) * Gh);
                    for (int b = part * Gh; b < b1; b += 32) {       // 32 partial rows in flight per thread
                        float t[32];
#pragma unroll
                        for (int u = 0; u < 32; ++u) t[u] = (b + u < b1 && b + u < ntiles) ? __ldcg(src + (size_t)(b + u) * stride) : 0.f;
                        // the pairwise tree, level by level with constant indices: written as a loop over w, it was not
                        // unrolled and t went to the stack, each loaded value stored there as it arrived
#pragma unroll
                        for (int u = 0; u < 16; ++u) t[u] += t[u + 16];
#pragma unroll
                        for (int u = 0; u < 8; ++u) t[u] += t[u + 8];
#pragma unroll
                        for (int u = 0; u < 4; ++u) t[u] += t[u + 4];
                        t[0] += t[2]; t[1] += t[3];
                        t[0] += t[1];
                        sacc += t[0];
                    }
                }
                sPart[tid] = sacc;
                stamp(29);
                epi_bar_sync();
                if (part == 0 && valid) {
                    const int qg = noff + p0 + pi;
                    float g = sPart[tid] + sPart[256 + tid];
                    if (net != 0 && p.critic_norm_coef > 0.f) {
                        const float th = base == 0 ? pre_th : __ldcg(p.theta_rw + qg);      // base 0: this thread owns qg
                        g += 2.f * p.critic_norm_coef * th; st2 += th * th;
                    }
                    __stcg(p.grad + qg, g);
                    ssq += g * g;
                    if (base == 0) g_raw = g;
                    else sPart[tid] = g;                   // spec: to its owner, thread pi (only it reads this slot now)
                }
                epi_bar_sync();
                if (spec && base > 0 && own && tid >= 256) g_raw = sPart[tid - 256];      // spec: S <= 512, base 256 is the last chunk
            }
            // X of the next minibatch's first tile flies under the norm, Adam and restaging phases.  Gathered at the start of
            // the boundary, its 16 registers were live through the statistics and the slice reduction, which then spilled
            // and waited on the gathered rows.  The row list was written before net_barrier, whose bar.sync orders it
            // before these reads.
            if (next_x) prefetch_x(sRowBuf + rpar * XT);
            ssq = warp_sum(ssq); st2 = warp_sum(st2);
            if (lane == 0) { sPart[256 + warp] = ssq; sPart[272 + warp] = st2; }       // the hand-over slots stay untouched
            epi_bar_sync();
            if (tid == 0) {
                float a = 0.f, b = 0.f;
                for (int w = 0; w < 16; ++w) { a += sPart[256 + w]; b += sPart[272 + w]; }
                __stcg(p.sumsq_part + (net * 2 + 0) * G + blockIdx.x, a);
                __stcg(p.sumsq_part + (net * 2 + 1) * G + blockIdx.x, b);
            }
            stamp(30);
            if (dbg_on && own) p.dbg[(tid == 0 ? 0 : X3_DBG_REGION) + X3_DBG_REGION - 1] = __float_as_int(pre_th + pre_m + pre_v);     // waits for the state
            stamp(31);
            // torch-Adam step of one parameter (+ its three bf16 pieces in the weight-tile image)
            auto adam_store = [&](int qg, float g, float th, float m, float v, bool img) {
                const float th_new = adam_update(g, th, m, v, {sScal[8], sScal[9]});
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
            if (spec && own) adam_store(noff + p0 + tid, g_raw, pre_th, pre_m, pre_v, true);
            stamp(24);
            net_barrier();                                             // every slice norm of this network is in L2
            stamp(25);
            if (warp == 0) {
                float tot = 0.f, t2 = 0.f;
                for (int b = lane; b < G; b += 32) { tot += __ldcg(p.sumsq_part + (net * 2 + 0) * G + b); t2 += __ldcg(p.sumsq_part + (net * 2 + 1) * G + b); }
                tot = warp_sum(tot); t2 = warp_sum(t2);
                if (lane == 0) {
                    sScal[0] = (p.max_grad_norm > 0.f) ? clip_coef(tot, p.max_grad_norm) : 1.0f;
                    sScal[3] = t2;
                }
            } else if (warp == 1 && blockIdx.x == 0) {               // loss statistics of this minibatch (logger means)
                float acc[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
                for (int b = lane; b < G; b += 32)
#pragma unroll
                    for (int i = 0; i < 5; ++i) acc[i] += __ldcg(p.stats_part + ((size_t)b * 3 + net) * 8 + (i < 4 ? i : 5));
#pragma unroll
                for (int i = 0; i < 5; ++i) acc[i] = warp_sum(acc[i]);
                if (lane == 0) { sScal[4] = acc[0]; sScal[5] = acc[1]; sScal[6] = acc[2]; sScal[7] = acc[3]; sScal[10] = acc[4]; }
            }
            epi_bar_sync();
            if (blockIdx.x == 0 && tid == 0)
                fold_minibatch_stats(p.train_stats, net, sScal[4], sScal[5], sScal[6], sScal[7], sScal[10], p.critic_norm_coef,
                                     sScal[3]);
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
                    mbar_expect_tx(bar(RDY_W), W_IMG);
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

// the instantiations of one activation (the DMU ones run one network: never ACT_MIXED)
template <int ACT>
static int x3_set_attr() {
    static bool attr = false;
    if (!attr) {
        const size_t smem = 1024 + X3_SMEM;
        OSB_CUDA(cudaFuncSetAttribute(minibatch_grad_x3_kernel<false, x3_apv(8, ACT), false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        OSB_CUDA(cudaFuncSetAttribute(minibatch_grad_x3_kernel<false, x3_apv(16, ACT), false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        OSB_CUDA(cudaFuncSetAttribute(minibatch_grad_x3_kernel<true, x3_apv(8, ACT), false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        OSB_CUDA(cudaFuncSetAttribute(minibatch_grad_x3_kernel<true, x3_apv(16, ACT), false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        if constexpr (ACT != ACT_MIXED) {
            OSB_CUDA(cudaFuncSetAttribute(minibatch_grad_x3_kernel<false, x3_apv(8, ACT), true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            OSB_CUDA(cudaFuncSetAttribute(minibatch_grad_x3_kernel<false, x3_apv(16, ACT), true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        }
        attr = true;
    }
    return OSB_OK;
}

extern "C" {

static long long* g_x3_dbg = nullptr;
// development aid: clock64 stamps of one CTA of the next launches go to buf (3 * 4096 + 1 long long, the last the CTA
// x | y << 16), NULL turns it off
int osb_x3_debug_buffer(long long* buf) { g_x3_dbg = buf; return OSB_OK; }

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
    int rc = x3_bind_acc(p, nb);
    if (rc) return rc;
    const bool single = (net_mask & (net_mask - 1)) == 0;
    p.spec = net_spec();
    const NetSpec& spec = p.spec;
    if (loss_two_pass(loss_kind) && (net_mask & 1)) {   // pass 1: actor forward only
        X3Args q = p;
        q.forward_only = 1; q.net_mask = 1;
        const int nb1 = osb_tc_grid_blocks(mb_count, 1);
        rc = with_act<false>(spec.act[0], [&](auto a) {
            if (int r = x3_set_attr<a.value>()) return r;
            if (A <= 8) minibatch_grad_x3_kernel<false, x3_apv(8, a.value), false><<<dim3(nb1, 1), NTX3, 1024 + X3_SMEM, (cudaStream_t)stream>>>(q);
            else minibatch_grad_x3_kernel<false, x3_apv(16, a.value), false><<<dim3(nb1, 1), NTX3, 1024 + X3_SMEM, (cudaStream_t)stream>>>(q);
            OSB_LAUNCH_CHECK();
            return OSB_OK;
        });
        if (rc) return rc;
        if ((rc = pass1_gate(stats_part, nb1, stop_flag, p.lc, (cudaStream_t)stream))) return rc;
    }
    return with_act<true>(launch_act(spec, net_mask), [&](auto a) {
        if (int r = x3_set_attr<a.value>()) return r;
        if (A <= 8) minibatch_grad_x3_kernel<false, x3_apv(8, a.value), false><<<dim3(nb, single ? 1 : 3), NTX3, 1024 + X3_SMEM, (cudaStream_t)stream>>>(p);
        else minibatch_grad_x3_kernel<false, x3_apv(16, a.value), false><<<dim3(nb, single ? 1 : 3), NTX3, 1024 + X3_SMEM, (cudaStream_t)stream>>>(p);
        OSB_LAUNCH_CHECK();
        return OSB_OK;
    });
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
    int rc = x3_bind_acc(p, nb);
    if (rc) return rc;
    const bool single = (net_mask & (net_mask - 1)) == 0;
    p.spec = net_spec();
    void* args[] = {&p};
    return with_act<true>(launch_act(p.spec, net_mask), [&](auto a) {
        if (int r = x3_set_attr<a.value>()) return r;
        osb_count_launch();
        OSB_CUDA(cudaLaunchCooperativeKernel(A <= 8 ? (void*)minibatch_grad_x3_kernel<true, x3_apv(8, a.value), false>
                                                    : (void*)minibatch_grad_x3_kernel<true, x3_apv(16, a.value), false>,
                                             dim3(nb, single ? 1 : 3), dim3(NTX3), args, 1024 + X3_SMEM, s));
        return OSB_OK;
    });
}

}  // extern "C"

// LOSS_DMU launch of the DMU instantiations (one network, grid.y == 1) on nb CTAs
static int launch_dmu_x3(X3Args& p, int nb, cudaStream_t stream) {
    p.lc.kind = LOSS_DMU; p.lc.focops_lam = 1.f;
    p.batch_size = p.b.mb_count; p.world = 1; p.dbg = nullptr;
    int rc = x3_bind_acc(p, nb);
    if (rc) return rc;
    p.spec = net_spec();
    const NetSpec& spec = p.spec;
    return with_act<false>(launch_act(spec, p.net_mask), [&](auto a) {
        if (int r = x3_set_attr<a.value>()) return r;
        if (p.A <= 8) minibatch_grad_x3_kernel<false, x3_apv(8, a.value), true><<<dim3(nb, 1), NTX3, 1024 + X3_SMEM, stream>>>(p);
        else minibatch_grad_x3_kernel<false, x3_apv(16, a.value), true><<<dim3(nb, 1), NTX3, 1024 + X3_SMEM, stream>>>(p);
        OSB_LAUNCH_CHECK();
        return OSB_OK;
    });
}

// LOSS_DMU launches behind osb_actor_dmu_backward and osb_critic_dv_backward (csrc/update.cu)
int osb::dmu_backward_x3(const float* theta_actor, int O, int A, const float* obs, const float* dmu, int rows, float* gpart,
                         float* stats_scratch, cudaStream_t stream) {
    OSB_CHECK_ARG(O <= 64 && A <= 16, "bf16x3 path needs O <= 64, A <= 16");
    X3Args p = {};
    p.b = Batch{obs, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, rows, 0u, 0, rows, 1};
    p.theta = theta_actor; p.gpart = gpart; p.stats_part = stats_scratch;
    p.O = O; p.A = A; p.P = actor_layout(O, A).size; p.net_mask = 1;
    p.fvp_dmu = dmu;
    return launch_dmu_x3(p, osb_tc_grid_blocks(rows, 1), stream);
}

int osb::fvp_backward_x3(const float* theta_actor, const float* vec, int O, int A, const float* obs, long long total,
                         int stride, const float* dmu, float* gpart, float* stats_scratch, cudaStream_t stream) {
    const long long nrows = (total + stride - 1) / stride;
    X3Args p = {};
    p.b = Batch{obs, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, total, 0u, 0, (int)nrows, stride};
    p.lc.kind = LOSS_FVP; p.theta = theta_actor; p.gpart = gpart; p.stats_part = stats_scratch;
    p.O = O; p.A = A; p.P = actor_layout(O, A).size; p.net_mask = 1;
    p.batch_size = (int)nrows; p.world = 1; p.dbg = nullptr;
    p.fvp_dmu = dmu; p.fvp_vec = vec; p.fvp_scale = 1.0f / ((float)nrows * (float)A);
    const int nb = osb_tc_grid_blocks(nrows, 1);
    int rc = x3_bind_acc(p, nb);
    if (rc) return rc;
    p.spec = net_spec();
    const NetSpec& spec = p.spec;
    return with_act<false>(spec.act[0], [&](auto a) {
        if (int r = x3_set_attr<a.value>()) return r;
        if (A <= 8) minibatch_grad_x3_kernel<false, x3_apv(8, a.value), false><<<dim3(nb, 1), NTX3, 1024 + X3_SMEM, stream>>>(p);
        else minibatch_grad_x3_kernel<false, x3_apv(16, a.value), false><<<dim3(nb, 1), NTX3, 1024 + X3_SMEM, stream>>>(p);
        OSB_LAUNCH_CHECK();
        return OSB_OK;
    });
}

int osb::dv_backward_x3(const float* theta, int O, int A, int net, const float* obs, const float* dv, float* value, int rows,
                        float* gpart, float* stats_scratch, cudaStream_t stream) {
    OSB_CHECK_ARG(O <= 64 && A <= 16, "bf16x3 path needs O <= 64, A <= 16");
    X3Args p = {};
    p.b = Batch{obs, nullptr, nullptr, nullptr, nullptr, dv, dv, nullptr, nullptr, rows, 0u, 0, rows, 1};
    p.theta = theta; p.gpart = gpart; p.stats_part = stats_scratch;
    p.O = O; p.A = A; p.P = actor_layout(O, A).size + 2 * critic_layout(O, A).size; p.net_mask = 1 << net;
    p.value_out = value;
    return launch_dmu_x3(p, osb_tc_grid_blocks(rows, 1 << net), stream);
}
