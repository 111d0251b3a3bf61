// Batched policy step on a trained model: the forwards of ConstraintActorCritic.step
// (models/actor_critic/constraint_actor_critic.py:L84-109) over B rows of normalised observations, outside the
// rollout.  Per selected network (net_mask bit 0 actor, bit 1 reward critic, bit 2 cost critic):
//   actor : mean[B][A] (GaussianLearningActor.mean), act = mean + sigma * eps (Normal.rsample with caller-supplied
//           standard-normal eps; eps == null: act = mean, predict(obs, deterministic=True)), logp[B] of act or of a
//           caller-supplied act_in (GaussianLearningActor.log_prob, gaussian_learning_actor.py:L64-139);
//   critic: value[B] (VCritic.forward, models/critic/v_critic.py:L75-92).
// The arithmetic is the rollout's (csrc/rollout.cu) in every precision mode: the tensor-core modes run the forward of
// csrc/tc_forward.cuh that the rollout and the evaluation kernels run, the fp32 mode the mlp.cuh tiles, and the actor
// head uses the same Gaussian helpers (csrc/gaussian.cuh) and log-prob summation tree, so a slab row of the rollout
// fed back through this kernel gives the action, log-prob and values the rollout stored.
//   precision 0: fp32 FMA tiles of 32 rows (csrc/mlp.cuh), any O;
//   precision 1: tf32 wgmma tiles of 128 rows (csrc/umma.cuh), layer 1 K-chunked for 64 < O <= 512;
//   precision 2: bf16x3 wgmma tiles of 128 rows (csrc/x3.cuh), O <= 64.
// Outside those bounds a tensor-core mode runs on the fp32 tiles, as the rollout does.
#include "common.cuh"
#include "gaussian.cuh"
#include "mlp.cuh"
#include "tc_forward.cuh"

namespace osb {

struct PolicyArgs {
    const float* theta;    // flat [actor | critic_r | critic_c]
    const float* obs;      // [B][O] normalised observations
    const float* eps;      // [B][A] standard-normal draws, or null
    const float* act_in;   // [B][A] actions to score, or null
    float* mean;           // [B][A] or null
    float* act;            // [B][A] or null
    float* logp;           // [B] or null
    float* value_r;        // [B] or null
    float* value_c;        // [B] or null
    float* acc;            // tensor-core tiles: accumulator images, one [128][TC_COLS] per CTA
    long long B;
    int O, A;
    int nets;              // network of grid row y: (nets >> 2y) & 3
    int vec;               // obs rows can be read as float4 (O % 4 == 0, 16-byte aligned base)
};

constexpr int PT = 32;            // rows per fp32 tile (the rollout's RT)
// the 4-byte-word region after the tensor-core operand tiles (offsets in words)
constexpr int PW_B1 = 0;                  // [64] layer biases
constexpr int PW_B2 = PW_B1 + 64;         // [64]
constexpr int PW_B3 = PW_B2 + 64;         // [16]
constexpr int PW_SD = PW_B3 + 16;         // [3][16] sigma, 2 sigma^2, log sigma per action
constexpr int PW_MU = PW_SD + 48;         // [128][16] mean of the tile's rows (actor CTAs)
constexpr int PW_WORDS = PW_MU + TC_ROWS * OUTP;

static size_t policy_tc_smem_bytes(bool x3) {
    return 1024 + (x3 ? TcTiles<true>::FLOATS : TcTiles<false>::FLOATS) + PW_WORDS * sizeof(float);
}
static size_t policy_fma_smem_bytes() { return (NETSMEM_FLOATS_FWD + 3 * PT * LD + PT * LDO + 48) * sizeof(float); }

__device__ __forceinline__ int policy_net(const PolicyArgs& p) { return (p.nets >> (2 * blockIdx.y)) & 3; }

// sigma = exp(log_std) and the log-prob constants of every action, as the rollout stages them
__device__ __forceinline__ void stage_sigma(const PolicyArgs& p, float* sSd) {
    const int a = threadIdx.x;
    if (a < 16) {
        const float sd = (a < p.A) ? expf(__ldg(p.theta + a)) : 1.f;   // log_std leads the actor's parameters
        sSd[a] = sd; sSd[16 + a] = __fmul_rn(2.f, __fmul_rn(sd, sd)); sSd[32 + a] = logf(sd);
    }
}

// The actor's outputs of `rows` rows from row r0 (sMu[e * ld + a] = mean of row r0 + e): thread -> (row e = tid / 8 + 32 i,
// lane q = tid % 8) over actions q, q + 8, log-prob terms summed in the rollout's tree.  rows % 32 == 0.
__device__ __forceinline__ void policy_head(const PolicyArgs& p, const float* sMu, int ld, const float* sSd, long long r0,
                                            int rows) {
    const int A = p.A, q = threadIdx.x & 7;
    for (int e = threadIdx.x >> 3; e < rows; e += NTHREADS / 8) {
        const long long row = r0 + e;
        const bool ok = row < p.B;
        float lp = 0.f;
        for (int a = q; a < A; a += 8) {
            const float mu = sMu[e * ld + a];
            const size_t i = (size_t)row * A + a;
            float term;
            if (p.act_in) {
                term = gaussian_log_prob(ok ? __ldg(p.act_in + i) : mu, mu, sSd[16 + a], sSd[32 + a]);
            } else {
                const float eps = (ok && p.eps) ? __ldg(p.eps + i) : 0.f;
                const float act = sample_action(mu, sSd[a], sSd[16 + a], sSd[32 + a], eps, term);
                if (ok && p.act) p.act[i] = act;
            }
            if (ok && p.mean) p.mean[i] = mu;
            lp += term;
        }
        lp += __shfl_xor_sync(0xffffffffu, lp, 1);
        lp += __shfl_xor_sync(0xffffffffu, lp, 2);
        lp += __shfl_xor_sync(0xffffffffu, lp, 4);
        if (ok && q == 0 && p.logp) p.logp[row] = lp;
    }
}

// ---------------------------------------------------------------------------------------------
// fp32 FMA tiles: one CTA per (32 rows, network), the GEMMs of rollout_step_kernel.
__global__ void __launch_bounds__(NTHREADS) policy_fma_kernel(PolicyArgs p) {
    extern __shared__ __align__(16) float smem[];
    NetSmem W;
    float* base = carve_net_smem<false>(smem, W);
    float* sX = base;  base += PT * LD;
    float* sH1 = base; base += PT * LD;
    float* sH2 = base; base += PT * LD;
    float* sO = base;  base += PT * LDO;
    float* sSd = base;

    const int net = policy_net(p);
    const long long r0 = (long long)blockIdx.x * PT;
    const int O = p.O;
    const int nchunks = (O + KC - 1) / KC;
    const NetLayout L = net_layout(net, O, p.A);
    const float* theta = p.theta + net_offset(net, O, p.A);
    auto load_chunk = [&](int kc) {   // W1 and X columns [kc * KC, kc * KC + KC), zero padded
        load_w1_chunk(theta, L, kc, W);
        for (int i = threadIdx.x; i < PT * KC; i += NTHREADS) {
            const int e = i / KC, k = i % KC, j = kc * KC + k;
            const long long row = r0 + e;
            sX[e * LD + k] = (row < p.B && j < O) ? __ldg(p.obs + row * O + j) : 0.f;
        }
    };
    load_net_rest<false>(theta, L, W);
    load_chunk(0);
    if (net == 0) stage_sigma(p, sSd);
    __syncthreads();
    mlp_hidden<PT>(sX, sH1, sH2, W, nchunks, load_chunk);
    mlp_out<PT>(sH2, sO, W, L.out);
    if (net == 0) {
        policy_head(p, sO, LDO, sSd, r0, PT);
    } else if (threadIdx.x < PT && r0 + threadIdx.x < p.B) {
        (net == 1 ? p.value_r : p.value_c)[r0 + threadIdx.x] = sO[threadIdx.x * LDO];
    }
}

// ---------------------------------------------------------------------------------------------
// Tensor-core tiles: grid (CTAs per network, networks), each CTA loops over tiles of 128 rows through the forward of
// rollout_step_tc_kernel (csrc/tc_forward.cuh; X3 = true: bf16x3, X3 = false: tf32).
template <bool X3>
__global__ void __launch_bounds__(NTHREADS, 2) policy_tc_kernel(PolicyArgs p) {
    using namespace umma;
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const uint32_t pad = (1024u - (smem_u32(smem_raw) & 1023u)) & 1023u;
    const uint32_t B0 = smem_u32(smem_raw) + pad;
    float* fbase = reinterpret_cast<float*>(smem_raw + pad + TcTiles<X3>::FLOATS);
    float* sB1 = fbase + PW_B1;
    float* sB2 = fbase + PW_B2;
    float* sB3 = fbase + PW_B3;
    float* sSd = fbase + PW_SD;
    float* sMu = fbase + PW_MU;
    __shared__ uint64_t bar;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int q = warp & 3, h = warp >> 2;
    const int net = policy_net(p);
    const int O = p.O;
    const NetLayout L = net_layout(net, O, p.A);
    const float* theta = p.theta + net_offset(net, O, p.A);
    const int nchunks = X3 ? 1 : (O + 63) >> 6;

    tc_stage_weights<X3>(B0, theta, L, O, sB1, sB2, sB3);
    if (net == 0) stage_sigma(p, sSd);
    if (tid == 0) { mbar_init(&bar, 1); mbar_init_fence(); }
    fence_async_smem();
    __syncthreads();
    const Acc tm = acc_cta(p.acc, TC_COLS);
    const uint32_t lane_base = (uint32_t)(q * 32) << 16;
    uint32_t phase = 0;
    const long long ntiles = (p.B + TC_ROWS - 1) / TC_ROWS;

#pragma unroll 1
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const long long r0 = tile * TC_ROWS;
        auto row_of = [&](int m) -> long long { return r0 + m < p.B ? r0 + m : -1; };
        tc_forward<X3>(B0, tm, &bar, phase, sB1, sB2, nchunks,
                       [&](int c) { tc_stage_rows<X3>(B0, p.obs, O, p.vec, c, theta, L, row_of); });
        if (h == 0) {
            float o16[16];
            acc_ld16(tm, lane_base + TC_C_OUT, o16);
            const int e = 32 * q + lane;
            if (net != 0) {
                if (r0 + e < p.B) (net == 1 ? p.value_r : p.value_c)[r0 + e] = o16[0] + sB3[0];
            } else {
#pragma unroll
                for (int a = 0; a < 16; ++a) sMu[e * OUTP + a] = o16[a] + sB3[a];
            }
        }
        __syncthreads();
        if (net == 0) {
            policy_head(p, sMu, OUTP, sSd, r0, TC_ROWS);
            __syncthreads();
        }
    }
}

static bool use_x3(int precision, int O) { return precision == 2 && O <= 64; }
static bool use_tf32(int precision, int O) { return precision == 1 && O <= 512; }

// CTAs per network of a tensor-core launch: about two per SM over the whole grid, never more than there are tiles
static int policy_tc_blocks(long long B, int nnets) {
    const long long tiles = (B + TC_ROWS - 1) / TC_ROWS;
    const int cap = (2 * grid_sms() + nnets - 1) / nnets;
    return (int)(tiles < cap ? tiles : cap);
}
// accumulator images for the largest tensor-core grid on this device (any B, any net_mask)
static size_t policy_acc_bytes() { return (size_t)(2 * grid_sms() + 2) * 128 * TC_COLS * sizeof(float); }

// One-time host actions: the kernels' shared-memory attributes and the accumulator images.  Never called on a
// capturing stream (see osb_policy_step).
static bool g_policy_attr = false;

static int policy_prepare() {
    if (!g_policy_attr) {
        OSB_CUDA(cudaFuncSetAttribute(policy_fma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)policy_fma_smem_bytes()));
        OSB_CUDA(cudaFuncSetAttribute(policy_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)policy_tc_smem_bytes(false)));
        OSB_CUDA(cudaFuncSetAttribute(policy_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)policy_tc_smem_bytes(true)));
        g_policy_attr = true;
    }
    if (!acc_scratch(ACC_POLICY, policy_acc_bytes())) return OSB_ERR_CUDA;
    return OSB_OK;
}

}  // namespace osb

using namespace osb;

extern "C" {

int osb_policy_prepare(void) { return policy_prepare(); }

int osb_policy_step(const float* theta, int O, int A, long long B, const float* obs, const float* eps,
                    const float* act_in, int net_mask, int precision, float* mean, float* act, float* logp,
                    float* value_r, float* value_c, void* stream) {
    OSB_CHECK_ARG(theta && obs, "theta and obs must not be NULL");
    OSB_CHECK_ARG(O >= 1 && A >= 1 && A <= OUTP && B >= 1, "bad dimensions (O >= 1, 1 <= A <= 16, B >= 1)");
    OSB_CHECK_ARG(net_mask >= 1 && net_mask <= 7, "net_mask must name at least one of bits 0-2");
    OSB_CHECK_ARG(precision >= 0 && precision <= 2, "precision must be 0, 1 or 2");
    OSB_CHECK_ARG(!(eps && act_in), "eps and act_in are exclusive");
    OSB_CHECK_ARG(!(act_in && act), "act is not written when act_in is given: pass NULL");
    OSB_CHECK_ARG(!(net_mask & 2) || value_r, "net_mask bit 1 needs value_r");
    OSB_CHECK_ARG(!(net_mask & 4) || value_c, "net_mask bit 2 needs value_c");
    cudaStream_t s = (cudaStream_t)stream;
    const bool tc = use_x3(precision, O) || use_tf32(precision, O);
    if (!g_policy_attr || (tc && acc_scratch_capacity(ACC_POLICY) < policy_acc_bytes())) {
        cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
        OSB_CUDA(cudaStreamIsCapturing(s, &cs));
        if (cs != cudaStreamCaptureStatusNone) {
            osb_set_error("osb_policy_step on a capturing stream needs its kernel attributes and accumulator images: "
                          "call osb_policy_prepare (or one eager osb_policy_step) before the capture");
            return OSB_ERR_UNSUPPORTED;
        }
        if (int rc = policy_prepare()) return rc;
    }
    PolicyArgs p{theta, obs, eps, act_in, mean, act, logp, value_r, value_c, nullptr, B, O, A, 0, 0};
    int nnets = 0;
    for (int net = 0; net < 3; ++net)
        if (net_mask & (1 << net)) p.nets |= net << (2 * nnets++);
    p.vec = (O & 3) == 0 && ((uintptr_t)obs & 15) == 0;
    if (tc) {
        const bool x3 = use_x3(precision, O);
        p.acc = acc_scratch(ACC_POLICY, policy_acc_bytes());
        if (!p.acc) return OSB_ERR_CUDA;
        const dim3 grid(policy_tc_blocks(B, nnets), nnets);
        if (x3) policy_tc_kernel<true><<<grid, NTHREADS, policy_tc_smem_bytes(true), s>>>(p);
        else policy_tc_kernel<false><<<grid, NTHREADS, policy_tc_smem_bytes(false), s>>>(p);
    } else {
        const dim3 grid((unsigned)((B + PT - 1) / PT), nnets);
        policy_fma_kernel<<<grid, NTHREADS, policy_fma_smem_bytes(), s>>>(p);
    }
    OSB_LAUNCH_CHECK();
    return OSB_OK;
}

}  // extern "C"
