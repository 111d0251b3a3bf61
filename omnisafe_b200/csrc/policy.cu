// Batched policy step on a trained model: the forwards of ConstraintActorCritic.step
// (models/actor_critic/constraint_actor_critic.py:L84-109) over B rows of normalised observations, outside the
// rollout.  Per selected network (net_mask bit 0 actor, bit 1 reward critic, bit 2 cost critic):
//   actor : mean[B][A] (GaussianLearningActor.mean), act = mean + sigma * eps (Normal.rsample with caller-supplied
//           standard-normal eps; eps == null: act = mean, predict(obs, deterministic=True)), logp[B] of act or of a
//           caller-supplied act_in (GaussianLearningActor.log_prob, gaussian_learning_actor.py:L64-139);
//   critic: value[B] (VCritic.forward, models/critic/v_critic.py:L75-92).
// The arithmetic is the rollout's (csrc/rollout.cu) in every precision mode: the same tiles, the same staging of the
// operands, the same Gaussian helpers (csrc/gaussian.cuh) and the same log-prob summation tree, so a slab row of the
// rollout fed back through this kernel gives the action, log-prob and values the rollout stored.
//   precision 0: fp32 FMA tiles of 32 rows (csrc/mlp.cuh), any O;
//   precision 1: tf32 wgmma tiles of 128 rows (csrc/umma.cuh), layer 1 K-chunked for 64 < O <= 512;
//   precision 2: bf16x3 wgmma tiles of 128 rows (csrc/x3.cuh), O <= 64.
// Outside those bounds a tensor-core mode runs on the fp32 tiles, as the rollout does.
#include "common.cuh"
#include "gaussian.cuh"
#include "mlp.cuh"
#include "umma.cuh"
#include "x3.cuh"

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
    float* acc;            // tensor-core tiles: accumulator images, one [128][P_COLS] per CTA
    long long B;
    int O, A;
    int nets;              // network of grid row y: (nets >> 2y) & 3
    int vec;               // obs rows can be read as float4 (O % 4 == 0, 16-byte aligned base)
};

constexpr int PT = 32;            // rows per fp32 tile (the rollout's RT)
constexpr int PTC = 128;          // rows per tensor-core tile (the rollout's RTC)
constexpr uint32_t P_COLS = 80;   // accumulator columns: Z [0, 64), OUT [64, 80)
// operand tiles (bytes after the 1024-byte alignment pad): tf32 X / H2 [128][64], H1 [128][64], W1, W2 [64][64], W3 [16][64];
// bf16x3: one activation buffer (X, H1, H2 in place) and the weights, three bf16 pieces each
constexpr uint32_t PX_SUB = PTC * 128, PX_WSUB = 64 * 128, PX_W3SUB = 16 * 128;
constexpr uint32_t P_FOFF_TF32 = 2 * PTC * 256 + 2 * 16384 + 4096, P_FOFF_X3 = 3 * PX_SUB + 6 * PX_WSUB + 3 * PX_W3SUB;
// the 4-byte-word region after the operand tiles (offsets in words)
constexpr int PW_B1 = 0;                  // [64] layer biases
constexpr int PW_B2 = PW_B1 + 64;         // [64]
constexpr int PW_B3 = PW_B2 + 64;         // [16]
constexpr int PW_SD = PW_B3 + 16;         // [3][16] sigma, 2 sigma^2, log sigma per action
constexpr int PW_MU = PW_SD + 48;         // [128][16] mean of the tile's rows (actor CTAs)
constexpr int PW_WORDS = PW_MU + PTC * OUTP;

static size_t policy_tc_smem_bytes(bool x3) { return 1024 + (x3 ? P_FOFF_X3 : P_FOFF_TF32) + PW_WORDS * sizeof(float); }
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
// Tensor-core tiles: grid (CTAs per network, networks), each CTA loops over tiles of 128 rows.  The three layer GEMMs,
// the operand staging and the epilogues are those of rollout_step_tc_kernel (X3 = true: bf16x3, X3 = false: tf32).
template <bool X3>
__global__ void __launch_bounds__(NTHREADS, 2) policy_tc_kernel(PolicyArgs p) {
    using namespace umma;
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const uint32_t pad = (1024u - (smem_u32(smem_raw) & 1023u)) & 1023u;
    const uint32_t B0 = smem_u32(smem_raw) + pad;       // X -> H2   (X3: X -> H1 -> H2, bf16x3)
    const uint32_t B2 = B0 + PTC * 256;                 // H1        (X3: unused)
    const uint32_t sW1 = X3 ? B0 + 3 * PX_SUB : B2 + PTC * 256;
    const uint32_t sW2 = sW1 + (X3 ? 3 * PX_WSUB : 16384u), sW3 = sW2 + (X3 ? 3 * PX_WSUB : 16384u);
    float* fbase = reinterpret_cast<float*>(smem_raw + pad + (X3 ? P_FOFF_X3 : P_FOFF_TF32));
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

    if constexpr (X3) {   // weights -> bf16x3 tiles
        for (int i = tid; i < 64 * 32; i += NTHREADS) {
            const int n = i >> 5, k = (i & 31) << 1;
            const float a1 = (k < O) ? __ldg(theta + L.off_w1 + n * O + k) : 0.f;
            const float b1 = (k + 1 < O) ? __ldg(theta + L.off_w1 + n * O + k + 1) : 0.f;
            const float a2 = __ldg(theta + L.off_w2 + n * 64 + k), b2 = __ldg(theta + L.off_w2 + n * 64 + k + 1);
            const uint32_t off = x3::off128(n, k);
            uint32_t w0, w1, w2;
            x3::split2(a1, b1, w0, w1, w2);
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(sW1 + off), "r"(w0) : "memory");
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(sW1 + PX_WSUB + off), "r"(w1) : "memory");
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(sW1 + 2 * PX_WSUB + off), "r"(w2) : "memory");
            x3::split2(a2, b2, w0, w1, w2);
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(sW2 + off), "r"(w0) : "memory");
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(sW2 + PX_WSUB + off), "r"(w1) : "memory");
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(sW2 + 2 * PX_WSUB + off), "r"(w2) : "memory");
        }
        for (int i = tid; i < 16 * 32; i += NTHREADS) {
            const int o = i >> 5, k = (i & 31) << 1;
            const float a = (o < L.out) ? __ldg(theta + L.off_w3 + o * 64 + k) : 0.f;
            const float b = (o < L.out) ? __ldg(theta + L.off_w3 + o * 64 + k + 1) : 0.f;
            const uint32_t off = x3::off128(o, k);
            uint32_t w0, w1, w2;
            x3::split2(a, b, w0, w1, w2);
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(sW3 + off), "r"(w0) : "memory");
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(sW3 + PX_W3SUB + off), "r"(w1) : "memory");
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(sW3 + 2 * PX_W3SUB + off), "r"(w2) : "memory");
        }
    } else {   // tf32 weights; W1 here only when it is one chunk, otherwise with each X chunk below
        const int k = tid & 63;
        for (int j = 0; j < 16; ++j) {
            const int n = (tid >> 6) + 4 * j;
            if (nchunks == 1) sts(tile_addr(sW1, n, k, 64), tf32r((k < O) ? __ldg(theta + L.off_w1 + n * O + k) : 0.f));
            sts(tile_addr(sW2, n, k, 64), tf32r(__ldg(theta + L.off_w2 + n * 64 + k)));
        }
        for (int j = 0; j < 4; ++j) {
            const int o = (tid >> 6) + 4 * j;
            sts(tile_addr(sW3, o, k, 16), tf32r((o < L.out) ? __ldg(theta + L.off_w3 + o * 64 + k) : 0.f));
        }
    }
    if (tid < 64) { sB1[tid] = __ldg(theta + L.off_b1 + tid); sB2[tid] = __ldg(theta + L.off_b2 + tid); }
    if (tid < 16) sB3[tid] = (tid < L.out) ? __ldg(theta + L.off_b3 + tid) : 0.f;
    if (net == 0) stage_sigma(p, sSd);
    if (tid == 0) { mbar_init(&bar, 1); mbar_init_fence(); }
    fence_async_smem();
    __syncthreads();
    const Acc tm = acc_cta(p.acc, P_COLS);
    const uint32_t lane_base = (uint32_t)(q * 32) << 16;
    constexpr uint32_t C_Z = 0, C_OUT = 64;
    uint32_t phase = 0;
    const long long ntiles = (p.B + PTC - 1) / PTC;

#pragma unroll 1
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const long long r0 = tile * PTC;
        if constexpr (X3) {
            // X tile: thread -> row tid / 2, 32-column half; the previous tile's MMAs have completed, the buffer is free
            const int xm = tid >> 1, xh = (tid & 1) << 5;
            const long long row = r0 + xm;
            const bool in = row < p.B;
#pragma unroll
            for (int c8 = 0; c8 < 4; ++c8) {
                const int c0 = xh + 8 * c8;
                float v[8];
                if (p.vec) {
#pragma unroll
                    for (int v4 = 0; v4 < 2; ++v4) {
                        const int c = c0 + 4 * v4;
                        const float4 x = (in && c < O) ? __ldg(reinterpret_cast<const float4*>(p.obs + row * O + c))
                                                       : make_float4(0.f, 0.f, 0.f, 0.f);
                        v[4 * v4] = x.x; v[4 * v4 + 1] = x.y; v[4 * v4 + 2] = x.z; v[4 * v4 + 3] = x.w;
                    }
                } else {
#pragma unroll
                    for (int i = 0; i < 8; ++i) v[i] = (in && c0 + i < O) ? __ldg(p.obs + row * O + c0 + i) : 0.f;
                }
                x3::store8_x3(B0, PX_SUB, xm, c0, v);
            }
            fence_async_smem();
            __syncthreads();
            const uint64_t dAct = x3::desc128(B0), dW1 = x3::desc128(sW1), dW2 = x3::desc128(sW2), dW3 = x3::desc128(sW3);
            if (warp < 4) {
                x3::gemm_x3(tm, C_Z, dAct, PX_SUB, 32u, dW1, PX_WSUB, 32u, x3::idesc_bf16(128, 64, 0, 0), 4, false);
                mma_commit(&bar);
            }
            mbar_wait(&bar, phase); phase ^= 1;
#pragma unroll
            for (int c8 = 0; c8 < 4; ++c8) {
                const int c0 = 32 * h + 8 * c8;
                float v[8];
                x3::acc_ld8(tm, lane_base + C_Z + (uint32_t)c0, v);
#pragma unroll
                for (int i = 0; i < 8; ++i) v[i] = x3::tanh_acc(v[i] + sB1[c0 + i]);
                x3::store8_x3(B0, PX_SUB, 32 * q + lane, c0, v);
            }
            fence_async_smem();
            __syncthreads();
            if (warp < 4) {
                x3::gemm_x3(tm, C_Z, dAct, PX_SUB, 32u, dW2, PX_WSUB, 32u, x3::idesc_bf16(128, 64, 0, 0), 4, false);
                mma_commit(&bar);
            }
            mbar_wait(&bar, phase); phase ^= 1;
#pragma unroll
            for (int c8 = 0; c8 < 4; ++c8) {
                const int c0 = 32 * h + 8 * c8;
                float v[8];
                x3::acc_ld8(tm, lane_base + C_Z + (uint32_t)c0, v);
#pragma unroll
                for (int i = 0; i < 8; ++i) v[i] = x3::tanh_acc(v[i] + sB2[c0 + i]);
                x3::store8_x3(B0, PX_SUB, 32 * q + lane, c0, v);
            }
            fence_async_smem();
            __syncthreads();
            if (warp < 4) {
                x3::gemm_x3(tm, C_OUT, dAct, PX_SUB, 32u, dW3, PX_W3SUB, 32u, x3::idesc_bf16(128, 16, 0, 0), 4, false);
                mma_commit(&bar);
            }
            mbar_wait(&bar, phase); phase ^= 1;
        } else {
#pragma unroll 1
            for (int c = 0; c < nchunks; ++c) {   // layer 1 as a K loop over 64-column chunks of X / W1
                const int k = tid & 63, col = c * 64 + k;
                if (nchunks > 1) {
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
                        const long long row = r0 + (tid >> 6) + 4 * (16 * half + j);
                        xv[j] = (row < p.B && col < O) ? __ldg(p.obs + row * O + col) : 0.f;
                    }
#pragma unroll
                    for (int j = 0; j < 16; ++j) sts(tile_addr(B0, (tid >> 6) + 4 * (16 * half + j), k, PTC), tf32r(xv[j]));
                }
                fence_async_smem();
                __syncthreads();
                if (warp < 4) { tc_gemm(tm, C_Z, B0, PTC, sW1, 64, 128, 64, 64, c > 0); mma_commit(&bar); }
                mbar_wait(&bar, phase); phase ^= 1;
            }
            {
                float v[32];
                acc_ld32(tm, lane_base + C_Z + 32 * h, v);
#pragma unroll
                for (int i = 0; i < 32; ++i) v[i] = tanh_fast(v[i] + sB1[32 * h + i]);
                store_row32(B2, 32 * q + lane, 32 * h, PTC, v);
            }
            fence_async_smem();
            __syncthreads();
            if (warp < 4) { tc_gemm(tm, C_Z, B2, PTC, sW2, 64, 128, 64, 64, false); mma_commit(&bar); }
            mbar_wait(&bar, phase); phase ^= 1;
            {
                float v[32];
                acc_ld32(tm, lane_base + C_Z + 32 * h, v);
#pragma unroll
                for (int i = 0; i < 32; ++i) v[i] = tanh_fast(v[i] + sB2[32 * h + i]);
                store_row32(B0, 32 * q + lane, 32 * h, PTC, v);
            }
            fence_async_smem();
            __syncthreads();
            if (warp < 4) { tc_gemm(tm, C_OUT, B0, PTC, sW3, 16, 128, 16, 64, false); mma_commit(&bar); }
            mbar_wait(&bar, phase); phase ^= 1;
        }
        if (h == 0) {
            float o16[16];
            acc_ld16(tm, lane_base + C_OUT, o16);
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
            policy_head(p, sMu, OUTP, sSd, r0, PTC);
            __syncthreads();
        }
    }
}

static bool use_x3(int precision, int O) { return precision == 2 && O <= 64; }
static bool use_tf32(int precision, int O) { return precision == 1 && O <= 512; }

// CTAs per network of a tensor-core launch: about two per SM over the whole grid, never more than there are tiles
static int policy_tc_blocks(long long B, int nnets) {
    const long long tiles = (B + PTC - 1) / PTC;
    const int cap = (2 * grid_sms() + nnets - 1) / nnets;
    return (int)(tiles < cap ? tiles : cap);
}
// accumulator images for the largest tensor-core grid on this device (any B, any net_mask)
static size_t policy_acc_bytes() { return (size_t)(2 * grid_sms() + 2) * 128 * P_COLS * sizeof(float); }

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
