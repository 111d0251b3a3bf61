// Split-bf16 (parity-grade tensor-core) full-batch actor forward: the bf16x3 variant of actor_eval_kernel
// (csrc/update.cu) / actor_eval_tc_kernel (csrc/eval_tc.cu).  Stores mu(theta) per row (old-policy snapshot,
// trpo.py:L177 / policy_gradient.py:L383-392) or reduces sum KL(old||new), sum ratio*adv, sum ratio*adv_c,
// sum ratio, count, sum ratio*adv_r in fp64.
//
// One activation buffer per CTA: X, H1 and H2 overwrite each other in place (each layer's epilogue starts after
// that layer's MMAs have completed), so a CTA needs 48 KB + 54 KB of weights and TWO CTAs share an SM: one
// CTA's epilogue runs under the other's MMAs.
#include "common.cuh"
#include "loss.cuh"
#include "mlp.cuh"
#include "x3.cuh"

namespace osb {

using namespace x3;

constexpr int EX_T = 128;
constexpr int EX_NT = 256;                                           // 8 warps: lane quarter q = warp % 4, column half h = warp / 4
constexpr uint32_t EX_SUB = EX_T * 128, EX_ACT = 3 * EX_SUB;         // [128][64] bf16 x3
constexpr uint32_t EX_WSUB = 64 * 128, EX_W = 3 * EX_WSUB, EX_W3SUB = 16 * 128, EX_W3 = 3 * EX_W3SUB;
constexpr uint32_t EXO_ACT = 0, EXO_W1 = EX_ACT, EXO_W2 = EXO_W1 + EX_W, EXO_W3 = EXO_W2 + EX_W, EXO_MISC = EXO_W3 + EX_W3;
// misc floats: b1[64] b2[64] b3[16] ls[64]; then double red[32]; long long rows[128]; barrier
constexpr uint32_t EXO_RED = EXO_MISC + (64 + 64 + 16 + 64) * 4, EXO_ROWS = EXO_RED + 32 * 8, EXO_BAR = EXO_ROWS + EX_T * 8,
                   EX_SMEM = EXO_BAR + 8;
constexpr uint32_t EX_COLS = 80;                                     // accumulator columns: Z [0, 64), OUT [64, 80)

struct EvalX3Args {
    const float* obs; const float* act; const float* logp; const float* adv_r; const float* adv_c;
    const float* mu_old; const float* logstd_old; const float* moments; const float* lagrange;
    const float* theta; float* mu_store; double* part;
    float* acc;         // accumulator images, [gridDim.x][128][EX_COLS]
    long long total; int stride, O, A;
};

__global__ void __launch_bounds__(EX_NT, 2) actor_eval_x3_kernel(EvalX3Args p) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const uint32_t pad = (1024u - (smem_u32(smem_raw) & 1023u)) & 1023u;
    const uint32_t sbase = smem_u32(smem_raw) + pad;
    uint8_t* gbase = smem_raw + pad;
    float* sB1 = reinterpret_cast<float*>(gbase + EXO_MISC);
    float* sB2 = sB1 + 64;
    float* sB3 = sB2 + 64;      // [16]
    float* sLs = sB3 + 16;      // [64] evaluation policy constants of csrc/loss.cuh
    double* sRedD = reinterpret_cast<double*>(gbase + EXO_RED);
    long long* sRow = reinterpret_cast<long long*>(gbase + EXO_ROWS);
    const uint32_t bar = sbase + EXO_BAR;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int q = warp & 3, h = warp >> 2;
    const int O = p.O, A = p.A;
    const NetLayout L = actor_layout(O, A);
    const float* theta = p.theta;
    // ---- weights -> bf16x3 tiles ----------------------------------------------------------------------------
    for (int i = tid; i < 64 * 32; i += EX_NT) {
        const int n = i >> 5, k = (i & 31) << 1;
        const float a1 = (k < O) ? __ldg(theta + L.off_w1 + n * O + k) : 0.f;
        const float b1 = (k + 1 < O) ? __ldg(theta + L.off_w1 + n * O + k + 1) : 0.f;
        const float a2 = __ldg(theta + L.off_w2 + n * 64 + k), b2 = __ldg(theta + L.off_w2 + n * 64 + k + 1);
        uint32_t w0, w1, w2;
        const uint32_t off = off128(n, k);
        split2(a1, b1, w0, w1, w2);
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sbase + EXO_W1 + off), "r"(w0) : "memory");
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sbase + EXO_W1 + EX_WSUB + off), "r"(w1) : "memory");
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sbase + EXO_W1 + 2 * EX_WSUB + off), "r"(w2) : "memory");
        split2(a2, b2, w0, w1, w2);
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sbase + EXO_W2 + off), "r"(w0) : "memory");
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sbase + EXO_W2 + EX_WSUB + off), "r"(w1) : "memory");
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sbase + EXO_W2 + 2 * EX_WSUB + off), "r"(w2) : "memory");
    }
    for (int i = tid; i < 16 * 32; i += EX_NT) {
        const int o = i >> 5, k = (i & 31) << 1;
        const float a = (o < A) ? __ldg(theta + L.off_w3 + o * 64 + k) : 0.f;
        const float b = (o < A) ? __ldg(theta + L.off_w3 + o * 64 + k + 1) : 0.f;
        uint32_t w0, w1, w2;
        split2(a, b, w0, w1, w2);
        const uint32_t off = off128(o, k);
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sbase + EXO_W3 + off), "r"(w0) : "memory");
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sbase + EXO_W3 + EX_W3SUB + off), "r"(w1) : "memory");
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sbase + EXO_W3 + 2 * EX_W3SUB + off), "r"(w2) : "memory");
    }
    if (tid < 64) { sB1[tid] = __ldg(theta + L.off_b1 + tid); sB2[tid] = __ldg(theta + L.off_b2 + tid); }
    if (tid < 16) {
        sB3[tid] = (tid < A) ? __ldg(theta + L.off_b3 + tid) : 0.f;
        stage_eval_policy(sLs, tid, (tid < A) ? __ldg(theta + L.off_logstd + tid) : 0.f,
                          (tid < A && p.logstd_old) ? __ldg(p.logstd_old + tid) : 0.f);
    }
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(bar), "r"(1u) : "memory");
        mbar_init_fence();
    }
    fence_async_smem();
    __syncthreads();
    const Acc tm = acc_cta(p.acc, EX_COLS);
    const uint32_t lane_base = (uint32_t)(q * 32) << 16;
    constexpr uint32_t C_Z = 0, C_OUT = 64;
    uint32_t phase = 0;
    const uint64_t dAct = desc128(sbase + EXO_ACT), dW1 = desc128(sbase + EXO_W1), dW2 = desc128(sbase + EXO_W2), dW3 = desc128(sbase + EXO_W3);
    const uint32_t id_fwd = idesc_bf16(128, 64, 0, 0), id_out = idesc_bf16(128, 16, 0, 0);

    const long long nrows = (p.total + p.stride - 1) / p.stride;
    const long long ntiles = (nrows + EX_T - 1) / EX_T;
    const AdvNorm an = adv_norm(p.moments, p.lagrange);
    double acc[6] = {0, 0, 0, 0, 0, 0};
    const int xm = tid >> 1, xh = (tid & 1) << 5;          // X gather: row, 32-column half
    const bool vec = (O & 3) == 0;
    const int s_row = 32 * q + lane;

    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        {   // X tile: row xm, columns xh .. xh + 31  (the previous tile's MMAs have completed: the buffer is free)
            const long long k = tile * EX_T + xm;
            const long long row = (k < nrows) ? k * p.stride : -1;
            if ((tid & 1) == 0) sRow[xm] = row;
#pragma unroll
            for (int c8 = 0; c8 < 4; ++c8) {
                float v[8];
                const int c0 = xh + 8 * c8;
                if (vec) {
#pragma unroll
                    for (int v4 = 0; v4 < 2; ++v4) {
                        const int c = c0 + 4 * v4;
                        const float4 x = (row >= 0 && c < O) ? __ldg(reinterpret_cast<const float4*>(p.obs + row * O + c))
                                                             : make_float4(0.f, 0.f, 0.f, 0.f);
                        v[4 * v4] = x.x; v[4 * v4 + 1] = x.y; v[4 * v4 + 2] = x.z; v[4 * v4 + 3] = x.w;
                    }
                } else {
#pragma unroll
                    for (int i = 0; i < 8; ++i) v[i] = (row >= 0 && c0 + i < O) ? __ldg(p.obs + row * O + c0 + i) : 0.f;
                }
                store8_x3(sbase + EXO_ACT, EX_SUB, xm, c0, v);
            }
        }
        fence_async_smem();
        __syncthreads();
        // per-sample inputs of the final statistics: requested now, they fly under the three layers
        const long long row = (h == 0) ? sRow[s_row] : -1;
        float pa[16], pm[16], plogp = 0.f, padvr = 0.f, padvc = 0.f;
#pragma unroll
        for (int a = 0; a < 16; ++a) { pa[a] = 0.f; pm[a] = 0.f; }
        if (row >= 0 && !p.mu_store) {
#pragma unroll
            for (int a = 0; a < 16; ++a)
                if (a < A) { pa[a] = __ldg(p.act + row * A + a); pm[a] = __ldg(p.mu_old + row * A + a); }
            plogp = __ldg(p.logp + row); padvr = __ldg(p.adv_r + row); padvc = __ldg(p.adv_c + row);
        }
        if (warp < 4) {
            gemm_x3(tm, C_Z, dAct, EX_SUB, 32u, dW1, EX_WSUB, 32u, id_fwd, 4, false);
            mma_commit_a(bar);
        }
        mbar_wait_a(bar, phase); phase ^= 1;
#pragma unroll
        for (int c8 = 0; c8 < 4; ++c8) {                    // H1 over X
            const int c0 = 32 * h + 8 * c8;
            float v[8];
            acc_ld8(tm, lane_base + C_Z + (uint32_t)c0, v);
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = tanh_acc(v[i] + sB1[c0 + i]);
            store8_x3(sbase + EXO_ACT, EX_SUB, s_row, c0, v);
        }
        fence_async_smem();
        __syncthreads();
        if (warp < 4) {
            gemm_x3(tm, C_Z, dAct, EX_SUB, 32u, dW2, EX_WSUB, 32u, id_fwd, 4, false);
            mma_commit_a(bar);
        }
        mbar_wait_a(bar, phase); phase ^= 1;
#pragma unroll
        for (int c8 = 0; c8 < 4; ++c8) {                    // H2 over H1
            const int c0 = 32 * h + 8 * c8;
            float v[8];
            acc_ld8(tm, lane_base + C_Z + (uint32_t)c0, v);
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = tanh_acc(v[i] + sB2[c0 + i]);
            store8_x3(sbase + EXO_ACT, EX_SUB, s_row, c0, v);
        }
        fence_async_smem();
        __syncthreads();
        if (warp < 4) {
            gemm_x3(tm, C_OUT, dAct, EX_SUB, 32u, dW3, EX_W3SUB, 32u, id_out, 4, false);
            mma_commit_a(bar);
        }
        mbar_wait_a(bar, phase); phase ^= 1;
        if (h == 0) {
            float o16[16];
            acc_ld16(tm, lane_base + C_OUT, o16);
            if (row >= 0) {
                if (p.mu_store) {
                    for (int a = 0; a < A; ++a) p.mu_store[row * A + a] = o16[a] + sB3[a];
                } else {
                    float mu[16];
#pragma unroll
                    for (int a = 0; a < 16; ++a) mu[a] = o16[a] + sB3[a];
                    eval_sample<16>(an, A, mu, pa, pm, plogp, padvr, padvc, sLs, acc);
                }
            }
        }
        __syncthreads();          // the OUT MMAs (readers of the buffer) completed; every thread is done with sRow
    }
    if (!p.mu_store) {
#pragma unroll
        for (int i = 0; i < 6; ++i) acc[i] = warp_sum(acc[i]);
        if (h == 0 && lane == 0)
            for (int i = 0; i < 6; ++i) sRedD[q * 8 + i] = acc[i];
        __syncthreads();
        if (tid < 6) p.part[(size_t)blockIdx.x * 8 + tid] = sRedD[tid] + sRedD[8 + tid] + sRedD[16 + tid] + sRedD[24 + tid];
    }
    __syncthreads();
}

}  // namespace osb

using namespace osb;

extern "C" {

// Split-bf16 variant of osb_actor_eval (O <= 64): same arguments and outputs, fp32-level accuracy.
int osb_actor_eval_x3(const float* theta_actor, int O, int A, const float* obs, const float* act,
                      const float* logp, const float* adv_r, const float* adv_c, const float* mu_old,
                      const float* logstd_old, const float* moments, const float* lagrange,
                      long long total, int stride, float* mu_store, double* workspace, double* out,
                      void* stream) {
    OSB_CHECK_ARG(theta_actor && obs && total > 0 && stride > 0 && O > 0 && O <= 64 && A > 0 && A <= 16, "bad argument (bf16x3 evaluation needs O <= 64)");
    OSB_CHECK_ARG(mu_store || (act && logp && adv_r && adv_c && mu_old && logstd_old && workspace && out), "null input");
    EvalX3Args p{obs, act, logp, adv_r, adv_c, mu_old, logstd_old, moments, lagrange, theta_actor, mu_store, workspace, nullptr, total, stride, O, A};
    const size_t smem = 1024 + EX_SMEM;
    static bool attr = false;
    if (!attr) {
        OSB_CUDA(cudaFuncSetAttribute(actor_eval_x3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr = true;
    }
    const long long nrows = (total + stride - 1) / stride;
    const long long tiles = (nrows + EX_T - 1) / EX_T;
    const int cap = 2 * grid_sms();
    const int blocks = (int)(tiles < cap ? tiles : cap);
    p.acc = acc_scratch(ACC_EVAL_X3, (size_t)blocks * 128 * EX_COLS * sizeof(float));
    if (!p.acc) return OSB_ERR_CUDA;
    cudaStream_t s = (cudaStream_t)stream;
    actor_eval_x3_kernel<<<blocks, EX_NT, smem, s>>>(p);
    OSB_LAUNCH_CHECK();
    return mu_store ? OSB_OK : eval_reduce(workspace, blocks, out, s);
}

}  // extern "C"
