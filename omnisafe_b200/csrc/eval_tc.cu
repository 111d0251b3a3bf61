// Tensor-core full-batch actor forward: the fast variants of actor_eval_kernel (csrc/update.cu), on the forward of
// csrc/tc_forward.cuh (X3 = false: tf32, O <= 512; X3 = true: split-bf16, O <= 64, fp32-level accuracy).  Stores
// mu(theta) per row (old-policy snapshot, trpo.py:L177 / policy_gradient.py:L383-392) or reduces sum KL(old||new),
// sum ratio*adv, sum ratio*adv_c, sum ratio, count, sum ratio*adv_r in fp64.
// Two CTAs per SM (~100 KB smem each) so one CTA's epilogue overlaps the other's MMA.
#include "common.cuh"
#include "loss.cuh"
#include "tc_forward.cuh"

namespace osb {

using namespace umma;

// the region after the operand tiles: floats b1[64] b2[64] b3[16] ls[64], then double red[4][8], long long rows[128]
constexpr int EW_B1 = 0, EW_B2 = 64, EW_B3 = 128, EW_LS = 144, EW_RED = 208, EW_ROWS = EW_RED + 2 * 32, EW_WORDS = EW_ROWS + 2 * TC_ROWS;

struct EvalTcArgs {
    const float* obs; const float* act; const float* logp; const float* adv_r; const float* adv_c;
    const float* mu_old; const float* logstd_old; const float* moments; const float* lagrange;
    const float* theta; float* mu_store; double* part;
    float* acc;         // accumulator images, [gridDim.x][128][TC_COLS]
    long long total; int stride, O, A;
};

template <bool X3>
__global__ void __launch_bounds__(NTHREADS, 2) actor_eval_tc_kernel(EvalTcArgs p) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const uint32_t pad = (1024u - (smem_u32(smem_raw) & 1023u)) & 1023u;
    const uint32_t B0 = smem_u32(smem_raw) + pad;
    float* fbase = reinterpret_cast<float*>(smem_raw + pad + TcTiles<X3>::FLOATS);
    float* sB1 = fbase + EW_B1;
    float* sB2 = fbase + EW_B2;
    float* sB3 = fbase + EW_B3;      // [16]
    float* sLs = fbase + EW_LS;      // [64] evaluation policy constants of csrc/loss.cuh
    double* sRedD = reinterpret_cast<double*>(fbase + EW_RED);       // [4][8]
    long long* sRow = reinterpret_cast<long long*>(fbase + EW_ROWS);  // [128]
    __shared__ uint64_t bar;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int q = warp & 3, h = warp >> 2;
    const int O = p.O, A = p.A;
    const NetLayout L = actor_layout(O, A);
    const float* theta = p.theta;
    tc_stage_weights<X3, 1>(B0, theta, L, O, sB1, sB2, sB3);   // batched, the bf16x3 staging costs this kernel 6 registers
    if (tid < 16)
        stage_eval_policy(sLs, tid, (tid < A) ? __ldg(theta + L.off_logstd + tid) : 0.f,
                          (tid < A && p.logstd_old) ? __ldg(p.logstd_old + tid) : 0.f);
    if (tid == 0) { mbar_init(&bar, 1); mbar_init_fence(); }
    fence_async_smem();
    __syncthreads();
    const Acc tm = acc_cta(p.acc, TC_COLS);
    const uint32_t lane_base = (uint32_t)(q * 32) << 16;
    uint32_t phase = 0;

    const int nchunks = X3 ? 1 : (O + 63) >> 6;
    const bool vec = (O & 3) == 0;
    const long long nrows = (p.total + p.stride - 1) / p.stride;
    const long long ntiles = (nrows + TC_ROWS - 1) / TC_ROWS;
    const AdvNorm an = adv_norm(p.moments, p.lagrange);
    double acc[6] = {0, 0, 0, 0, 0, 0};

    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        if (tid < TC_ROWS) {
            const long long k = tile * TC_ROWS + tid;
            sRow[tid] = (k < nrows) ? k * p.stride : -1;
        }
        __syncthreads();
        // per-sample inputs of the final statistics, requested early so that they fly under the MMAs: bf16x3 before the
        // forward, tf32 (whose epilogues hold more registers) once layer 2 completed
        const long long row = (h == 0) ? sRow[32 * q + lane] : -1;
        float pa[16], pm[16], plogp = 0.f, padvr = 0.f, padvc = 0.f;
        auto load_sample = [&] {
#pragma unroll
            for (int a = 0; a < 16; ++a) { pa[a] = 0.f; pm[a] = 0.f; }
            if (row >= 0 && !p.mu_store) {
#pragma unroll
                for (int a = 0; a < 16; ++a)
                    if (a < A) { pa[a] = __ldg(p.act + row * A + a); pm[a] = __ldg(p.mu_old + row * A + a); }
                plogp = __ldg(p.logp + row); padvr = __ldg(p.adv_r + row); padvc = __ldg(p.adv_c + row);
            }
        };
        if constexpr (X3) load_sample();
        tc_forward<X3>(
            B0, tm, &bar, phase, sB1, sB2, nchunks,
            [&](int c) { tc_stage_rows<X3>(B0, p.obs, O, vec, c, theta, L, [&](int m) { return sRow[m]; }); },
            [&](int l) {
                if (!X3 && l == 2) load_sample();
            });
        if (h == 0) {
            float o16[16];
            acc_ld16(tm, lane_base + TC_C_OUT, o16);
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

// 1024: the alignment pad in front of the operand tiles
template <bool X3>
static int actor_eval_tc(const float* theta_actor, int O, int A, const float* obs, const float* act, const float* logp,
                         const float* adv_r, const float* adv_c, const float* mu_old, const float* logstd_old,
                         const float* moments, const float* lagrange, long long total, int stride, float* mu_store,
                         double* workspace, double* out, void* stream) {
    EvalTcArgs p{obs, act, logp, adv_r, adv_c, mu_old, logstd_old, moments, lagrange, theta_actor, mu_store, workspace, nullptr, total, stride, O, A};
    const size_t smem = 1024 + TcTiles<X3>::FLOATS + EW_WORDS * sizeof(float);
    static bool attr = false;
    if (!attr) {
        OSB_CUDA(cudaFuncSetAttribute(actor_eval_tc_kernel<X3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr = true;
    }
    const long long nrows = (total + stride - 1) / stride;
    const long long tiles = (nrows + TC_ROWS - 1) / TC_ROWS;
    const int cap = 2 * grid_sms();
    const int blocks = (int)(tiles < cap ? tiles : cap);
    p.acc = acc_scratch(X3 ? ACC_EVAL_X3 : ACC_EVAL_TC, (size_t)blocks * 128 * TC_COLS * sizeof(float));
    if (!p.acc) return OSB_ERR_CUDA;
    cudaStream_t s = (cudaStream_t)stream;
    actor_eval_tc_kernel<X3><<<blocks, NTHREADS, smem, s>>>(p);
    OSB_LAUNCH_CHECK();
    return mu_store ? OSB_OK : eval_reduce(workspace, blocks, out, s);
}

}  // namespace osb

using namespace osb;

extern "C" {

// Tensor-core variant of osb_actor_eval (O <= 512; layer 1 K-chunked above 64); same arguments and outputs.
int osb_actor_eval_tc(const float* theta_actor, int O, int A, const float* obs, const float* act,
                      const float* logp, const float* adv_r, const float* adv_c, const float* mu_old,
                      const float* logstd_old, const float* moments, const float* lagrange,
                      long long total, int stride, float* mu_store, double* workspace, double* out,
                      void* stream) {
    OSB_CHECK_ARG(theta_actor && obs && total > 0 && stride > 0 && O > 0 && O <= 512 && A > 0 && A <= 16, "bad argument (O <= 512)");
    OSB_CHECK_ARG(mu_store || (act && logp && adv_r && adv_c && mu_old && logstd_old && workspace && out), "null input");
    return actor_eval_tc<false>(theta_actor, O, A, obs, act, logp, adv_r, adv_c, mu_old, logstd_old, moments, lagrange,
                                total, stride, mu_store, workspace, out, stream);
}

// Split-bf16 variant of osb_actor_eval (O <= 64): same arguments and outputs, fp32-level accuracy.
int osb_actor_eval_x3(const float* theta_actor, int O, int A, const float* obs, const float* act,
                      const float* logp, const float* adv_r, const float* adv_c, const float* mu_old,
                      const float* logstd_old, const float* moments, const float* lagrange,
                      long long total, int stride, float* mu_store, double* workspace, double* out,
                      void* stream) {
    OSB_CHECK_ARG(theta_actor && obs && total > 0 && stride > 0 && O > 0 && O <= 64 && A > 0 && A <= 16, "bad argument (bf16x3 evaluation needs O <= 64)");
    OSB_CHECK_ARG(mu_store || (act && logp && adv_r && adv_c && mu_old && logstd_old && workspace && out), "null input");
    return actor_eval_tc<true>(theta_actor, O, A, obs, act, logp, adv_r, adv_c, mu_old, logstd_old, moments, lagrange,
                               total, stride, mu_store, workspace, out, stream);
}

}  // extern "C"
