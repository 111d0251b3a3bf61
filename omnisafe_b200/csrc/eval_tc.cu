// Tensor-core (wgmma, TF32) full-batch actor forward: the fast variant of actor_eval_kernel
// (csrc/update.cu).  Stores mu(theta) per row (old-policy snapshot) or reduces
// sum KL(old||new), sum ratio*adv, sum ratio*adv_c, sum ratio, count, sum ratio*adv_r in fp64.
// Two CTAs per SM (~100 KB smem each) so one CTA's epilogue overlaps the other's MMA.
#include "common.cuh"
#include "loss.cuh"
#include "mlp.cuh"
#include "umma.cuh"

namespace osb {

using namespace umma;

constexpr int ET = 128;
constexpr uint32_t EBUF = ET * 64 * 4;
constexpr uint32_t E_COLS = 80;            // accumulator columns: Z [0, 64), OUT [64, 80)

struct EvalTcArgs {
    const float* obs; const float* act; const float* logp; const float* adv_r; const float* adv_c;
    const float* mu_old; const float* logstd_old; const float* moments; const float* lagrange;
    const float* theta; float* mu_store; double* part;
    float* acc;         // accumulator images, [gridDim.x][128][E_COLS]
    long long total; int stride, O, A;
};

__global__ void __launch_bounds__(NTHREADS, 2) actor_eval_tc_kernel(EvalTcArgs p) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const uint32_t pad = (1024u - (smem_u32(smem_raw) & 1023u)) & 1023u;
    const uint32_t B0 = smem_u32(smem_raw) + pad;   // X -> H2
    const uint32_t B2 = B0 + EBUF;                  // H1
    const uint32_t sW1 = B2 + EBUF, sW2 = sW1 + 16384, sW3 = sW2 + 16384;
    float* sB1 = reinterpret_cast<float*>(smem_raw + pad + 2 * EBUF + 2 * 16384 + 4096);
    float* sB2 = sB1 + 64;
    float* sB3 = sB2 + 64;      // [16]
    float* sLs = sB3 + 16;      // [64] evaluation policy constants of csrc/loss.cuh
    double* sRedD = reinterpret_cast<double*>(sLs + 64);       // [4][8]
    long long* sRow = reinterpret_cast<long long*>(sRedD + 32);  // [128]
    __shared__ uint64_t bar;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int q = warp & 3, h = warp >> 2;
    const int O = p.O, A = p.A;
    const NetLayout L = actor_layout(O, A);
    const float* theta = p.theta;
    {
        float w1v[16], w2v[16], w3v[4];
        const int k = tid & 63;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const int n = (tid >> 6) + 4 * j;
            w1v[j] = (k < O && O <= 64) ? __ldg(theta + L.off_w1 + n * O + k) : 0.f;
            w2v[j] = __ldg(theta + L.off_w2 + n * 64 + k);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int o = (tid >> 6) + 4 * j;
            w3v[j] = (o < A) ? __ldg(theta + L.off_w3 + o * 64 + k) : 0.f;
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
    if (tid < 16) {
        sB3[tid] = (tid < A) ? __ldg(theta + L.off_b3 + tid) : 0.f;
        stage_eval_policy(sLs, tid, (tid < A) ? __ldg(theta + L.off_logstd + tid) : 0.f,
                          (tid < A && p.logstd_old) ? __ldg(p.logstd_old + tid) : 0.f);
    }
    if (tid == 0) { mbar_init(&bar, 1); mbar_init_fence(); }
    __syncthreads();
    const Acc tm = acc_cta(p.acc, E_COLS);
    const uint32_t lane_base = (uint32_t)(q * 32) << 16;
    constexpr uint32_t C_Z = 0, C_OUT = 64;
    uint32_t phase = 0;

    const int nchunks = (O + 63) >> 6;
    const long long nrows = (p.total + p.stride - 1) / p.stride;
    const long long ntiles = (nrows + ET - 1) / ET;
    const AdvNorm an = adv_norm(p.moments, p.lagrange);
    double acc[6] = {0, 0, 0, 0, 0, 0};

    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        if (tid < ET) {
            const long long k = tile * ET + tid;
            sRow[tid] = (k < nrows) ? k * p.stride : -1;
        }
        __syncthreads();
        for (int c = 0; c < nchunks; ++c) {     // layer 1 as a K loop over 64-column chunks of X / W1 (one chunk if O <= 64)
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
                    const long long row = sRow[(tid >> 6) + 4 * (16 * half + j)];
                    xv[j] = (row >= 0 && col < O) ? __ldg(p.obs + row * O + col) : 0.f;
                }
#pragma unroll
                for (int j = 0; j < 16; ++j) sts(tile_addr(B0, (tid >> 6) + 4 * (16 * half + j), k, ET), tf32r(xv[j]));
            }
            fence_async_smem();
            __syncthreads();
            if (warp < 4) { tc_gemm(tm, C_Z, B0, ET, sW1, 64, 128, 64, 64, c > 0); mma_commit(&bar); }
            mbar_wait(&bar, phase); phase ^= 1;
        }
        {
            float v[32];
            acc_ld32(tm, lane_base + C_Z + 32 * h, v);
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] = tanh_fast(v[i] + sB1[32 * h + i]);
            store_row32(B2, 32 * q + lane, 32 * h, ET, v);
        }
        fence_async_smem();
        __syncthreads();
        if (warp < 4) { tc_gemm(tm, C_Z, B2, ET, sW2, 64, 128, 64, 64, false); mma_commit(&bar); }
        mbar_wait(&bar, phase); phase ^= 1;
        {
            float v[32];
            acc_ld32(tm, lane_base + C_Z + 32 * h, v);
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] = tanh_fast(v[i] + sB2[32 * h + i]);
            store_row32(B0, 32 * q + lane, 32 * h, ET, v);
        }
        fence_async_smem();
        __syncthreads();
        if (warp < 4) { tc_gemm(tm, C_OUT, B0, ET, sW3, 16, 128, 16, 64, false); mma_commit(&bar); }
        // per-sample scalars: requested before the wait (warps 4-7 while warpgroup 0 computes the output layer)
        const long long row = (h == 0) ? sRow[32 * q + lane] : -1;
        float pa[16], pm[16], plogp = 0.f, padvr = 0.f, padvc = 0.f;
#pragma unroll
        for (int a = 0; a < 16; ++a) { pa[a] = 0.f; pm[a] = 0.f; }
        if (row >= 0 && !p.mu_store) {
#pragma unroll
            for (int a = 0; a < 16; ++a)
                if (a < A) { pa[a] = __ldg(p.act + row * A + a); pm[a] = __ldg(p.mu_old + row * A + a); }
            plogp = __ldg(p.logp + row); padvr = __ldg(p.adv_r + row); padvc = __ldg(p.adv_c + row);
        }
        mbar_wait(&bar, phase); phase ^= 1;
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
        __syncthreads();
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

// Tensor-core variant of osb_actor_eval (O <= 512; layer 1 K-chunked above 64); same arguments and outputs.
int osb_actor_eval_tc(const float* theta_actor, int O, int A, const float* obs, const float* act,
                      const float* logp, const float* adv_r, const float* adv_c, const float* mu_old,
                      const float* logstd_old, const float* moments, const float* lagrange,
                      long long total, int stride, float* mu_store, double* workspace, double* out,
                      void* stream) {
    OSB_CHECK_ARG(theta_actor && obs && total > 0 && stride > 0 && O > 0 && O <= 512 && A > 0 && A <= 16, "bad argument (O <= 512)");
    OSB_CHECK_ARG(mu_store || (act && logp && adv_r && adv_c && mu_old && logstd_old && workspace && out), "null input");
    EvalTcArgs p{obs, act, logp, adv_r, adv_c, mu_old, logstd_old, moments, lagrange, theta_actor, mu_store, workspace, nullptr, total, stride, O, A};
    const size_t smem = 1024 + 2 * (size_t)EBUF + 2 * 16384 + 4096 + (64 + 64 + 16 + 64) * 4 + 32 * 8 + 128 * 8 + 64;
    static bool attr = false;
    if (!attr) {
        OSB_CUDA(cudaFuncSetAttribute(actor_eval_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr = true;
    }
    const long long nrows = (total + stride - 1) / stride;
    const long long tiles = (nrows + ET - 1) / ET;
    const int cap = 2 * grid_sms();
    const int blocks = (int)(tiles < cap ? tiles : cap);
    p.acc = acc_scratch(ACC_EVAL_TC, (size_t)blocks * 128 * E_COLS * sizeof(float));
    if (!p.acc) return OSB_ERR_CUDA;
    cudaStream_t s = (cudaStream_t)stream;
    actor_eval_tc_kernel<<<blocks, NTHREADS, smem, s>>>(p);
    OSB_LAUNCH_CHECK();
    return mu_store ? OSB_OK : eval_reduce(workspace, blocks, out, s);
}

}  // extern "C"
