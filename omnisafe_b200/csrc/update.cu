// Fused learner kernels: minibatch forward + loss + backward of the actor / reward-critic /
// cost-critic trunks (fp32 FMA parity path), full-batch actor evaluation (KL / surrogates) and the
// Fisher-vector product for CPO / TRPO-Lag.
//
// Replaces the reference's
//   PolicyGradient._update minibatch body   algorithms/on_policy/base/policy_gradient.py:L369-381
//   _update_reward_critic / _update_cost_critic / _update_actor            :L407-524
//   NaturalPG._fvp                          base/natural_pg.py:L74-119  (analytic Gauss-Newton form)
// with the per-sample losses and evaluation statistics of csrc/loss.cuh.
//
// One CTA = one network x a strided set of 128-sample tiles.  Samples are addressed by slab row
// (t*N + i); a minibatch is a window of the sample order of csrc/loss.cuh (supplied permutation or
// keyed Feistel bijection) -- no gather buffers are materialised.
#include "common.cuh"
#include "loss.cuh"
#include "mlp.cuh"

namespace osb {

constexpr int UT = 128;  // samples per tile
static_assert(OUTP == 16, "policy constants of csrc/loss.cuh are laid out 16 per field");

// stats slots (per launch, summed over CTAs in fixed order)
enum { ST_N = 8 };

struct GradArgs {
    Batch b;
    LossParams lc;
    const float* theta;
    float* gpart;          // [gridDim.x][P] partial gradients (each CTA writes its network's segment)
    float* stats_part;     // [gridDim.x][3][ST_N]
    const int* stop_flag;  // device flag: non-zero -> kernel is a no-op (KL early stop)
    int O, A, P;
    int net_mask;          // bit n set -> process network n
    int forward_only;      // pass 1 of FOCOPS / P3O: actor forward + statistics only (no gradients written)
};

// gather chunk kc of the observation rows of a tile into sX (zero padded)
__device__ __forceinline__ void gather_obs(const float* __restrict__ obs, const long long* sRow, int O,
                                           int kc, float* sX) {
    const int c0 = kc * KC;
    for (int i = threadIdx.x; i < UT * KC; i += NTHREADS) {
        const int m = i / KC, k = i % KC;
        const long long row = sRow[m];
        const int j = c0 + k;
        sX[m * LD + k] = (row >= 0 && j < O) ? __ldg(obs + row * O + j) : 0.f;
    }
}

// deterministic CTA reduction of `nv` per-thread values held by threads < UT (4 warps).
template <int NV>
__device__ __forceinline__ void block_reduce_store(float (&v)[NV], float* sRed, float* out, bool add) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < NV; ++i) v[i] = warp_sum(v[i]);
    if (w < UT / 32 && lane == 0)
#pragma unroll
        for (int i = 0; i < NV; ++i) sRed[w * NV + i] = v[i];
    __syncthreads();
    if (threadIdx.x < NV) {
        float s = 0.f;
        for (int ww = 0; ww < UT / 32; ++ww) s += sRed[ww * NV + threadIdx.x];
        out[threadIdx.x] = add ? out[threadIdx.x] + s : s;
    }
    __syncthreads();
}

__global__ void __launch_bounds__(NTHREADS, 1) minibatch_grad_kernel(GradArgs p) {
    if (p.stop_flag && *p.stop_flag) return;
    const int net = blockIdx.y;
    if (!((p.net_mask >> net) & 1)) return;

    extern __shared__ __align__(16) float smem[];
    NetSmem W;
    float* base = carve_net_smem<true>(smem, W);
    float* sX = base;  base += UT * LD;
    float* sH1 = base; base += UT * LD;
    float* sH2 = base; base += UT * LD;
    float* sD = base;  base += UT * LD;
    float* sO = base;  base += UT * LDO;
    float* sRed = base; base += 4 * 2 * OUTP;
    float* sPol = base; base += 3 * OUTP;   // policy constants of csrc/loss.cuh
    float* sOld = base; base += 2 * OUTP;
    float* sDls = base; base += OUTP;       // accumulated d log_std
    float* sStat = base; base += ST_N;
    long long* sRow = reinterpret_cast<long long*>(base);  // [UT] (8-byte aligned: offsets are even)

    const int O = p.O, A = p.A;
    const int nchunks = (O + KC - 1) / KC;
    const NetLayout L = net_layout(net, O, A);
    const int noff = net_offset(net, O, A);
    const float* theta = p.theta + noff;
    float* gout = p.gpart + (size_t)blockIdx.x * p.P + noff;
    const int ntiles = (p.b.mb_count + UT - 1) / UT;
    const float inv_b = 1.0f / (float)p.b.mb_count;

    load_net_rest<true>(theta, L, W);
    load_w1_chunk(theta, L, 0, W);
    if (threadIdx.x < OUTP) {
        const bool act = net == 0 && threadIdx.x < A;
        stage_policy(sPol, threadIdx.x, act ? __ldg(theta + L.off_logstd + threadIdx.x) : 0.f);
        stage_policy_old(sOld, threadIdx.x, (act && p.lc.logstd_old) ? __ldg(p.lc.logstd_old + threadIdx.x) : 0.f);
        sDls[threadIdx.x] = 0.f;
    }
    if (threadIdx.x < ST_N) sStat[threadIdx.x] = 0.f;

    float aw1[4][4], aw2[4][4], aw3[4];
    float ab1 = 0.f, ab2 = 0.f, ab3 = 0.f;
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        aw3[a] = 0.f;
#pragma unroll
        for (int b = 0; b < 4; ++b) { aw1[a][b] = 0.f; aw2[a][b] = 0.f; }
    }
    const AdvNorm an = adv_norm(p.b.moments, p.lc.lagrange);
    bool first_tile = true;

    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        __syncthreads();
        if (threadIdx.x < UT) {
            const int local = tile * UT + threadIdx.x;
            sRow[threadIdx.x] = (local < p.b.mb_count) ? sample_row(p.b, p.b.mb_start + local) : -1;
        }
        __syncthreads();
        gather_obs(p.b.obs, sRow, O, 0, sX);
        if (nchunks > 1) load_w1_chunk(theta, L, 0, W);
        __syncthreads();
        auto load_chunk = [&](int kc) { load_w1_chunk(theta, L, kc, W); gather_obs(p.b.obs, sRow, O, kc, sX); };
        mlp_hidden<UT>(sX, sH1, sH2, W, nchunks, load_chunk);
        mlp_out<UT>(sH2, sO, W, L.out);

        // ---- per-sample loss and dL/dOUT (threads < UT), dOUT overwrites sO ---------------------
        {
            float st[5] = {0.f, 0.f, 0.f, 0.f, 0.f};   // loss, ratio, kl, count, focops mask
            float dls[OUTP];
#pragma unroll
            for (int a = 0; a < OUTP; ++a) dls[a] = 0.f;
            if (threadIdx.x < UT) {
                const int m = threadIdx.x;
                const long long row = sRow[m];
                if (row < 0) {
                    for (int o = 0; o < OUTP; ++o) sO[m * LDO + o] = 0.f;
                } else if (net != 0) {
                    const float v = sO[m * LDO];
                    const float tgt = __ldg((net == 1 ? p.b.tv_r : p.b.tv_c) + row);
                    const float d = v - tgt;
                    st[0] = d * d;
                    st[3] = 1.f;
                    sO[m * LDO] = 2.f * d * inv_b;                       // d mse / d v
                    for (int o = 1; o < OUTP; ++o) sO[m * LDO + o] = 0.f;
                } else {
                    float mu[OUTP], act[OUTP];
#pragma unroll
                    for (int a = 0; a < OUTP; ++a) {
                        mu[a] = 0.f; act[a] = 0.f;
                        if (a < A) {
                            mu[a] = sO[m * LDO + a];
                            act[a] = __ldg(p.b.act + row * A + a);
                        }
                    }
                    // dOUT overwrites OUT: columns >= A are zero
                    for (int a = A; a < OUTP; ++a) sO[m * LDO + a] = 0.f;
                    actor_sample_loss<true, OUTP>(p.lc, an, A, inv_b, mu, act,
                                                                       [&](int a) { return __ldg(p.lc.mu_old + row * A + a); },
                                                                       __ldg(p.b.logp + row),
                                                                       __ldg(p.b.adv_r + row), __ldg(p.b.adv_c + row), sPol, sOld, st,
                                                                       [&](int a, float dm, float dl) { sO[m * LDO + a] = dm; dls[a] = dl; });
                }
            }
            block_reduce_store<5>(st, sRed, sStat, true);
            if (net == 0) block_reduce_store<OUTP>(dls, sRed, sDls, true);
        }
        __syncthreads();
        if (p.forward_only) { first_tile = false; continue; }

        // ---- backward ---------------------------------------------------------------------------
        {   // dW3[o][k] += sum_s dOUT[s][o] * H2[s][k];  db3[o] += sum_s dOUT[s][o]
            const int k = threadIdx.x & 63, og = threadIdx.x >> 6;
            for (int s = 0; s < UT; ++s) {
                const float h = sH2[s * LD + k];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int o = og + 4 * i;
                    if (o < L.out) aw3[i] = fmaf(sO[s * LDO + o], h, aw3[i]);
                }
            }
            if (threadIdx.x < L.out) {
                float c = 0.f;
                for (int s = 0; s < UT; ++s) c += sO[s * LDO + threadIdx.x];
                ab3 += c;
            }
        }
        {   // dZ2 = (dOUT . W3) * (1 - H2^2) -> sD
            float acc[UT / 16][4];
            gemm_nt<UT, LDO, LDO>(sO, W.w3t, OUTP, acc);
            const int tm = threadIdx.x >> 4, tn = threadIdx.x & 15;
#pragma unroll
            for (int i = 0; i < UT / 16; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int mm = tm + 16 * i, n = tn + 16 * j;
                    const float h = sH2[mm * LD + n];
                    sD[mm * LD + n] = acc[i][j] * (1.f - h * h);
                }
        }
        __syncthreads();
        {   // dW2 += dZ2^T . H1 ; db2
            float acc[4][4];
            gemm_tn<UT, LD, LD>(sD, sH1, acc);
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
                for (int b = 0; b < 4; ++b) aw2[a][b] += acc[a][b];
            if (threadIdx.x < HID) {
                float c = 0.f;
                for (int s = 0; s < UT; ++s) c += sD[s * LD + threadIdx.x];
                ab2 += c;
            }
        }
        {   // dZ1 = (dZ2 . W2) * (1 - H1^2) -> sH2 (H2 is dead now)
            float acc[UT / 16][4];
            gemm_nt<UT, LD, LD>(sD, W.w2t, HID, acc);
            __syncthreads();   // all reads of sH2 (dW3 above) and sD are done before overwriting sH2
            const int tm = threadIdx.x >> 4, tn = threadIdx.x & 15;
#pragma unroll
            for (int i = 0; i < UT / 16; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int mm = tm + 16 * i, n = tn + 16 * j;
                    const float h = sH1[mm * LD + n];
                    sH2[mm * LD + n] = acc[i][j] * (1.f - h * h);
                }
        }
        __syncthreads();
        {   // dW1 += dZ1^T . X (per obs chunk) ; db1
            if (threadIdx.x < HID) {
                float c = 0.f;
                for (int s = 0; s < UT; ++s) c += sH2[s * LD + threadIdx.x];
                ab1 += c;
            }
            if (nchunks == 1) {
                float acc[4][4];
                gemm_tn<UT, LD, LD>(sH2, sX, acc);
#pragma unroll
                for (int a = 0; a < 4; ++a)
#pragma unroll
                    for (int b = 0; b < 4; ++b) aw1[a][b] += acc[a][b];
            } else {
                const int j0 = (threadIdx.x >> 4) * 4, k0 = (threadIdx.x & 15) * 4;
                for (int kc = 0; kc < nchunks; ++kc) {
                    __syncthreads();
                    gather_obs(p.b.obs, sRow, O, kc, sX);
                    __syncthreads();
                    float acc[4][4];
                    gemm_tn<UT, LD, LD>(sH2, sX, acc);
#pragma unroll
                    for (int a = 0; a < 4; ++a)
#pragma unroll
                        for (int b = 0; b < 4; ++b) {
                            const int col = kc * KC + k0 + b;
                            if (col < O) {
                                float* g = gout + L.off_w1 + (j0 + a) * O + col;
                                *g = first_tile ? acc[a][b] : *g + acc[a][b];
                            }
                        }
                }
            }
        }
        first_tile = false;
    }

    // ---- write this CTA's partial gradient segment ----------------------------------------------
    if (p.forward_only) {
        __syncthreads();
        if (threadIdx.x < ST_N)
            p.stats_part[((size_t)blockIdx.x * 3 + net) * ST_N + threadIdx.x] = sStat[threadIdx.x];
        return;
    }
    {
        const int j0 = (threadIdx.x >> 4) * 4, k0 = (threadIdx.x & 15) * 4;
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b) {
                gout[L.off_w2 + (j0 + a) * HID + k0 + b] = aw2[a][b];
                if (nchunks == 1 && k0 + b < O) gout[L.off_w1 + (j0 + a) * O + k0 + b] = aw1[a][b];
            }
        if (nchunks > 1 && first_tile)   // CTA without tiles: zero its W1 segment
            for (int i = threadIdx.x; i < HID * O; i += NTHREADS) gout[L.off_w1 + i] = 0.f;
        const int k = threadIdx.x & 63, og = threadIdx.x >> 6;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int o = og + 4 * i;
            if (o < L.out) gout[L.off_w3 + o * HID + k] = aw3[i];
        }
        if (threadIdx.x < HID) { gout[L.off_b1 + threadIdx.x] = ab1; gout[L.off_b2 + threadIdx.x] = ab2; }
        if (threadIdx.x < L.out) gout[L.off_b3 + threadIdx.x] = ab3;
        __syncthreads();
        if (net == 0 && threadIdx.x < A) {
            float g = sDls[threadIdx.x];
            // entropy bonus: loss -= coef * mean(entropy); d entropy / d log_std_a = 1 (mean over A)
            if (blockIdx.x == 0 && loss_has_entropy(p.lc.kind)) g -= p.lc.entropy_coef / (float)A;
            gout[L.off_logstd + threadIdx.x] = g;
        }
        if (threadIdx.x < ST_N)
            p.stats_part[((size_t)blockIdx.x * 3 + net) * ST_N + threadIdx.x] = sStat[threadIdx.x];
    }
}

// ---------------------------------------------------------------------------------------------
// Full-batch actor evaluation: mu_new for every sample, then either store it (old policy snapshot)
// or reduce  sum KL(old||new), sum ratio*adv, sum ratio*adv_c, sum ratio  (fp64 partials).
struct EvalArgs {
    Batch b;                 // perm unused: rows [0, total)
    const float* mu_old;     // [rows][A]
    const float* theta;      // actor parameters (first segment of flat theta, or a trial vector)
    const float* logstd_old; // [A]
    const float* lagrange;   // lambda or null
    float* mu_store;         // [rows][A] or null
    double* part;            // [gridDim.x][8]
    int O, A;
    int stride;              // evaluate rows 0, stride, 2*stride, ... (fvp_sample_freq)
};

__global__ void __launch_bounds__(NTHREADS, 1) actor_eval_kernel(EvalArgs p) {
    extern __shared__ __align__(16) float smem[];
    NetSmem W;
    float* base = carve_net_smem<false>(smem, W);
    float* sX = base;  base += UT * LD;
    float* sH1 = base; base += UT * LD;
    float* sH2 = base; base += UT * LD;
    float* sO = base;  base += UT * LDO;
    float* sPol = base; base += 4 * OUTP;   // evaluation policy constants of csrc/loss.cuh
    double* sRedD = reinterpret_cast<double*>(base); base += 2 * 4 * 8;
    long long* sRow = reinterpret_cast<long long*>(base);

    const int O = p.O, A = p.A;
    const int nchunks = (O + KC - 1) / KC;
    const NetLayout L = actor_layout(O, A);
    load_net_rest<false>(p.theta, L, W);
    load_w1_chunk(p.theta, L, 0, W);
    if (threadIdx.x < OUTP) {
        const bool act = threadIdx.x < A;
        stage_eval_policy(sPol, threadIdx.x, act ? __ldg(p.theta + L.off_logstd + threadIdx.x) : 0.f,
                          (act && p.logstd_old) ? __ldg(p.logstd_old + threadIdx.x) : 0.f);
    }
    const long long nrows = (p.b.total + p.stride - 1) / p.stride;
    const long long ntiles = (nrows + UT - 1) / UT;
    const AdvNorm an = adv_norm(p.b.moments, p.lagrange);
    double acc[6] = {0, 0, 0, 0, 0, 0};  // kl, ratio*adv, ratio*adv_c, ratio, count, ratio*adv_r(std)

    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        __syncthreads();
        if (threadIdx.x < UT) {
            const long long k = tile * UT + threadIdx.x;
            sRow[threadIdx.x] = (k < nrows) ? k * p.stride : -1;
        }
        __syncthreads();
        gather_obs(p.b.obs, sRow, O, 0, sX);
        if (nchunks > 1) load_w1_chunk(p.theta, L, 0, W);
        __syncthreads();
        auto load_chunk = [&](int kc) { load_w1_chunk(p.theta, L, kc, W); gather_obs(p.b.obs, sRow, O, kc, sX); };
        mlp_hidden<UT>(sX, sH1, sH2, W, nchunks, load_chunk);
        mlp_out<UT>(sH2, sO, W, A);
        if (threadIdx.x < UT) {
            const long long row = sRow[threadIdx.x];
            if (row >= 0) {
                if (p.mu_store) {
                    for (int a = 0; a < A; ++a) p.mu_store[row * A + a] = sO[threadIdx.x * LDO + a];
                } else {
                    float mu[OUTP], act[OUTP], mo[OUTP];
#pragma unroll
                    for (int a = 0; a < OUTP; ++a) {
                        mu[a] = 0.f; act[a] = 0.f; mo[a] = 0.f;
                        if (a < A) {
                            mu[a] = sO[threadIdx.x * LDO + a];
                            act[a] = __ldg(p.b.act + row * A + a);
                            mo[a] = __ldg(p.mu_old + row * A + a);
                        }
                    }
                    eval_sample<OUTP>(an, A, mu, act, mo, __ldg(p.b.logp + row), __ldg(p.b.adv_r + row),
                                      __ldg(p.b.adv_c + row), sPol, acc);
                }
            }
        }
    }
    if (!p.mu_store) {
        __syncthreads();
        const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
        for (int i = 0; i < 6; ++i) acc[i] = warp_sum(acc[i]);
        if (lane == 0)
            for (int i = 0; i < 6; ++i) sRedD[w * 8 + i] = acc[i];
        __syncthreads();
        if (threadIdx.x < 6) {
            double s = 0.0;
            for (int ww = 0; ww < NTHREADS / 32; ++ww) s += sRedD[ww * 8 + threadIdx.x];
            p.part[(size_t)blockIdx.x * 8 + threadIdx.x] = s;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Fisher-vector product of the Gaussian policy (analytic Gauss-Newton form of NaturalPG._fvp):
//   F v = [ (2/A) v_logstd ;  (1/(B A)) sum_s J_mu(s)^T diag(sigma^-2) J_mu(s) v_mu ]
// computed per tile as a forward-mode tangent pass (JVP) followed by the ordinary backward (VJP).
struct FvpArgs {
    const float* obs;
    long long total;
    int stride;
    const float* theta;   // actor params
    const float* vec;     // [P_actor] direction
    float* gpart;         // [gridDim.x][P_actor]
    int O, A;
};

__device__ __forceinline__ void load_mat64(const float* __restrict__ src, int ld_src, int col0,
                                           int ncols_valid, float* dst) {
    // dst[n][k] (LD stride) <- src[n*ld_src + col0 + k], zero padded, n < 64, k < 64
    for (int i = threadIdx.x; i < HID * KC; i += NTHREADS) {
        const int n = i / KC, k = i % KC;
        dst[n * LD + k] = (k < ncols_valid) ? __ldg(src + n * ld_src + col0 + k) : 0.f;
    }
}

__global__ void __launch_bounds__(NTHREADS, 1) fvp_kernel(FvpArgs p) {
    extern __shared__ __align__(16) float smem[];
    NetSmem W;
    float* base = carve_net_smem<true>(smem, W);
    float* vslot = base; base += HID * LD;    // V.w1 chunk during layer 1, then V.w2
    float* vw3 = base;   base += OUTP * LD;
    float* vb1 = base;   base += HID;
    float* vb2 = base;   base += HID;
    float* vb3 = base;   base += OUTP;
    float* sX = base;  base += UT * LD;       // X chunk; aliased as sT (tangents / dZ2) in between
    float* sH1 = base; base += UT * LD;
    float* sH2 = base; base += UT * LD;
    float* sO = base;  base += UT * LDO;
    float* sSig = base; base += OUTP;
    long long* sRow = reinterpret_cast<long long*>(base);
    float* sT = sX;

    const int O = p.O, A = p.A;
    const int nchunks = (O + KC - 1) / KC;
    const NetLayout L = actor_layout(O, A);
    float* gout = p.gpart + (size_t)blockIdx.x * L.size;
    load_net_rest<true>(p.theta, L, W);
    for (int i = threadIdx.x; i < OUTP * HID; i += NTHREADS) {
        const int o = i / HID, k = i % HID;
        vw3[o * LD + k] = (o < A) ? __ldg(p.vec + L.off_w3 + o * HID + k) : 0.f;
    }
    if (threadIdx.x < HID) {
        vb1[threadIdx.x] = __ldg(p.vec + L.off_b1 + threadIdx.x);
        vb2[threadIdx.x] = __ldg(p.vec + L.off_b2 + threadIdx.x);
    }
    if (threadIdx.x < OUTP) {
        vb3[threadIdx.x] = threadIdx.x < A ? __ldg(p.vec + L.off_b3 + threadIdx.x) : 0.f;
        sSig[threadIdx.x] = threadIdx.x < A ? expf(__ldg(p.theta + L.off_logstd + threadIdx.x)) : 1.f;
    }
    const long long nrows = (p.total + p.stride - 1) / p.stride;
    const long long ntiles = (nrows + UT - 1) / UT;
    const float scale = 1.0f / ((float)nrows * (float)A);

    float aw1[4][4], aw2[4][4], aw3[4];
    float ab1 = 0.f, ab2 = 0.f, ab3 = 0.f;
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        aw3[a] = 0.f;
#pragma unroll
        for (int b = 0; b < 4; ++b) { aw1[a][b] = 0.f; aw2[a][b] = 0.f; }
    }
    bool first_tile = true;
    const int tm = threadIdx.x >> 4, tn = threadIdx.x & 15;

    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        __syncthreads();
        if (threadIdx.x < UT) {
            const long long k = tile * UT + threadIdx.x;
            sRow[threadIdx.x] = (k < nrows) ? k * p.stride : -1;
        }
        __syncthreads();
        // layer 1: Z1 = X W1^T + b1, tangent dZ1 = X V1^T + vb1 (chunked over obs dims)
        float z[UT / 16][4], dz[UT / 16][4], acc[UT / 16][4];
#pragma unroll
        for (int i = 0; i < UT / 16; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) { z[i][j] = 0.f; dz[i][j] = 0.f; }
        for (int kc = 0; kc < nchunks; ++kc) {
            if (kc > 0) __syncthreads();
            gather_obs(p.obs, sRow, O, kc, sX);
            load_w1_chunk(p.theta, L, kc, W);
            load_mat64(p.vec + L.off_w1, O, kc * KC, min(KC, O - kc * KC), vslot);
            __syncthreads();
            gemm_nt<UT, LD, LD>(sX, W.w1, KC, acc);
#pragma unroll
            for (int i = 0; i < UT / 16; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) z[i][j] += acc[i][j];
            gemm_nt<UT, LD, LD>(sX, vslot, KC, acc);
#pragma unroll
            for (int i = 0; i < UT / 16; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) dz[i][j] += acc[i][j];
        }
        __syncthreads();   // sX / vslot fully consumed: sT aliases sX, vslot receives V.w2
        load_mat64(p.vec + L.off_w2, HID, 0, HID, vslot);
#pragma unroll
        for (int i = 0; i < UT / 16; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int mm = tm + 16 * i, n = tn + 16 * j;
                const float h = tanhf(z[i][j] + W.b1[n]);
                sH1[mm * LD + n] = h;
                sT[mm * LD + n] = (1.f - h * h) * (dz[i][j] + vb1[n]);   // dH1
            }
        __syncthreads();
        // layer 2: Z2 = H1 W2^T + b2 ; dZ2 = H1 V2^T + dH1 W2^T + vb2
        gemm_nt<UT, LD, LD>(sH1, W.w2, HID, z);
        gemm_nt<UT, LD, LD>(sH1, vslot, HID, dz);
        gemm_nt<UT, LD, LD>(sT, W.w2, HID, acc);
        __syncthreads();
#pragma unroll
        for (int i = 0; i < UT / 16; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int mm = tm + 16 * i, n = tn + 16 * j;
                const float h = tanhf(z[i][j] + W.b2[n]);
                sH2[mm * LD + n] = h;
                sT[mm * LD + n] = (1.f - h * h) * (dz[i][j] + acc[i][j] + vb2[n]);   // dH2
            }
        __syncthreads();
        // output tangent: dMu = H2 V3^T + dH2 W3^T + vb3 ; dOUT = dMu / sigma^2 * scale
        {
            constexpr int NG = NTHREADS / UT;
            const int m = threadIdx.x % UT, og = threadIdx.x / UT;
            const bool rowok = sRow[m] >= 0;
            for (int o = og; o < OUTP; o += NG) {
                float c = 0.f;
                if (o < A && rowok) {
                    for (int k = 0; k < HID; ++k)
                        c += sH2[m * LD + k] * vw3[o * LD + k] + sT[m * LD + k] * W.w3[o * LD + k];
                    c = (c + vb3[o]) / (sSig[o] * sSig[o]) * scale;
                }
                sO[m * LDO + o] = c;
            }
        }
        __syncthreads();
        // ordinary backward with dOUT in sO
        {
            const int k = threadIdx.x & 63, og = threadIdx.x >> 6;
            for (int s = 0; s < UT; ++s) {
                const float h = sH2[s * LD + k];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int o = og + 4 * i;
                    if (o < A) aw3[i] = fmaf(sO[s * LDO + o], h, aw3[i]);
                }
            }
            if (threadIdx.x < A) {
                float c = 0.f;
                for (int s = 0; s < UT; ++s) c += sO[s * LDO + threadIdx.x];
                ab3 += c;
            }
        }
        gemm_nt<UT, LDO, LDO>(sO, W.w3t, OUTP, acc);
        __syncthreads();  // sT (dH2) fully consumed above
#pragma unroll
        for (int i = 0; i < UT / 16; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int mm = tm + 16 * i, n = tn + 16 * j;
                const float h = sH2[mm * LD + n];
                sT[mm * LD + n] = acc[i][j] * (1.f - h * h);   // dZ2
            }
        __syncthreads();
        {
            float g[4][4];
            gemm_tn<UT, LD, LD>(sT, sH1, g);
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
                for (int b = 0; b < 4; ++b) aw2[a][b] += g[a][b];
            if (threadIdx.x < HID) {
                float c = 0.f;
                for (int s = 0; s < UT; ++s) c += sT[s * LD + threadIdx.x];
                ab2 += c;
            }
        }
        gemm_nt<UT, LD, LD>(sT, W.w2t, HID, acc);
        __syncthreads();   // dZ2 (sT == sX) dead from here on
#pragma unroll
        for (int i = 0; i < UT / 16; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int mm = tm + 16 * i, n = tn + 16 * j;
                const float h = sH1[mm * LD + n];
                sH2[mm * LD + n] = acc[i][j] * (1.f - h * h);   // dZ1
            }
        {
            const int j0 = (threadIdx.x >> 4) * 4, k0 = (threadIdx.x & 15) * 4;
            for (int kc = 0; kc < nchunks; ++kc) {
                if (kc > 0) __syncthreads();
                gather_obs(p.obs, sRow, O, kc, sX);
                __syncthreads();
                if (kc == 0 && threadIdx.x < HID) {
                    float c = 0.f;
                    for (int s = 0; s < UT; ++s) c += sH2[s * LD + threadIdx.x];
                    ab1 += c;
                }
                float g[4][4];
                gemm_tn<UT, LD, LD>(sH2, sX, g);
                if (nchunks == 1) {
#pragma unroll
                    for (int a = 0; a < 4; ++a)
#pragma unroll
                        for (int b = 0; b < 4; ++b) aw1[a][b] += g[a][b];
                } else {
#pragma unroll
                    for (int a = 0; a < 4; ++a)
#pragma unroll
                        for (int b = 0; b < 4; ++b) {
                            const int col = kc * KC + k0 + b;
                            if (col < O) {
                                float* q = gout + L.off_w1 + (j0 + a) * O + col;
                                *q = first_tile ? g[a][b] : *q + g[a][b];
                            }
                        }
                }
            }
        }
        first_tile = false;
    }
    {
        const int j0 = (threadIdx.x >> 4) * 4, k0 = (threadIdx.x & 15) * 4;
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b) {
                gout[L.off_w2 + (j0 + a) * HID + k0 + b] = aw2[a][b];
                if (nchunks == 1 && k0 + b < O) gout[L.off_w1 + (j0 + a) * O + k0 + b] = aw1[a][b];
            }
        if (nchunks > 1 && first_tile)
            for (int i = threadIdx.x; i < HID * O; i += NTHREADS) gout[L.off_w1 + i] = 0.f;
        const int k = threadIdx.x & 63, og = threadIdx.x >> 6;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int o = og + 4 * i;
            if (o < A) gout[L.off_w3 + o * HID + k] = aw3[i];
        }
        if (threadIdx.x < HID) { gout[L.off_b1 + threadIdx.x] = ab1; gout[L.off_b2 + threadIdx.x] = ab2; }
        if (threadIdx.x < A) {
            gout[L.off_b3 + threadIdx.x] = ab3;
            // log_std block of the Fisher matrix: (2/A) v, counted once (CTA 0)
            gout[L.off_logstd + threadIdx.x] = (blockIdx.x == 0) ? 2.f / (float)A * __ldg(p.vec + L.off_logstd + threadIdx.x) : 0.f;
        }
    }
}

}  // namespace osb

using namespace osb;

static size_t grad_smem_bytes() {
    size_t f = NETSMEM_FLOATS_BWD + 4 * UT * LD + UT * LDO + 4 * 2 * OUTP + 6 * OUTP + ST_N;
    return f * sizeof(float) + UT * sizeof(long long) + 16;
}
static size_t eval_smem_bytes() {
    size_t f = NETSMEM_FLOATS_FWD + 3 * UT * LD + UT * LDO + 4 * OUTP + 2 * 2 * 4 * 8;
    return f * sizeof(float) + UT * sizeof(long long) + 16;
}
static size_t fvp_smem_bytes() {
    size_t f = NETSMEM_FLOATS_BWD + HID * LD + OUTP * LD + 2 * HID + OUTP + 3 * UT * LD + UT * LDO + OUTP;
    return f * sizeof(float) + UT * sizeof(long long) + 16;
}

extern "C" {

// CTAs per network: the three networks of a minibatch step share the 132 SMs in one wave
int osb_update_grid_blocks(int mb_count) {
    int tiles = (mb_count + UT - 1) / UT;
    const int cap = grid_sms() / 3;
    return tiles < cap ? tiles : cap;
}

// One minibatch: fused forward + loss + backward for the networks in `net_mask`.
// gpart must hold osb_update_grid_blocks(mb_count) * P floats, stats_part that many * 3 * 8 floats.
int osb_minibatch_grad(const float* theta, int O, int A, const float* obs, const float* act,
                       const float* logp, const float* adv_r, const float* adv_c,
                       const float* tv_r, const float* tv_c, const float* mu_old,
                       const float* moments, const int* perm, long long total, unsigned perm_seed,
                       long long mb_start, int mb_count, int loss_kind, float clip,
                       float entropy_coef, float focops_lam, float focops_eta,
                       const float* lagrange, const float* logstd_old, int net_mask, float* gpart,
                       float* stats_part, const int* stop_flag, void* stream) {
    OSB_CHECK_ARG(theta && obs && act && logp && adv_r && adv_c && tv_r && tv_c && moments, "null input");
    OSB_CHECK_ARG(O > 0 && A > 0 && A <= OUTP && mb_count > 0 && total > 0, "bad dims");
    OSB_CHECK_ARG(mb_start >= 0 && mb_start + mb_count <= total, "minibatch window out of range");
    OSB_CHECK_ARG(loss_kind != LOSS_FOCOPS || (mu_old && logstd_old), "FOCOPS needs mu_old/logstd_old");
    GradArgs p;
    p.b = Batch{obs, act, logp, adv_r, adv_c, tv_r, tv_c, moments, perm, total, perm_seed, mb_start, mb_count, 0};
    p.lc = LossParams{loss_kind, clip, entropy_coef, focops_lam, focops_eta, lagrange, mu_old, logstd_old, nullptr};
    p.forward_only = 0;
    p.theta = theta; p.gpart = gpart; p.stats_part = stats_part; p.stop_flag = stop_flag;
    p.O = O; p.A = A;
    p.P = actor_layout(O, A).size + 2 * critic_layout(O, A).size;
    p.net_mask = net_mask;
    const size_t smem = grad_smem_bytes();
    static bool attr = false;
    if (!attr) {
        OSB_CUDA(cudaFuncSetAttribute(minibatch_grad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr = true;
    }
    dim3 grid(osb_update_grid_blocks(mb_count), 3);
    if (loss_two_pass(loss_kind) && (net_mask & 1)) {   // pass 1: actor forward only
        GradArgs q = p;
        q.forward_only = 1; q.net_mask = 1;
        minibatch_grad_kernel<<<grid, NTHREADS, smem, (cudaStream_t)stream>>>(q);
        OSB_LAUNCH_CHECK();
        const int rc = pass1_gate(stats_part, (int)grid.x, stop_flag, p.lc, (cudaStream_t)stream);
        if (rc) return rc;
    }
    minibatch_grad_kernel<<<grid, NTHREADS, smem, (cudaStream_t)stream>>>(p);
    OSB_LAUNCH_CHECK();
    return OSB_OK;
}

// Full-batch actor pass.  mu_store != NULL: write mu(theta) for every row (old-policy snapshot).
// Otherwise out[8] <- {sum_s sum_a KL(old||new), sum ratio*adv, sum ratio*adv_c, sum ratio, count,
// sum ratio*adv_r, 0, 0} (fp64) where adv = (adv_r_std - lambda*adv_c_centered)/(1+lambda).
int osb_actor_eval(const float* theta_actor, int O, int A, const float* obs, const float* act,
                   const float* logp, const float* adv_r, const float* adv_c, const float* mu_old,
                   const float* logstd_old, const float* moments, const float* lagrange,
                   long long total, int stride, float* mu_store, double* workspace, double* out,
                   void* stream) {
    OSB_CHECK_ARG(theta_actor && obs && total > 0 && stride > 0, "bad argument");
    OSB_CHECK_ARG(mu_store || (act && logp && adv_r && adv_c && mu_old && logstd_old && workspace && out), "null input");
    EvalArgs p;
    p.b = Batch{obs, act, logp, adv_r, adv_c, nullptr, nullptr, moments, nullptr, total, 0u, 0, 0, 0};
    p.mu_old = mu_old; p.theta = theta_actor; p.logstd_old = logstd_old; p.lagrange = lagrange; p.mu_store = mu_store;
    p.part = workspace; p.O = O; p.A = A; p.stride = stride;
    const size_t smem = eval_smem_bytes();
    static bool attr = false;
    if (!attr) {
        OSB_CUDA(cudaFuncSetAttribute(actor_eval_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr = true;
    }
    const long long nrows = (total + stride - 1) / stride;
    long long tiles = (nrows + UT - 1) / UT;
    const int cap = 2 * grid_sms();
    const int blocks = (int)(tiles < cap ? tiles : cap);
    cudaStream_t s = (cudaStream_t)stream;
    actor_eval_kernel<<<blocks, NTHREADS, smem, s>>>(p);
    OSB_LAUNCH_CHECK();
    return mu_store ? OSB_OK : eval_reduce(workspace, blocks, out, s);
}

int osb_fvp_grid_blocks(long long total, int stride) {
    const long long nrows = (total + stride - 1) / stride;
    const long long tiles = (nrows + UT - 1) / UT;
    const int cap = grid_sms();
    return (int)(tiles < cap ? tiles : cap);
}

// gpart[blocks][P_actor] <- per-CTA partials of F v (without damping); reduce with osb_reduce_partials.
int osb_fvp_partials(const float* theta_actor, const float* vec, int O, int A, const float* obs,
                     long long total, int stride, float* gpart, void* stream) {
    OSB_CHECK_ARG(theta_actor && vec && obs && gpart && total > 0 && stride > 0, "bad argument");
    FvpArgs p{obs, total, stride, theta_actor, vec, gpart, O, A};
    const size_t smem = fvp_smem_bytes();
    static bool attr = false;
    if (!attr) {
        OSB_CUDA(cudaFuncSetAttribute(fvp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr = true;
    }
    fvp_kernel<<<osb_fvp_grid_blocks(total, stride), NTHREADS, smem, (cudaStream_t)stream>>>(p);
    OSB_LAUNCH_CHECK();
    return OSB_OK;
}

}  // extern "C"
