// Tensor-core full-batch actor forward: the fast variants of actor_eval_kernel (csrc/update.cu), on the forward of
// csrc/tc_forward.cuh.  Stores mu(theta) per row (old-policy snapshot, trpo.py:L177 / policy_gradient.py:L383-392) or
// reduces sum KL(old||new), sum ratio*adv, sum ratio*adv_c, sum ratio, count, sum ratio*adv_r in fp64.
//   actor_eval_tc_kernel  (tf32, O <= 512): 128-row tiles, two CTAs per SM (~100 KB smem each) so that one CTA's
//                         epilogue overlaps the other's MMA.
//   actor_eval_x3_kernel  (split-bf16, O <= 64, fp32-level accuracy): one persistent CTA per SM whose three
//                         warpgroups each run their own 64-row tiles, input tiles bulk-copied.
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
    float* acc;         // tf32: accumulator images, [gridDim.x][128][TC_COLS]
    long long total; int stride, O, A;
    double* out;        // bf16x3: the folded sums
};

template <int ACT>
__global__ void __launch_bounds__(NTHREADS, 2) actor_eval_tc_kernel(EvalTcArgs p, NetSpec spec) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const uint32_t pad = (1024u - (smem_u32(smem_raw) & 1023u)) & 1023u;
    const uint32_t B0 = smem_u32(smem_raw) + pad;
    float* fbase = reinterpret_cast<float*>(smem_raw + pad + TcTiles<false>::FLOATS);
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
    tc_stage_weights<false, 1>(B0, theta, L, O, sB1, sB2, sB3);
    if (tid < 16)
        stage_eval_policy(sLs, tid, (tid < A) ? __ldg(theta + L.off_logstd + tid) : 0.f,
                          (tid < A && p.logstd_old) ? __ldg(p.logstd_old + tid) : 0.f);
    if (tid == 0) { mbar_init(&bar, 1); mbar_init_fence(); }
    fence_async_smem();
    __syncthreads();
    const Acc tm = acc_cta(p.acc, TC_COLS);
    const uint32_t lane_base = (uint32_t)(q * 32) << 16;
    uint32_t phase = 0;

    const int nchunks = (O + 63) >> 6;
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
        // per-sample inputs of the final statistics, requested once layer 2 completed (the tf32 epilogues hold more
        // registers than a request before the forward leaves) so that they fly under the OUT MMAs
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
        tc_forward<false>(
            B0, tm, &bar, phase, sB1, sB2, nchunks, Hidden<ACT, umma::TanhFast>(spec, 0),
            [&](int c) { tc_stage_rows<false>(B0, p.obs, O, vec, c, theta, L, [&](int m) { return sRow[m]; }); },
            [&](int l) {
                if (l == 2) load_sample();
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

// ---- bf16x3 -------------------------------------------------------------------------------------------------------
// Warpgroup h of CTA b runs the 64-row tiles g, g + G, g + 2 G, ... (g = XW_WG b + h, G = XW_WG gridDim.x) through a
// raw input slot of its own: the tile's obs [64][O], and in KL mode act [64][A], mu_old [64][A], logp, adv_r, adv_c
// [64], each a contiguous run of the slabs.  One thread of the warpgroup bulk-copies (cp.async.bulk) the next tile's obs
// as soon as this tile's obs is split, and its KL runs once this tile's statistics are taken, each on its own mbarrier:
// both land while a whole forward runs.
// A tile whose runs are not 16-byte multiples at 16-byte aligned addresses (stride > 1, an unaligned slab, a short last
// tile) is gathered into the slot by the warpgroup's threads instead.  The warpgroup then splits obs into its 64 rows
// of A fragments and runs tc_forward_x3_half; OUT goes through shared memory to one thread per row (KL) or to
// coalesced stores of mu (mu_store).  The warpgroups meet only around the weights and the final reduction.
// Shared memory: the weight tiles, the floats, the slots.  The activations never leave the warpgroup's registers
// (tc_forward_x3_half).
constexpr int XW_WG = 3, XW_THREADS = 128 * XW_WG;
constexpr int XW_OUT_PITCH = 17;                         // floats per row of the OUT staging (odd: no bank conflicts)
// floats after the weight tiles: b1[64] b2[64] b3[16] ls[64], double red[XW_THREADS / 32][8], out[64 XW_WG][XW_OUT_PITCH]
constexpr int XW_RED = 208, XW_OUT = XW_RED + 2 * 8 * (XW_THREADS / 32), XW_WORDS = XW_OUT + 64 * XW_WG * XW_OUT_PITCH;
constexpr uint32_t XW_FLOATS = TcTiles<true>::FLOATS - TcTiles<true>::W1;          // the weight tiles come first
constexpr uint32_t XW_RING = XW_FLOATS + ((XW_WORDS * 4 + 127) & ~127);          // raw input slots, 128-aligned

// bytes of one raw input slot: the obs run, then (KL) act, mu_old, logp, adv_r, adv_c; every run a multiple of 256 bytes
__host__ __device__ __forceinline__ uint32_t x3_slot_bytes(int O, int A, bool kl) {
    return 256u * (uint32_t)(O + (kl ? 2 * A + 3 : 0));
}

// one fp64 partial row per CTA, folded by the last CTA to finish (self-resetting; zero when the module loads)
__device__ unsigned int g_eval_x3_ticket;

template <int ACT>
__global__ void __launch_bounds__(XW_THREADS, 1) actor_eval_x3_kernel(EvalTcArgs p, NetSpec spec) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const uint32_t pad = (1024u - (smem_u32(smem_raw) & 1023u)) & 1023u;
    const uint32_t B0 = smem_u32(smem_raw) + pad;
    const uint32_t W = B0 - TcTiles<true>::W1;                        // the weight tiles at B0 (TcTiles<true> offsets from W)
    float* fbase = reinterpret_cast<float*>(smem_raw + pad + XW_FLOATS);
    float* sB1 = fbase + EW_B1;
    float* sB2 = fbase + EW_B2;
    float* sB3 = fbase + EW_B3;      // [16]
    float* sLs = fbase + EW_LS;      // [64] evaluation policy constants of csrc/loss.cuh
    double* sRedD = reinterpret_cast<double*>(fbase + XW_RED);       // [warp][8]
    float* sOut = fbase + XW_OUT;                                    // [64 XW_WG][XW_OUT_PITCH]
    __shared__ uint64_t full[XW_WG][2];                              // the warpgroups' slots: obs, KL runs
    __shared__ int s_last;

    const int tid = threadIdx.x, lane = tid & 31;
    const int h = warpgroup_index(), t = tid & 127, nb = 1 + h;      // named barrier 1 + h: the warpgroup's 128 threads
    const int O = p.O, A = p.A;
    const bool kl = p.mu_store == nullptr;
    const uint32_t slot_bytes = x3_slot_bytes(O, A, kl);
    const uint32_t slot = B0 + XW_RING + (uint32_t)h * slot_bytes;
    const float* raw = reinterpret_cast<const float*>(smem_raw + pad + XW_RING + (size_t)h * slot_bytes);
    const uint32_t o_act = 256u * O, o_mu = o_act + 256u * A, o_logp = o_mu + 256u * A, o_advr = o_logp + 256u, o_advc = o_advr + 256u;
    const long long nrows = (p.total + p.stride - 1) / p.stride;
    const long long ntiles = (nrows + 63) >> 6;
    const long long g = XW_WG * (long long)blockIdx.x + h, G = XW_WG * (long long)gridDim.x;
    auto aligned = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15u) == 0; };
    const bool bulk_any = p.stride == 1 && aligned(p.obs) &&
                          (!kl || (aligned(p.act) && aligned(p.mu_old) && aligned(p.logp) && aligned(p.adv_r) && aligned(p.adv_c)));
    auto rows_of = [&](long long u) { return (int)min(64ll, nrows - 64 * u); };
    // every run of the tile a whole number of 16-byte units (a full tile always is)
    auto bulk = [&](long long u) {
        const int n = rows_of(u);
        return bulk_any && (n == 64 || ((n * O) % 4 == 0 && (!kl || ((n * A) % 4 == 0 && n % 4 == 0))));
    };
    // one thread: the obs run (part 0) or the KL runs (part 1) of tile u into the slot, on the part's mbarrier
    auto issue = [&](long long u, int part) {
        const uint32_t bar = smem_u32(&full[h][part]);
        const int n = rows_of(u);
        const long long k0 = 64 * u;
        auto copy = [&](uint32_t d, const float* src, uint32_t bytes) {
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
                         ::"r"(slot + d), "l"(src), "r"(bytes), "r"(bar) : "memory");
        };
        fence_async_smem();                          // the slot's generic accesses before the async writes
        if (part == 0) {
            mbar_expect_tx(bar, 4u * n * O);
            copy(0, p.obs + k0 * O, 4u * n * O);
        } else {
            mbar_expect_tx(bar, 4u * n * (2 * A + 3));
            copy(o_act, p.act + k0 * A, 4u * n * A);
            copy(o_mu, p.mu_old + k0 * A, 4u * n * A);
            copy(o_logp, p.logp + k0, 4u * n);
            copy(o_advr, p.adv_r + k0, 4u * n);
            copy(o_advc, p.adv_c + k0, 4u * n);
        }
    };

    if (tid == 0) {
        for (int i = 0; i < 2 * XW_WG; ++i) mbar_init_a(smem_u32(&full[i >> 1][i & 1]), 1);
        mbar_init_fence();
    }
    __syncthreads();
    if (t == 0 && g < ntiles && bulk(g))            // the first tiles load while the weights are staged
        for (int part = 0; part < (kl ? 2 : 1); ++part) issue(g, part);
    const NetLayout L = actor_layout(O, A);
    if (tid < NTHREADS) tc_stage_weights<true, 1>(W, p.theta, L, O, sB1, sB2, sB3);   // staged by 256 threads
    if (tid < 16)
        stage_eval_policy(sLs, tid, (tid < A) ? __ldg(p.theta + L.off_logstd + tid) : 0.f,
                          (tid < A && p.logstd_old) ? __ldg(p.logstd_old + tid) : 0.f);
    fence_async_smem();
    __syncthreads();

    const AdvNorm an = adv_norm(p.moments, p.lagrange);
    double acc[6] = {0, 0, 0, 0, 0, 0};
    uint32_t phase_o = 0, phase_k = 0;               // parities of the slot's next obs / KL-run bulk completions
    auto wg_sync = [&] { asm volatile("bar.sync %0, 128;\n" ::"r"(nb) : "memory"); };
    const float* so = sOut + 64 * h * XW_OUT_PITCH;
    // The statistics of tile v from its OUT rows and its KL runs: one thread per row, eval_sample as the other kernels.
    auto stats = [&](long long v) {
        const int n = rows_of(v);
        if (bulk(v)) {
            mbar_wait_a(smem_u32(&full[h][1]), phase_k);
            phase_k ^= 1u;
        } else {                                     // gathered: rows 64 v .. 64 v + n - 1 of the strided slabs
            float* w = const_cast<float*>(raw);
            for (int i = t; i < n * A; i += 128) {
                const long long r = (64 * v + i / A) * p.stride * A + i % A;
                w[o_act / 4 + i] = __ldg(p.act + r);
                w[o_mu / 4 + i] = __ldg(p.mu_old + r);
            }
            for (int i = t; i < n; i += 128) {
                const long long r = (64 * v + i) * p.stride;
                w[o_logp / 4 + i] = __ldg(p.logp + r);
                w[o_advr / 4 + i] = __ldg(p.adv_r + r);
                w[o_advc / 4 + i] = __ldg(p.adv_c + r);
            }
            wg_sync();
        }
        if (t < n) {
            float mu[16], pa[16], pm[16];
#pragma unroll
            for (int a = 0; a < 16; ++a) {
                mu[a] = so[t * XW_OUT_PITCH + a] + sB3[a];
                pa[a] = (a < A) ? raw[o_act / 4 + t * A + a] : 0.f;
                pm[a] = (a < A) ? raw[o_mu / 4 + t * A + a] : 0.f;
            }
            eval_sample<16>(an, A, mu, pa, pm, raw[o_logp / 4 + t], raw[o_advr / 4 + t], raw[o_advc / 4 + t], sLs, acc);
        }
        wg_sync();                                   // the KL runs and the warpgroup's OUT rows are free
    };
    for (long long u = g; u < ntiles; u += G) {
        const int n = rows_of(u);
        const long long k0 = 64 * u;
        const bool bulk_u = bulk(u), bulk_next = u + G < ntiles && bulk(u + G);
        if (bulk_u) {
            mbar_wait_a(smem_u32(&full[h][0]), phase_o);
            phase_o ^= 1u;
        } else {                                     // gathered: rows k0 .. k0 + n - 1 of the strided obs
            float* w = const_cast<float*>(raw);
            for (int i = t; i < n * O; i += 128) w[i] = __ldg(p.obs + (k0 + i / O) * p.stride * O + i % O);
            wg_sync();
        }
        uint32_t xa[3][4][4];                        // obs as layer 1's A fragments, zero past O and past the last row
        {
            const int r0 = 16 * (t >> 5) + (lane >> 2);
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int rr = 0; rr < 2; ++rr) {
                    const int r = r0 + 8 * rr, c = 8 * j + 2 * (lane & 3), q = 2 * (j & 1) + rr;
                    x3::split2((r < n && c < O) ? raw[r * O + c] : 0.f, (r < n && c + 1 < O) ? raw[r * O + c + 1] : 0.f,
                               xa[0][j >> 1][q], xa[1][j >> 1][q], xa[2][j >> 1][q]);
                }
        }
        wg_sync();                                   // every thread has read its obs
        if (t == 0 && bulk_next) issue(u + G, 0);    // the obs run is free: the next tile's flies under this forward
        float o[8];
        tc_forward_x3_half(W, xa, sB1, sB2, Hidden<ACT, x3::TanhAcc>(spec, 0), o);
        {
            const int w = t >> 5;
#pragma unroll
            for (int rr = 0; rr < 2; ++rr)
#pragma unroll
                for (int jj = 0; jj < 2; ++jj) {
                    float* d = sOut + (64 * h + 16 * w + (lane >> 2) + 8 * rr) * XW_OUT_PITCH + 8 * jj + 2 * (lane & 3);
                    d[0] = o[4 * jj + 2 * rr]; d[1] = o[4 * jj + 2 * rr + 1];
                }
        }
        wg_sync();
        if (kl) {
            stats(u);
            if (t == 0 && bulk_next) issue(u + G, 1);
        } else {
            for (int i = t; i < n * A; i += 128) {
                const int r = i / A, a = i - r * A;
                p.mu_store[(k0 + r) * p.stride * A + a] = so[r * XW_OUT_PITCH + a] + sB3[a];
            }
            wg_sync();                               // the warpgroup's OUT rows are free
        }
    }
    if (kl) {
        const int warp = tid >> 5;
#pragma unroll
        for (int i = 0; i < 6; ++i) acc[i] = warp_sum(acc[i]);
        if (lane == 0)
            for (int i = 0; i < 6; ++i) sRedD[warp * 8 + i] = acc[i];
        __syncthreads();
        if (tid == 0) {
            for (int i = 0; i < 6; ++i) {
                double v = 0.0;
                for (int w = 0; w < XW_THREADS / 32; ++w) v += sRedD[w * 8 + i];
                p.part[(size_t)blockIdx.x * 8 + i] = v;
            }
            __threadfence();
            s_last = (atomicAdd(&g_eval_x3_ticket, 1u) == gridDim.x - 1) ? 1 : 0;
        }
        __syncthreads();
        if (s_last) {                                // fixed order: lane l sums CTAs l, l + 32, ...; then the shuffle tree
            __threadfence();
            if (warp < 6) {
                double v = 0.0;
                for (int b = lane; b < (int)gridDim.x; b += 32) v += __ldcg(p.part + (size_t)b * 8 + warp);
                v = warp_sum(v);
                if (lane == 0) p.out[warp] = v;
            } else if (warp < 8 && lane == 0) {
                p.out[warp] = 0.0;
            }
            if (tid == 0) g_eval_x3_ticket = 0u;
        }
    }
}

// 1024: the alignment pad in front of the operand tiles
static int actor_eval_tc(const float* theta_actor, int O, int A, const float* obs, const float* act, const float* logp,
                         const float* adv_r, const float* adv_c, const float* mu_old, const float* logstd_old,
                         const float* moments, const float* lagrange, long long total, int stride, float* mu_store,
                         double* workspace, double* out, void* stream) {
    EvalTcArgs p{obs, act, logp, adv_r, adv_c, mu_old, logstd_old, moments, lagrange, theta_actor, mu_store, workspace, nullptr, total, stride, O, A, out};
    const size_t smem = 1024 + TcTiles<false>::FLOATS + EW_WORDS * sizeof(float);
    const long long nrows = (total + stride - 1) / stride;
    const long long tiles = (nrows + TC_ROWS - 1) / TC_ROWS;
    const int cap = 2 * grid_sms();
    const int blocks = (int)(tiles < cap ? tiles : cap);
    p.acc = acc_scratch(ACC_EVAL_TC, (size_t)blocks * 128 * TC_COLS * sizeof(float));
    if (!p.acc) return OSB_ERR_CUDA;
    cudaStream_t s = (cudaStream_t)stream;
    const NetSpec spec = net_spec();
    const int rc = with_act<false>(spec.act[0], [&](auto a) {
        static bool attr = false;
        if (!attr) {
            OSB_CUDA(cudaFuncSetAttribute(actor_eval_tc_kernel<a.value>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            attr = true;
        }
        actor_eval_tc_kernel<a.value><<<blocks, NTHREADS, smem, s>>>(p, spec);
        OSB_LAUNCH_CHECK();
        return OSB_OK;
    });
    if (rc) return rc;
    return mu_store ? OSB_OK : eval_reduce(workspace, blocks, out, s);
}

static int actor_eval_x3(const float* theta_actor, int O, int A, const float* obs, const float* act, const float* logp,
                         const float* adv_r, const float* adv_c, const float* mu_old, const float* logstd_old,
                         const float* moments, const float* lagrange, long long total, int stride, float* mu_store,
                         double* workspace, double* out, void* stream) {
    EvalTcArgs p{obs, act, logp, adv_r, adv_c, mu_old, logstd_old, moments, lagrange, theta_actor, mu_store, workspace, nullptr, total, stride, O, A, out};
    const size_t smem = 1024 + XW_RING + XW_WG * x3_slot_bytes(O, A, mu_store == nullptr);
    const long long nrows = (total + stride - 1) / stride;
    const long long groups = (nrows + 64 * XW_WG - 1) / (64 * XW_WG);     // 64-row tiles, XW_WG per CTA at a time
    const int blocks = (int)(groups < grid_sms() ? groups : grid_sms());
    const NetSpec spec = net_spec();
    return with_act<false>(spec.act[0], [&](auto a) {
        static bool attr = false;
        if (!attr) {
            const size_t most = 1024 + XW_RING + XW_WG * x3_slot_bytes(64, 16, true);
            OSB_CUDA(cudaFuncSetAttribute(actor_eval_x3_kernel<a.value>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)most));
            attr = true;
        }
        actor_eval_x3_kernel<a.value><<<blocks, XW_THREADS, smem, (cudaStream_t)stream>>>(p, spec);
        OSB_LAUNCH_CHECK();
        return OSB_OK;
    });
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
    return actor_eval_tc(theta_actor, O, A, obs, act, logp, adv_r, adv_c, mu_old, logstd_old, moments, lagrange,
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
    return actor_eval_x3(theta_actor, O, A, obs, act, logp, adv_r, adv_c, mu_old, logstd_old, moments, lagrange,
                         total, stride, mu_store, workspace, out, stream);
}

}  // extern "C"
