// Dual (reward + cost) GAE as a segmented reverse inclusive scan -- sm_90a.
//
// Replaces the per-path Python recursions of the reference:
//   omnisafe/common/buffer/onpolicy_buffer.py:L148-203 (finish_path)
//   omnisafe/common/buffer/onpolicy_buffer.py:L299-303 (gae branch)
//   omnisafe/utils/math.py:L59-82                      (discount_cumsum, fp64 carry)
//   omnisafe/common/buffer/vector_onpolicy_buffer.py:L125-136 + utils/distributed.py:L382-388
//       (advantage statistics; produced here as fp64 partial sums in the epilogue)
//
// Layout: time-major SoA slabs [T][N] (env index contiguous) so that the rollout kernel appends a
// step with coalesced stores and this kernel reads rows with coalesced 128 B requests.
//
// Parallelisation: block = 16 envs (x) x 32 time-chunks (y) x 4 steps per thread (512 threads).  Every thread
// folds its 4 steps into an affine map  A_in -> b + a*A_in  (fp64), the 32 chunk maps of one env are
// combined with a warp-shuffle suffix scan (after a shared-memory transpose so that lanes run along
// time), and a second local pass replays the reference's sequential arithmetic
// (separately rounded fp64 mul/add) from the exact carry-in.  Tiles of 128 steps are walked from
// the end of the horizon to its start with a per-env carry.
#include "common.cuh"
#include <cuda.h>
#include <stdlib.h>
#include <string.h>

namespace osb {

constexpr int GE = 16;         // envs per block
constexpr int GC = 32;         // chunks per tile
constexpr int GL = 4;          // steps per chunk
constexpr int GT = GC * GL;    // steps per tile
constexpr int GPAD = GE + 1;
constexpr int GTHREADS = GE * GC;   // 512

struct GaeArgs {
    const float* rew;
    const float* cost;
    const float* val_r;
    const float* val_c;
    const uint8_t* flags;
    const float* boot_r;
    const float* boot_c;
    float* adv_r;
    float* adv_c;
    float* tv_r;
    float* tv_c;
    float* disc_ret;  // may be null
    double* partials; // [gridDim.x][4]
    double* sums;     // [4] written by the last block
    unsigned int* ticket;
    int T, N;
    float gamma_f;    // (float)gamma : fp32 delta arithmetic (onpolicy_buffer.py:L301)
    float pen;        // penalty_coefficient (onpolicy_buffer.py:L185)
    double g;         // gamma            (discounted return)
    double gl_r;      // gamma * lam      (python double product)
    double gl_c;      // gamma * lam_c
    long long* dbg;   // optional clock64 stamps of CTA 0 (tools/gae_stage_times.py), normally null
};

struct GaeTile {      // one thread's 4 steps (+ the value after them) of one env
    float r[GL], c[GL], vr[GL + 1], vc[GL + 1];
    unsigned f[GL];
};

__device__ __forceinline__ void gae_load_tile(const GaeArgs& p, int env, bool env_ok, int t0, GaeTile& d) {
    const int N = p.N, T = p.T;
#pragma unroll
    for (int i = 0; i < GL; ++i) {
        const int t = t0 + i;
        const bool ok = env_ok && t >= 0;
        const size_t idx = (size_t)(ok ? t : 0) * N + (env_ok ? env : 0);
        d.r[i] = ok ? __ldg(p.rew + idx) : 0.f;
        d.c[i] = ok ? __ldg(p.cost + idx) : 0.f;
        d.vr[i] = ok ? __ldg(p.val_r + idx) : 0.f;
        d.vc[i] = ok ? __ldg(p.val_c + idx) : 0.f;
        d.f[i] = ok ? (unsigned)__ldg(p.flags + idx) : 0u;
    }
    const int t = t0 + GL;
    const bool ok = env_ok && t >= 0 && t < T;
    const size_t idx = (size_t)(ok ? t : 0) * N + (env_ok ? env : 0);
    d.vr[GL] = ok ? __ldg(p.val_r + idx) : 0.f;
    d.vc[GL] = ok ? __ldg(p.val_c + idx) : 0.f;
}

// MULTI = more than one 128-step tile: prefetches the next tile (more registers, 1 CTA per SM);
// the single-tile instantiation fits 64 registers so that two CTAs share an SM.
// EST = advantage estimator (onpolicy_buffer.py:L299-331):
//   0 'gae'      adv = scan(delta, gamma*lam),  target = adv + V                    (L299-303)
//   1 'gae-rtg'  adv = scan(delta, gamma*lam),  target = discount_cumsum(rewards)   (L305-310)
//   2 'plain'    adv = delta,                   target = discount_cumsum(rewards)   (L328-331)
//   3 'vtrace'   on-policy V-trace (behaviour == target policy, so rho = c = 1, L312-326, L338-405):
//                v_t = V_t + delta_t + gamma (v_{t+1} - V_{t+1}),  adv_t = r_t + gamma v_{t+1} - V_t,
//                target = v.  The scan carries e_t = v_t - V_t (the lambda = 1 GAE recurrence) in fp64;
//                the replay pass redoes the reference's fp32 operations from that carry.
// where `rewards` is the penalised reward path INCLUDING its bootstrap slot (finish_path subtracts
// penalty * costs in place, L185) and the cost targets use the same gamma (L192-196).
// RET = produce discounted_ret (third scan); training keeps no discounted_ret, so the hot instantiation drops it.
template <bool MULTI, int EST, bool RET>
__global__ void __launch_bounds__(GTHREADS, (MULTI || EST == 1 || EST == 3) ? 1 : 2) gae_dual_kernel(GaeArgs p) {
    constexpr int NQ = (EST == 0 || EST == 3) ? 3 : 4;    // scanned quantities: adv_r, adv_c, reward-to-go, cost-to-go
    __shared__ double sa[NQ * GC * GPAD];
    __shared__ double sb[NQ * GC * GPAD];
    __shared__ double carry[NQ * GE];
    __shared__ double red[3 * (GTHREADS / 32)];
    __shared__ int s_last;

    const int x = threadIdx.x, y = threadIdx.y;     // env lane (16), time chunk (32)
    const int lin = y * GE + x;
    const int tw = lin >> 5, tl = lin & 31;          // transposed role: warp tw <-> env tw, lane tl <-> chunk
    const int env = blockIdx.x * GE + x;
    const bool env_ok = env < p.N;
    const int N = p.N, T = p.T;
    const int ntiles = (T + GT - 1) / GT;

    if (lin < NQ * GE) carry[lin] = 0.0;
    constexpr bool want_g = (EST == 1 || EST == 2) || RET;

    double st_r = 0.0, st_r2 = 0.0, st_c = 0.0;
    GaeTile cur;
    gae_load_tile(p, env, env_ok, T - GT + y * GL, cur);
    __syncthreads();

    for (int k = 0; k < ntiles; ++k) {
        const int t0 = T - (k + 1) * GT + y * GL;  // first step of my chunk (may be < 0)
        if (!MULTI && k > 0) gae_load_tile(p, env, env_ok, t0, cur);   // no prefetch in the 2-CTA/SM variant
        // fp32 deltas with the reference's three separately rounded ops; bootstrap at path ends.
        float dr[GL], dc[GL], bootr[GL], bootc[GL], r[GL], c[GL], vr[GL], vc[GL];
        bool end[GL], valid[GL];
#pragma unroll
        for (int i = 0; i < GL; ++i) {
            const int t = t0 + i;
            valid[i] = env_ok && t >= 0;
            end[i] = valid[i] && (cur.f[i] != 0u || t == T - 1);
            float nr = cur.vr[i + 1], nc = cur.vc[i + 1];
            if (end[i]) {
                const bool term = (cur.f[i] & OSB_FLAG_TERMINATED) != 0u;
                const size_t idx = (size_t)t * N + env;
                nr = term ? 0.f : __ldg(p.boot_r + idx);
                nc = term ? 0.f : __ldg(p.boot_c + idx);
            }
            const float rp = __fadd_rn(cur.r[i], -__fmul_rn(p.pen, cur.c[i]));
            // reward-to-go estimators run on the penalised path, bootstrap slot included
            bootr[i] = (EST == 0 || EST == 3) ? nr : __fadd_rn(nr, -__fmul_rn(p.pen, nc));
            bootc[i] = nc;
            dr[i] = __fadd_rn(__fadd_rn(rp, __fmul_rn(p.gamma_f, nr)), -cur.vr[i]);
            dc[i] = __fadd_rn(__fadd_rn(cur.c[i], __fmul_rn(p.gamma_f, nc)), -cur.vc[i]);
            r[i] = (EST == 0 || EST == 3) ? cur.r[i] : rp; c[i] = cur.c[i]; vr[i] = cur.vr[i]; vc[i] = cur.vc[i];
        }
        const float cur_vr_last = cur.vr[GL], cur_vc_last = cur.vc[GL];
        float nvr[GL], nvc[GL];   // V_{t+1} inside the path (V-trace replay)
#pragma unroll
        for (int i = 0; i < GL; ++i) { nvr[i] = cur.vr[i + 1]; nvc[i] = cur.vc[i + 1]; }
        // prefetch the next (earlier) tile while this one is scanned
        if (MULTI && k + 1 < ntiles) gae_load_tile(p, env, env_ok, t0 - GT, cur);
        // pass 1: fold the chunk into affine maps (a, b) per quantity.
        const double glr = (EST == 3) ? p.g : p.gl_r, glc = (EST == 3) ? p.g : p.gl_c;
        double ar = 1.0, br = 0.0, ac = 1.0, bc = 0.0, ag = 1.0, bg = 0.0, bh = 0.0;   // (ag, bh): cost-to-go
#pragma unroll
        for (int i = GL - 1; i >= 0; --i) {
            if (valid[i]) {
                if (end[i]) {
                    ar = 0.0; br = (double)dr[i];
                    ac = 0.0; bc = (double)dc[i];
                    if (want_g) { ag = 0.0; bg = (double)r[i] + p.g * (double)bootr[i]; }
                    if (EST == 1 || EST == 2) bh = (double)c[i] + p.g * (double)bootc[i];
                } else {
                    br = (double)dr[i] + glr * br; ar = glr * ar;
                    bc = (double)dc[i] + glc * bc; ac = glc * ac;
                    if (want_g) { bg = (double)r[i] + p.g * bg; ag = p.g * ag; }
                    if (EST == 1 || EST == 2) bh = (double)c[i] + p.g * bh;
                }
            }
        }
        sa[(0 * GC + y) * GPAD + x] = ar; sb[(0 * GC + y) * GPAD + x] = br;
        sa[(1 * GC + y) * GPAD + x] = ac; sb[(1 * GC + y) * GPAD + x] = bc;
        if (want_g) { sa[(2 * GC + y) * GPAD + x] = ag; sb[(2 * GC + y) * GPAD + x] = bg; }
        if (EST == 1 || EST == 2) { sa[(3 * GC + y) * GPAD + x] = ag; sb[(3 * GC + y) * GPAD + x] = bh; }
        __syncthreads();
        // transposed role: warp tw owns env tw of the block, lane tl = chunk index.
#pragma unroll
        for (int q = (EST == 2 ? 2 : 0); q < NQ; ++q) {
            if (q == 2 && !want_g) continue;
            double a = sa[(q * GC + tl) * GPAD + tw];
            double b = sb[(q * GC + tl) * GPAD + tw];
#pragma unroll
            for (int off = 1; off < GC; off <<= 1) {
                const double a2 = __shfl_down_sync(0xffffffffu, a, off);
                const double b2 = __shfl_down_sync(0xffffffffu, b, off);
                if (tl + off < GC) { b = b + a * b2; a = a * a2; }
            }
            const double cin = carry[q * GE + tw];
            const double full = b + a * cin;              // value at the first step of chunk tl
            double ain = __shfl_down_sync(0xffffffffu, full, 1);
            if (tl == GC - 1) ain = cin;                  // last chunk takes the tile carry
            __syncwarp();
            sb[(q * GC + tl) * GPAD + tw] = ain;
            if (tl == 0) carry[q * GE + tw] = full;
        }
        __syncthreads();
        // pass 2: replay sequentially from the exact carry-in with the reference's roundings.
        double Ar = sb[(0 * GC + y) * GPAD + x];
        double Ac = sb[(1 * GC + y) * GPAD + x];
        double Ag = want_g ? sb[(2 * GC + y) * GPAD + x] : 0.0;
        double Ah = (EST == 1 || EST == 2) ? sb[(3 * GC + y) * GPAD + x] : 0.0;
        // V-trace replay state: v_{t+1} of the step after this chunk (fp32, = V + e from the scan)
        float lv_r = 0.f, lv_c = 0.f;
        if (EST == 3) {
            lv_r = (float)((double)cur_vr_last + Ar);
            lv_c = (float)((double)cur_vc_last + Ac);
        }
#pragma unroll
        for (int i = GL - 1; i >= 0; --i) {
            if (EST == 3) {
                if (valid[i]) {
                    // values[index + 1] and last_v_s: the bootstrap slot at a path end, else V_{t+1} / v_{t+1}
                    const float vnr = end[i] ? bootr[i] : nvr[i], vnc = end[i] ? bootc[i] : nvc[i];
                    const float lr = end[i] ? bootr[i] : lv_r, lc = end[i] ? bootc[i] : lv_c;
                    const size_t idx = (size_t)(t0 + i) * N + env;
                    // policy_advantage = clip_rho * (r + gamma * v_{t+1} - V_t)        (L402-403)
                    const float rp = __fadd_rn(r[i], -__fmul_rn(p.pen, c[i]));
                    const float o_ar = __fadd_rn(__fadd_rn(rp, __fmul_rn(p.gamma_f, lr)), -vr[i]);
                    const float o_ac = __fadd_rn(__fadd_rn(c[i], __fmul_rn(p.gamma_f, lc)), -vc[i]);
                    // v_s[t] += delta + gamma * c * (last_v_s - V_{t+1})                 (L394-397)
                    lv_r = __fadd_rn(vr[i], __fadd_rn(dr[i], __fmul_rn(p.gamma_f, __fadd_rn(lr, -vnr))));
                    lv_c = __fadd_rn(vc[i], __fadd_rn(dc[i], __fmul_rn(p.gamma_f, __fadd_rn(lc, -vnc))));
                    Ag = end[i] ? __dadd_rn((double)r[i], __dmul_rn(p.g, (double)bootr[i]))
                                : __dadd_rn((double)r[i], __dmul_rn(p.g, Ag));
                    p.adv_r[idx] = o_ar; p.adv_c[idx] = o_ac;
                    p.tv_r[idx] = lv_r;  p.tv_c[idx] = lv_c;
                    if (RET && p.disc_ret) p.disc_ret[idx] = (float)Ag;
                    st_r += (double)o_ar; st_r2 += (double)o_ar * (double)o_ar; st_c += (double)o_ac;
                }
            } else if (valid[i]) {
                if (end[i]) {
                    Ar = (double)dr[i];
                    Ac = (double)dc[i];
                    if (want_g) Ag = __dadd_rn((double)r[i], __dmul_rn(p.g, (double)bootr[i]));
                    if (EST == 1 || EST == 2) Ah = __dadd_rn((double)c[i], __dmul_rn(p.g, (double)bootc[i]));
                } else {
                    Ar = __dadd_rn((double)dr[i], __dmul_rn(p.gl_r, Ar));
                    Ac = __dadd_rn((double)dc[i], __dmul_rn(p.gl_c, Ac));
                    if (want_g) Ag = __dadd_rn((double)r[i], __dmul_rn(p.g, Ag));
                    if (EST == 1 || EST == 2) Ah = __dadd_rn((double)c[i], __dmul_rn(p.g, Ah));
                }
                const size_t idx = (size_t)(t0 + i) * N + env;
                const float o_ar = (EST == 2) ? dr[i] : (float)Ar, o_ac = (EST == 2) ? dc[i] : (float)Ac;
                p.adv_r[idx] = o_ar;
                p.adv_c[idx] = o_ac;
                p.tv_r[idx] = (EST == 0) ? (float)(Ar + (double)vr[i]) : (float)Ag;
                p.tv_c[idx] = (EST == 0) ? (float)(Ac + (double)vc[i]) : (float)Ah;
                if (RET && p.disc_ret) p.disc_ret[idx] = (float)Ag;
                st_r += (double)o_ar;
                st_r2 += (double)o_ar * (double)o_ar;
                st_c += (double)o_ac;
            }
        }
        __syncthreads();
    }
    // epilogue: block partial sums for the advantage statistics (fixed order -> deterministic);
    // the last block to finish folds all partials into sums[4].
    st_r = warp_sum(st_r); st_r2 = warp_sum(st_r2); st_c = warp_sum(st_c);
    if (tl == 0) { red[0 * 16 + tw] = st_r; red[1 * 16 + tw] = st_r2; red[2 * 16 + tw] = st_c; }
    __syncthreads();
    if (lin == 0) {
        double a = 0, b = 0, c = 0;
        for (int w = 0; w < GTHREADS / 32; ++w) { a += red[w]; b += red[16 + w]; c += red[32 + w]; }
        double* o = p.partials + (size_t)blockIdx.x * 4;
        o[0] = a; o[1] = b; o[2] = c;
        const int nenv = min(GE, N - (int)blockIdx.x * GE);
        o[3] = (double)nenv * (double)T;
        __threadfence();
        s_last = (atomicAdd(p.ticket, 1u) == gridDim.x - 1) ? 1 : 0;
    }
    __syncthreads();
    if (s_last && lin < 32) {
        __threadfence();
        double acc[4] = {0, 0, 0, 0};
        for (int bb = lin; bb < (int)gridDim.x; bb += 32)
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[q] += __ldcg(p.partials + (size_t)bb * 4 + q);
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[q] = warp_sum(acc[q]);
        if (lin == 0) {
            for (int q = 0; q < 4; ++q) p.sums[q] = acc[q];
            *p.ticket = 0u;
        }
    }
}


// =====================================================================================================
// Streaming variant of the training instantiation ('gae', no discounted_ret): the hot path of
// VectorOnPolicyBuffer.finish_path (onpolicy_buffer.py:L148-203, L299-303; utils/math.py:L59-82).
//
// One CTA owns 32 envs (one full 128 B line per slab row) and walks the horizon backwards in tiles of 128
// steps.  The five input planes of a tile (reward, cost, value_r, value_c, flags) are streamed into shared
// memory with TMA (cp.async.bulk.tensor.2d, one box per plane, completion on mbarriers), two stages deep and
// in two halves: A = reward / cost / flags (free again after pass 1), B = the value planes (read until the end
// of pass 2); one elected thread refills the free halves right after the tile's only block barrier, which
// proves that every warp is done with them -- no empty barriers, no producer warp.  16 warps own 8
// consecutive steps each (lanes = envs: every shared-memory and global access is a full line, no
// transposes): pass 1 forms the fp32 deltas with the reference's three roundings and folds the chunk into
// an affine map (a, b), the barrier publishes the 16 maps, every warp composes the maps of the later chunks
// onto the tile carry (<= 15 fp64 FMAs), pass 2 replays the reference's separately rounded fp64 recurrence
// from that carry-in and stores the four output rows straight from registers (coalesced 128 B stores).
// Path ends and the bootstrap values of cut paths (sparse) are fetched one tile ahead.
constexpr int SW = 16;                                  // warps = time chunks per tile
constexpr int SL = 8;                                   // steps per chunk
constexpr int ST = SW * SL;                             // 128 steps per tile
constexpr int SE = 32;                                  // envs per CTA
constexpr int STHREADS = SW * 32;
constexpr uint32_t S_PLANE = ST * SE * 4;               // reward / cost plane of a tile
constexpr uint32_t S_PLANE_V = (ST + 1) * SE * 4;       // value planes carry one more row: V_{t+1} of the tile's last step
constexpr uint32_t S_FLAGS = ST * SE;
constexpr uint32_t S_OFF_REW = 0, S_OFF_COST = S_PLANE, S_OFF_VR = 2 * S_PLANE, S_OFF_VC = 2 * S_PLANE + S_PLANE_V,
                   S_OFF_FL = 2 * S_PLANE + 2 * S_PLANE_V, S_STAGE = S_OFF_FL + S_FLAGS;            // 69 888 B
constexpr int NSTG = 2;                                  // stages of the input pipeline
constexpr uint32_t S_OFF_MAPS = NSTG * S_STAGE;                                 // double [2][SW][4][32]: (a_r, b_r, a_c, b_c) per chunk
constexpr uint32_t S_OFF_CARRY = S_OFF_MAPS + 2 * SW * 4 * 32 * 8;           // double [2][2][32]
constexpr uint32_t S_OFF_RED = S_OFF_CARRY + 2 * 2 * 32 * 8;                 // double [3][SW]
constexpr uint32_t S_OFF_BARS = S_OFF_RED + 3 * SW * 8;                      // fullA[2] (reward, cost, flags), fullB[2] (values)
constexpr uint32_t S_SMEM = S_OFF_BARS + 2 * NSTG * 8 + 16;

struct GaeMaps { CUtensorMap rew, cost, val_r, val_c, flags; };

__device__ __forceinline__ uint32_t s_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void s_mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void s_mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void s_mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool s_mbar_test(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0u;
}
__device__ __forceinline__ void s_mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
                     : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    } while (!ok);
}
// one box of a [T][N] plane -> shared memory; coordinates (env, step) may lie outside the tensor (zero fill)
__device__ __forceinline__ void s_tma_load(uint32_t dst, const CUtensorMap* tm, int env0, int t0, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];\n"
                 ::"r"(dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(env0), "r"(t0), "r"(bar) : "memory");
}

// 16 bytes global -> shared, asynchronously (LDGSTS); src_bytes == 0 zero-fills (rows / envs outside the slab)
__device__ __forceinline__ void s_cp16(uint32_t dst, const void* src, uint32_t src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
// this thread's earlier cp.async copies arrive on the mbarrier when they have landed (counted in the barrier's expected arrivals)
__device__ __forceinline__ void s_cp_arrive(uint32_t bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];\n" ::"r"(bar) : "memory");
}

// TMA = false (OSB_GAE_LDGSTS=1): every thread copies 16-byte pieces of the tile with cp.async (LDGSTS) -- ~9 copies per thread
//   and tile, each thread's batch arriving on the stage's mbarrier.
// TMA = true (default): one elected thread issues cp.async.bulk.tensor.2d boxes {32 envs x 128 (129) steps}.
//   A box of 128-byte rows 4N bytes apart costs one row request per row: the per-SM request rate, not DRAM, bounds it.
// MODE 0: both halves by cp.async; MODE 1: both by TMA; MODE 2: the A half (reward, cost, flags) by TMA and the B half
// (values) by cp.async -- two independent load paths working side by side.
template <int MODE>
__global__ void __launch_bounds__(STHREADS, 1) gae_stream_kernel(const __grid_constant__ GaeMaps tm, GaeArgs p, double gl8_r, double gl8_c) {
    extern __shared__ __align__(128) uint8_t s_raw[];
    const uint32_t pad = (128u - (s_u32(s_raw) & 127u)) & 127u;
    uint8_t* sm = s_raw + pad;
    const uint32_t sb = s_u32(sm);
    double* sMaps = reinterpret_cast<double*>(sm + S_OFF_MAPS);
    double* sCarry = reinterpret_cast<double*>(sm + S_OFF_CARRY);
    double* sRed = reinterpret_cast<double*>(sm + S_OFF_RED);
    __shared__ int s_last;
    const uint32_t bars = sb + S_OFF_BARS;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int N = p.N, T = p.T;
    const int env0 = blockIdx.x * SE, env = env0 + lane;
    const bool env_ok = env < N;
    const int ntiles = (T + ST - 1) / ST;

    auto fullA = [&](int s) { return bars + (uint32_t)s * 8u; };
    auto fullB = [&](int s) { return bars + (uint32_t)(NSTG + s) * 8u; };
    // the two halves of a tile's load (one elected thread).  A = reward, cost, flags: dead after pass 1 of the tile that
    // used the stage; B = the two value planes: read until the end of pass 2.
    // one 16-byte piece c of a [rows][32 envs] float plane of tile k (8 pieces per row)
    auto cp_f32 = [&](const float* plane, uint32_t dst, int t0, int c) {
        const int row = c >> 3, part = c & 7, t = t0 + row, e = env0 + 4 * part;
        const bool ok = t >= 0 && t < T && e < N;
        s_cp16(dst + (uint32_t)c * 16u, plane + (ok ? (size_t)t * N + e : 0), ok ? 16u : 0u);
    };
    auto load_A = [&](int k) {
        const int s = k % NSTG, t0 = T - (k + 1) * ST;
        const uint32_t dst = sb + (uint32_t)s * S_STAGE;
        if constexpr (MODE != 0) {
            if (tid == 0) {
                s_mbar_expect_tx(fullA(s), 2 * S_PLANE + S_FLAGS);
                s_tma_load(dst + S_OFF_REW, &tm.rew, env0, t0, fullA(s));
                s_tma_load(dst + S_OFF_COST, &tm.cost, env0, t0, fullA(s));
                s_tma_load(dst + S_OFF_FL, &tm.flags, env0, t0, fullA(s));
            }
        } else {
#pragma unroll
            for (int j = 0; j < ST * 8 / STHREADS; ++j) {
                cp_f32(p.rew, dst + S_OFF_REW, t0, tid + j * STHREADS);
                cp_f32(p.cost, dst + S_OFF_COST, t0, tid + j * STHREADS);
            }
            if (tid < ST * 2) {                                          // flags: 2 pieces of 16 envs per row
                const int row = tid >> 1, part = tid & 1, t = t0 + row, e = env0 + 16 * part;
                const bool ok = t >= 0 && e < N;
                s_cp16(dst + S_OFF_FL + (uint32_t)tid * 16u, p.flags + (ok ? (size_t)t * N + e : 0), ok ? 16u : 0u);
            }
            s_cp_arrive(fullA(s));
        }
    };
    auto load_B = [&](int k) {
        const int s = k % NSTG, t0 = T - (k + 1) * ST;
        const uint32_t dst = sb + (uint32_t)s * S_STAGE;
        if constexpr (MODE == 1) {
            if (tid == 0) {
                s_mbar_expect_tx(fullB(s), 2 * S_PLANE_V);
                s_tma_load(dst + S_OFF_VR, &tm.val_r, env0, t0, fullB(s));
                s_tma_load(dst + S_OFF_VC, &tm.val_c, env0, t0, fullB(s));
            }
        } else {
            for (int c = tid; c < (ST + 1) * 8; c += STHREADS) {
                cp_f32(p.val_r, dst + S_OFF_VR, t0, c);
                cp_f32(p.val_c, dst + S_OFF_VC, t0, c);
            }
            s_cp_arrive(fullB(s));
        }
    };
    if (tid == 0) {
        for (int i = 0; i < NSTG; ++i) { s_mbar_init(fullA(i), MODE != 0 ? 1u : (uint32_t)STHREADS); s_mbar_init(fullB(i), MODE == 1 ? 1u : (uint32_t)STHREADS); }
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    if (tid < 2 * 2 * 32) sCarry[tid] = 0.0;
    __syncthreads();
    for (int j = 0; j < NSTG && j < ntiles; ++j) { load_A(j); load_B(j); }

    double st_r = 0.0, st_r2 = 0.0, st_c = 0.0;
    {
        // ============================ consumers: warp = 8 consecutive steps, lane = env ======================
        const int row0 = warp * SL;
        const float gam = p.gamma_f, pen = p.pen;
        const double glr = p.gl_r, glc = p.gl_c;
        float bootr[SL], bootc[SL];
        unsigned endmask = 0u;       // bit i: step row0 + i ends a path (flag set or last step of the epoch)
        // path ends of my chunk of tile k + the bootstrap values of the cut paths (sparse: only truncated / epoch-end
        // steps need one; terminated paths bootstrap with 0)
        auto fetch_boot = [&](int k) {
            const uint8_t* fl = sm + (uint32_t)(k % NSTG) * S_STAGE + S_OFF_FL + row0 * SE + lane;
            const int t0 = T - (k + 1) * ST + row0;
            unsigned em = 0u, need = 0u;
#pragma unroll
            for (int i = 0; i < SL; ++i) {
                const unsigned f = fl[i * SE];
                const bool end = (f != 0u) || (t0 + i == T - 1);
                em |= (end ? 1u : 0u) << i;
                need |= ((end && !(f & OSB_FLAG_TERMINATED) && env_ok && t0 + i >= 0) ? 1u : 0u) << i;
                bootr[i] = 0.f; bootc[i] = 0.f;
            }
            endmask = em;
            if (__any_sync(0xffffffffu, need != 0u)) {
#pragma unroll
                for (int i = 0; i < SL; ++i) {
                    if ((need >> i) & 1u) {
                        const size_t idx = (size_t)(t0 + i) * N + env;
                        bootr[i] = __ldg(p.boot_r + idx);
                        bootc[i] = __ldg(p.boot_c + idx);
                    }
                }
            }
        };
        const bool dbg_on = p.dbg != nullptr && blockIdx.x == 0 && lane == 0 && (warp == 0 || warp == SW - 1);
        int dbg_n = 0;
        auto stamp = [&](int id) {
            if (dbg_on && dbg_n < 250) {
                long long* d = p.dbg + (warp == 0 ? 0 : 512);
                d[1 + 2 * dbg_n] = id; d[2 + 2 * dbg_n] = clock64(); ++dbg_n; d[0] = dbg_n;
            }
        };
        stamp(0);
        s_mbar_wait(fullA(0), 0u);
        stamp(1);
        fetch_boot(0);
#pragma unroll 1
        for (int k = 0; k < ntiles; ++k) {
            stamp(2);
            const int s = k & 1;                              // parity of the map / carry buffers
            const int sg = k % NSTG, sgn = (k + 1) % NSTG;    // input stage of this tile / of the next one
            const uint32_t phn = (uint32_t)(((k + 1) / NSTG) & 1);
            const int t0 = T - (k + 1) * ST + row0;          // first step of my chunk (negative only in the last tile)
            const uint8_t* stg = sm + (uint32_t)sg * S_STAGE;
            const float* sRew = reinterpret_cast<const float*>(stg + S_OFF_REW) + row0 * SE + lane;
            const float* sCost = reinterpret_cast<const float*>(stg + S_OFF_COST) + row0 * SE + lane;
            const float* sVr = reinterpret_cast<const float*>(stg + S_OFF_VR) + row0 * SE + lane;
            const float* sVc = reinterpret_cast<const float*>(stg + S_OFF_VC) + row0 * SE + lane;
            const unsigned em = endmask;
            s_mbar_wait(fullB(sg), (uint32_t)((k / NSTG) & 1));
            stamp(8);
            // ---- pass 1: fp32 deltas (three separately rounded ops, onpolicy_buffer.py:L301) + chunk map ----
            // (rows with t < 0 of the last tile and lanes past N see TMA zero fill: they are computed and discarded)
            double dr[SL], dc[SL];
            {
                // (a) the eight rows are independent: loads, fp32 arithmetic and conversions pipeline freely
                float fr[SL], fc[SL];
                float nvr = sVr[SL * SE], nvc = sVc[SL * SE];
#pragma unroll
                for (int i = SL - 1; i >= 0; --i) {
                    const float r = sRew[i * SE], c = sCost[i * SE], vr = sVr[i * SE], vc = sVc[i * SE];
                    const bool end = (em >> i) & 1u;
                    const float nr = end ? bootr[i] : nvr, nc = end ? bootc[i] : nvc;
                    const float rp = __fadd_rn(r, -__fmul_rn(pen, c));
                    fr[i] = __fadd_rn(__fadd_rn(rp, __fmul_rn(gam, nr)), -vr);
                    fc[i] = __fadd_rn(__fadd_rn(c, __fmul_rn(gam, nc)), -vc);
                    nvr = vr; nvc = vc;
                }
#pragma unroll
                for (int i = 0; i < SL; ++i) { dr[i] = (double)fr[i]; dc[i] = (double)fc[i]; }
            }
            // (b) the chunk's affine map: the only sequential part of pass 1
            double br = 0.0, bc = 0.0;
#pragma unroll
            for (int i = SL - 1; i >= 0; --i) {
                const bool end = (em >> i) & 1u;
                br = fma(glr, end ? 0.0 : br, dr[i]);
                bc = fma(glc, end ? 0.0 : bc, dc[i]);
            }
            {
                double* m = sMaps + ((size_t)(s * SW + warp) * 4) * 32 + lane;
                m[0] = em ? 0.0 : gl8_r; m[32] = br; m[64] = em ? 0.0 : gl8_c; m[96] = bc;
            }
            stamp(3);
            asm volatile("bar.sync 1, %0;\n" ::"n"(SW * 32) : "memory");
            stamp(4);
            // every warp is past pass 1 of this tile and past pass 2 of the previous one: the A half of this stage and
            // the B half of the other stage are free -> refill them (tile k + 2 resp. k + 1; B of tile 1 went out at start)
            if (k + NSTG < ntiles) load_A(k + NSTG);
            if (k >= 1 && k + NSTG - 1 < ntiles) load_B(k + NSTG - 1);
            // ---- path ends / bootstrap values of the next tile (its A half was requested a whole tile ago) ----------
            const bool more = k + 1 < ntiles;
            bool fetched = false;
            if (more && s_mbar_test(fullA(sgn), phn)) { fetch_boot(k + 1); fetched = true; }
            // ---- carry-in: compose the maps of the later chunks of this tile onto the tile carry -------------
            double Ar = sCarry[((s ^ 1) * 2 + 0) * 32 + lane], Ac = sCarry[((s ^ 1) * 2 + 1) * 32 + lane];
#pragma unroll
            for (int w2 = SW - 1; w2 > 0; --w2) {
                if (w2 > warp) {                                         // warp-uniform
                    const double* m = sMaps + ((size_t)(s * SW + w2) * 4) * 32 + lane;
                    Ar = fma(m[0], Ar, m[32]);
                    Ac = fma(m[64], Ac, m[96]);
                }
            }
            stamp(5);
            // ---- pass 2: the reference's sequential fp64 recurrence (utils/math.py:L77) from the carry-in -----
            const bool partial = t0 < 0;                                 // warp-uniform; only in the last tile
            float* o_base = p.adv_r + (ptrdiff_t)t0 * N + env;           // never dereferenced where t < 0 / env >= N
            const ptrdiff_t d_ac = p.adv_c - p.adv_r, d_tr = p.tv_r - p.adv_r, d_tc = p.tv_c - p.adv_r;
            // A path end restarts the recurrence (x + d * 0 == x exactly).  Each row's roundings / stores sit in their own
            // guarded block on purpose: bursts of 64-bit conversions (XU pipe) issued back to back throttle the shared
            // memory / special-function queue.  The statistics sum the fp64
            // advantages before their rounding to fp32 (|difference| <= 2^-25 relative per element, random sign).
#pragma unroll
            for (int i = SL - 1; i >= 0; --i) {
                const bool end = (em >> i) & 1u;
                Ar = __dadd_rn(dr[i], __dmul_rn(glr, end ? 0.0 : Ar));
                Ac = __dadd_rn(dc[i], __dmul_rn(glc, end ? 0.0 : Ac));
                if (!partial || t0 + i >= 0) {
                    if (env_ok) {
                        float* o = o_base + (ptrdiff_t)i * N;
                        o[0] = (float)Ar; o[d_ac] = (float)Ac;
                        o[d_tr] = (float)(Ar + (double)sVr[i * SE]); o[d_tc] = (float)(Ac + (double)sVc[i * SE]);
                    }
                    st_r += Ar; st_r2 = fma(Ar, Ar, st_r2); st_c += Ac;
                }
            }
            if (warp == 0) { sCarry[(s * 2 + 0) * 32 + lane] = Ar; sCarry[(s * 2 + 1) * 32 + lane] = Ac; }
            stamp(fetched ? 6 : 7);
            if (more && !fetched) { s_mbar_wait(fullA(sgn), phn); fetch_boot(k + 1); }
        }
        st_r = warp_sum(st_r); st_r2 = warp_sum(st_r2); st_c = warp_sum(st_c);
        if (lane == 0) { sRed[warp] = st_r; sRed[SW + warp] = st_r2; sRed[2 * SW + warp] = st_c; }
    }
    __syncthreads();
    if (tid == 0) {
        double a = 0, b = 0, c = 0;
        for (int w = 0; w < SW; ++w) { a += sRed[w]; b += sRed[SW + w]; c += sRed[2 * SW + w]; }
        double* o = p.partials + (size_t)blockIdx.x * 4;
        o[0] = a; o[1] = b; o[2] = c;
        o[3] = (double)min(SE, N - env0) * (double)T;
        __threadfence();
        s_last = (atomicAdd(p.ticket, 1u) == gridDim.x - 1) ? 1 : 0;
    }
    __syncthreads();
    if (s_last && tid < 32) {
        __threadfence();
        double acc[4] = {0, 0, 0, 0};
        for (int bb = tid; bb < (int)gridDim.x; bb += 32)
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[q] += __ldcg(p.partials + (size_t)bb * 4 + q);
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[q] = warp_sum(acc[q]);
        if (tid == 0) {
            for (int q = 0; q < 4; ++q) p.sums[q] = acc[q];
            *p.ticket = 0u;
        }
    }
}

// sums[4] = {sum adv_r, sum adv_r^2, sum adv_c, count}; one warp, fixed order.
__global__ void gae_stats_reduce_kernel(const double* __restrict__ partials, int nblocks,
                                        double* __restrict__ sums) {
    double acc[4] = {0, 0, 0, 0};
    for (int b = threadIdx.x; b < nblocks; b += 32)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[q] += partials[(size_t)b * 4 + q];
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[q] = warp_sum(acc[q]);
    if (threadIdx.x == 0)
        for (int q = 0; q < 4; ++q) sums[q] = acc[q];
}

// moments[4] = {mean_r, std_r + 1e-8, mean_c, 1}  (vector_onpolicy_buffer.py:L131-136)
__global__ void adv_moments_kernel(const double* __restrict__ sums, int standardize_r,
                                   int standardize_c, float* __restrict__ moments) {
    if (threadIdx.x != 0) return;
    const double n = sums[3];
    const double mean_r = sums[0] / n;
    double var = sums[1] / n - mean_r * mean_r;
    if (var < 0.0) var = 0.0;
    const float mean_rf = (float)mean_r;
    const float std_rf = (float)sqrt(var);
    moments[0] = standardize_r ? mean_rf : 0.f;
    moments[1] = standardize_r ? __fadd_rn(std_rf, 1e-8f) : 1.f;
    moments[2] = standardize_c ? (float)(sums[2] / n) : 0.f;
    moments[3] = 1.f;
}

// materialise the standardised advantages (what VectorOnPolicyBuffer.get() returns)
__global__ void adv_standardize_kernel(const float* __restrict__ adv_r,
                                       const float* __restrict__ adv_c,
                                       const float* __restrict__ moments, size_t n,
                                       float* __restrict__ out_r, float* __restrict__ out_c) {
    const float m_r = moments[0], s_r = moments[1], m_c = moments[2];
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (size_t)gridDim.x * blockDim.x) {
        out_r[i] = __fdiv_rn(__fadd_rn(adv_r[i], -m_r), s_r);
        out_c[i] = __fadd_rn(adv_c[i], -m_c);
    }
}

// Batched discount_cumsum (utils/math.py:L59-82): one warp per row, lanes along time,
// fp64 affine warp-shuffle suffix scan.  x: [rows][len] fp32 or fp64, out: [rows][len] fp64.
template <typename TIn>
__global__ void discount_cumsum_kernel(const TIn* __restrict__ x, int rows, int len,
                                       double discount, double* __restrict__ out) {
    const int row = blockIdx.x * (blockDim.x / 32) + (threadIdx.x / 32);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const int per = (len + 31) / 32;
    const int lo = lane * per, hi = min(len, lo + per);
    const TIn* xr = x + (size_t)row * len;
    double* orow = out + (size_t)row * len;
    double a = 1.0, b = 0.0;
    for (int i = hi - 1; i >= lo; --i) {
        if (i == len - 1) { b = (double)xr[i]; a = 0.0; }
        else { b = (double)xr[i] + discount * b; a = discount * a; }
    }
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const double a2 = __shfl_down_sync(0xffffffffu, a, off);
        const double b2 = __shfl_down_sync(0xffffffffu, b, off);
        if (lane + off < 32) { b = b + a * b2; a = a * a2; }
    }
    double cum = __shfl_down_sync(0xffffffffu, b, 1);
    if (lane == 31) cum = 0.0;
    for (int i = hi - 1; i >= lo; --i) {
        if (i == len - 1) cum = (double)xr[i];
        else cum = __dadd_rn((double)xr[i], __dmul_rn(discount, cum));
        orow[i] = cum;
    }
}

}  // namespace osb

using namespace osb;

// ---- tensor maps of the streaming kernel (driver entry point through the runtime: no -lcuda) ------------
typedef CUresult (*osb_encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                        const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                        CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static osb_encode_tiled_fn osb_encode_tiled() {
    static osb_encode_tiled_fn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<osb_encode_tiled_fn>(f);
        (void)cudaGetLastError();
    }
    return fn;
}
// [T][N] plane -> 2-D map (dim 0 = env, dim 1 = step), box = 32 envs x `rows` steps
static bool osb_plane_map(CUtensorMap* m, const void* base, int T, int N, int elem, int rows) {
    osb_encode_tiled_fn enc = osb_encode_tiled();
    if (!enc) return false;
    const cuuint64_t dims[2] = {(cuuint64_t)N, (cuuint64_t)T};
    const cuuint64_t strides[1] = {(cuuint64_t)N * (cuuint64_t)elem};
    const cuuint32_t box[2] = {(cuuint32_t)SE, (cuuint32_t)rows};
    const cuuint32_t estr[2] = {1u, 1u};
    return enc(m, elem == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_UINT8, 2u, const_cast<void*>(base), dims,
               strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
// returns 0 when launched, 1 when the shape / alignment / driver does not allow the TMA path (caller falls back)
static int osb_gae_stream_launch(const GaeArgs& a, cudaStream_t s) {
    static const bool legacy = getenv("OSB_GAE_LEGACY") != nullptr;
    if (legacy || (a.N & 15) != 0) return 1;                      // row strides of the u8 plane must be 16 B multiples
    const uintptr_t al = (uintptr_t)a.rew | (uintptr_t)a.cost | (uintptr_t)a.val_r | (uintptr_t)a.val_c | (uintptr_t)a.flags;
    if (al & 15u) return 1;
    static const int mode = getenv("OSB_GAE_LDGSTS") ? 0 : getenv("OSB_GAE_TMA") ? 1 : getenv("OSB_GAE_MIXED") ? 2 : 1;
    const bool use_tma = mode != 0;
    static GaeMaps maps = {};
    if (use_tma) {
        struct Key { const void* p[5]; int T, N; };
        static Key key = {};
        static bool have = false;
        const Key now = {{a.rew, a.cost, a.val_r, a.val_c, a.flags}, a.T, a.N};
        if (!have || memcmp(&key, &now, sizeof(Key)) != 0) {
            if (!osb_plane_map(&maps.rew, a.rew, a.T, a.N, 4, ST) || !osb_plane_map(&maps.cost, a.cost, a.T, a.N, 4, ST) ||
                !osb_plane_map(&maps.val_r, a.val_r, a.T, a.N, 4, ST + 1) || !osb_plane_map(&maps.val_c, a.val_c, a.T, a.N, 4, ST + 1) ||
                !osb_plane_map(&maps.flags, a.flags, a.T, a.N, 1, ST)) { have = false; return 1; }
            key = now; have = true;
        }
    }
    static bool attr = false;
    if (!attr) {
        if (cudaFuncSetAttribute(gae_stream_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(S_SMEM + 128)) != cudaSuccess ||
            cudaFuncSetAttribute(gae_stream_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(S_SMEM + 128)) != cudaSuccess ||
            cudaFuncSetAttribute(gae_stream_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(S_SMEM + 128)) != cudaSuccess) { (void)cudaGetLastError(); return 1; }
        attr = true;
    }
    double g8r = 1.0, g8c = 1.0;
    for (int i = 0; i < SL; ++i) { g8r *= a.gl_r; g8c *= a.gl_c; }
    const int nblk = (a.N + SE - 1) / SE;
    if (mode == 1) gae_stream_kernel<1><<<nblk, STHREADS, S_SMEM + 128, s>>>(maps, a, g8r, g8c);
    else if (mode == 2) gae_stream_kernel<2><<<nblk, STHREADS, S_SMEM + 128, s>>>(maps, a, g8r, g8c);
    else gae_stream_kernel<0><<<nblk, STHREADS, S_SMEM + 128, s>>>(maps, a, g8r, g8c);
    return 0;
}

extern "C" {

// partials [blocks][4] + one 8-byte ticket slot (zero-initialised by the caller, self-resetting)
static long long* g_gae_dbg = nullptr;
// development aid: clock64 stamps of CTA 0 of the next streaming-GAE launches go to buf (1024 long long), NULL turns it off
int osb_gae_debug_buffer(long long* buf) { g_gae_dbg = buf; return OSB_OK; }

int osb_gae_workspace_doubles(int n_envs) { return ((n_envs + GE - 1) / GE) * 4 + 8; }

int osb_adv_estimate(const float* rew, const float* cost, const float* val_r, const float* val_c,
                     const uint8_t* flags, const float* boot_r, const float* boot_c, int T, int N,
                     double gamma, double lam, double lam_c, double penalty_coef, int estimator,
                     float* adv_r, float* adv_c, float* tv_r, float* tv_c, float* disc_ret,
                     double* workspace, double* sums, void* stream) {
    OSB_CHECK_ARG(T > 0 && N > 0, "T, N must be positive");
    OSB_CHECK_ARG(estimator >= 0 && estimator <= 3, "estimator: 0 gae, 1 gae-rtg, 2 plain, 3 vtrace");
    OSB_CHECK_ARG(estimator == 0 || estimator == 3 || disc_ret == nullptr || penalty_coef == 0.0,
                  "reward-to-go estimators share the scan with discounted_ret: needs penalty_coef == 0 or disc_ret == NULL");
    OSB_CHECK_ARG(rew && cost && val_r && val_c && flags && boot_r && boot_c, "null input slab");
    OSB_CHECK_ARG(adv_r && adv_c && tv_r && tv_c && workspace && sums, "null output");
    GaeArgs a;
    a.rew = rew; a.cost = cost; a.val_r = val_r; a.val_c = val_c; a.flags = flags;
    a.boot_r = boot_r; a.boot_c = boot_c;
    a.adv_r = adv_r; a.adv_c = adv_c; a.tv_r = tv_r; a.tv_c = tv_c; a.disc_ret = disc_ret;
    a.partials = workspace;
    a.T = T; a.N = N;
    a.gamma_f = (float)gamma; a.pen = (float)penalty_coef;
    a.g = gamma; a.gl_r = gamma * lam; a.gl_c = gamma * lam_c;
    a.dbg = g_gae_dbg;
    const int nblocks = (N + GE - 1) / GE;
    a.sums = sums;
    a.ticket = reinterpret_cast<unsigned int*>(workspace + (size_t)nblocks * 4 + 1);
    cudaStream_t s = (cudaStream_t)stream;
    // the 64-register instantiation (two CTAs per SM) is the default: it keeps two CTAs per SM resident, which the
    // register-hungry prefetching variant does not; that one is kept for experiments (OSB_GAE_PREFETCH=1)
    static const bool prefetch = getenv("OSB_GAE_PREFETCH") != nullptr;
    const bool ret = disc_ret != nullptr;
    const dim3 blk(GE, GC);
    if (estimator == 1) {
        if (ret) gae_dual_kernel<false, 1, true><<<nblocks, blk, 0, s>>>(a);
        else gae_dual_kernel<false, 1, false><<<nblocks, blk, 0, s>>>(a);
    } else if (estimator == 2) {
        if (ret) gae_dual_kernel<false, 2, true><<<nblocks, blk, 0, s>>>(a);
        else gae_dual_kernel<false, 2, false><<<nblocks, blk, 0, s>>>(a);
    } else if (estimator == 3) {
        if (ret) gae_dual_kernel<false, 3, true><<<nblocks, blk, 0, s>>>(a);
        else gae_dual_kernel<false, 3, false><<<nblocks, blk, 0, s>>>(a);
    } else if (prefetch && T > GT) {
        gae_dual_kernel<true, 0, true><<<nblocks, blk, 0, s>>>(a);
    } else if (ret) {
        gae_dual_kernel<false, 0, true><<<nblocks, blk, 0, s>>>(a);
    } else if (osb_gae_stream_launch(a, s) != 0) {
        // training path (no discounted_ret slab) when the TMA streaming kernel cannot take the shape (N % 16 != 0,
        // unaligned slabs) or OSB_GAE_LEGACY is set: the two-scan instantiation of the generic kernel
        gae_dual_kernel<false, 0, false><<<nblocks, blk, 0, s>>>(a);
    }
    OSB_LAUNCH_CHECK();
    return OSB_OK;
}

int osb_gae_dual(const float* rew, const float* cost, const float* val_r, const float* val_c,
                 const uint8_t* flags, const float* boot_r, const float* boot_c, int T, int N,
                 double gamma, double lam, double lam_c, double penalty_coef, float* adv_r,
                 float* adv_c, float* tv_r, float* tv_c, float* disc_ret, double* workspace,
                 double* sums, void* stream) {
    return osb_adv_estimate(rew, cost, val_r, val_c, flags, boot_r, boot_c, T, N, gamma, lam, lam_c,
                            penalty_coef, 0, adv_r, adv_c, tv_r, tv_c, disc_ret, workspace, sums, stream);
}

int osb_adv_moments(const double* sums, int standardize_r, int standardize_c, float* moments,
                    void* stream) {
    OSB_CHECK_ARG(sums && moments, "null pointer");
    adv_moments_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(sums, standardize_r, standardize_c,
                                                          moments);
    OSB_LAUNCH_CHECK();
    return OSB_OK;
}

int osb_adv_standardize(const float* adv_r, const float* adv_c, const float* moments, long long n,
                        float* out_r, float* out_c, void* stream) {
    OSB_CHECK_ARG(adv_r && adv_c && moments && out_r && out_c && n >= 0, "bad argument");
    if (n == 0) return OSB_OK;
    int blocks = (int)((n + 255) / 256);
    if (blocks > 8 * grid_sms()) blocks = 8 * grid_sms();
    adv_standardize_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(adv_r, adv_c, moments,
                                                                    (size_t)n, out_r, out_c);
    OSB_LAUNCH_CHECK();
    return OSB_OK;
}

int osb_discount_cumsum(const void* x, int x_is_f64, int rows, int len, double discount,
                        double* out, void* stream) {
    OSB_CHECK_ARG(rows >= 0 && len >= 0 && out, "bad argument");
    if (rows == 0 || len == 0) return OSB_OK;
    OSB_CHECK_ARG(x != nullptr, "null input");
    const int wpb = 4;
    const int blocks = (rows + wpb - 1) / wpb;
    cudaStream_t s = (cudaStream_t)stream;
    if (x_is_f64)
        discount_cumsum_kernel<double><<<blocks, wpb * 32, 0, s>>>((const double*)x, rows, len,
                                                                   discount, out);
    else
        discount_cumsum_kernel<float><<<blocks, wpb * 32, 0, s>>>((const float*)x, rows, len,
                                                                  discount, out);
    OSB_LAUNCH_CHECK();
    return OSB_OK;
}

}  // extern "C"
