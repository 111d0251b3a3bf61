// Fused rollout step: HBM-resident synthetic Box envs + ObsNormalize + ActionScale + actor /
// reward-critic / cost-critic forwards + Gaussian sample / log-prob + slab append + episode stats.
//
// One launch per environment step replaces, per step, the reference's
//   ConstraintActorCritic.step        models/actor_critic/constraint_actor_critic.py:L84-109
//   ActionScale.step / ObsNormalize.step   envs/wrapper.py:L510-514, L231-241
//   Normalizer.normalize/_push        common/normalizer.py:L88-139
//   VectorOnPolicyBuffer.store        common/buffer/vector_onpolicy_buffer.py:L96-99
//   the per-env done loop             adapter/onpolicy_adapter.py:L114-136 (+ _log_value L155-157)
//
// Grid = (ceil(N/32) env tiles) x (3 networks).  Actor CTAs sample the action, run the env
// transition, append the step to the time-major slabs and feed the running-normaliser sums; critic
// CTAs write V_r / V_c and the bootstrap values of paths cut in the previous step.  The grid-wide
// ObsNormalize reduction is done with order-independent fixed-point atomics and folded into the statistics by the
// last CTA of the launch (norm_fold); the next launch (= kernel boundary = grid sync) consumes it.
#include "common.cuh"
#include "gaussian.cuh"
#include "mlp.cuh"
#include "normalizer.cuh"
#include "tc_forward.cuh"

namespace osb {

constexpr int RT = 32;                       // envs per tile
constexpr double FIX_SCALE = 68719476736.0;  // 2^36 fixed point for the normaliser sums

struct EnvSpec {
    int O, A;
    int max_episode_steps;
    uint32_t seed;
    uint32_t term_threshold;  // terminate iff hash < threshold (0 = never)
    uint32_t env_id_offset;   // global env id of local env 0 (rank * N)
    float cost_threshold;
    int obs_normalize;
};

struct EnvState {
    float* s_raw;        // [2][N][O] raw observation of the current state (by step parity:
                         //   launch t reads buffer t&1 and writes buffer (t+1)&1)
    float* final_raw;    // [2][N][O] raw final observation of envs that finished (by step parity)
    int* ep_step;        // [N]
    uint32_t* episode;   // [N]
    uint32_t* gstep;     // [N] total env steps taken (termination hash counter)
    float* ep_ret;       // [N] running episode return / cost / length (adapter bookkeeping)
    float* ep_cost;      // [N]
    int* ep_len;         // [N]
    const float* bias;   // [O]
};

// Saute / Simmer safety state (adapter/saute_adapter.py:L135-217, simmer_adapter.py:L97-131): the networks see
// [normalised obs | z]; z starts an epoch at `init`, z <- (z - cost / budget) / gamma after every step, the stored reward
// becomes `unsafe_reward` once z <= 0, z returns to 1 when the episode ends (final observations carry z = 1).
struct SauteSpec {
    float* safety;       // [2][N] by step parity (like s_raw), or null: plain OnPolicyAdapter
    float budget;        // per-step safety budget (saute_adapter.py:L62-68)
    float gamma;         // saute_gamma
    float unsafe_reward;
    float init;          // z at the epoch's reset: 1 (Saute) or the relative budget (Simmer)
};

// EarlyTerminatedAdapter.step (adapter/early_terminated_adapter.py:L56-98), per env: the accumulated cost (never cleared
// by ordinary episode ends) exceeding cost_limit terminates the episode: reward 0, terminated = 1, the env is reset and
// the accumulator cleared.
struct EarlySpec {
    float* cost_acc;     // [N] or null
    float cost_limit;
};

struct NormState {
    float* mean;    // [O] running mean            (Normalizer._mean)
    float* sumsq;   // [O] running sum of squares  (Normalizer._sumsq)
    float* std;     // [O] max(sqrt(sumsq/(count-1)), 1e-2)
    float* mean1;   // [O] stats after pushing only the final-observation rows
    float* std1;    // [O]
    long long* count;          // [2]: [0] running count, [1] count used for mean1/std1
    long long* acc_all;        // [2][O] fixed-point sum x, sum x^2 over all next-obs rows
    long long* acc_fin;        // [2][O] same over final-observation rows
    int* fin_count;            // [1]
    int* had_fin;              // [1] previous launch pushed final rows
    unsigned int* ticket;      // [1]
};

struct Slabs {
    float* obs;      // [T][N][O] normalised observation fed to the networks
    float* act;      // [T][N][A]
    float* logp;     // [T][N]
    float* rew;      // [T][N]
    float* cost;     // [T][N]
    float* val_r;    // [T][N]
    float* val_c;    // [T][N]
    float* boot_r;   // [T][N] bootstrap values at truncated / epoch-end path ends
    float* boot_c;   // [T][N]
    uint8_t* flags;  // [T][N]
    float* epfin;    // [3][T][N] (EpRet, EpCost, EpLen) written where an episode finished
};

// ---------------------------------------------------------------------------------------------
// env arithmetic (bit-identical to oracle/synthetic_env.py)
__device__ __forceinline__ float env_reset_value(const EnvSpec& e, uint32_t gid, uint32_t episode,
                                                 int j) {
    return u32_to_unit(hash4(e.seed, gid, episode, (uint32_t)j));
}
__device__ __forceinline__ float env_next_value(float s, float a, float b) {
    float v = __fadd_rn(__fadd_rn(__fmul_rn(0.95f, s), __fmul_rn(0.1f, a)), b);
    return fminf(fmaxf(v, -10.f), 10.f);
}

// Normalizer._push of a batch of n rows given by its fixed-point sums x, x^2
__device__ void norm_push(float& mean, float& sumsq, long long count_old, long long n,
                          long long sx_fix, long long sxx_fix) {
    const double sx = (double)sx_fix / FIX_SCALE, sxx = (double)sxx_fix / FIX_SCALE;
    const double mraw = sx / (double)n;
    double m2 = sxx - (double)n * mraw * mraw;
    if (m2 < 0.0) m2 = 0.0;
    norm_push_moments(mean, sumsq, count_old, n, mraw, m2);
}

// The running statistics a fold updates: NormState's own, or a CTA's shared-memory copy of them (the persistent kernel).
struct NormStats {
    float *mean, *sumsq, *std, *mean1, *std1;
    long long* count;   // [2]
    int* had_fin;
};

// A fold's arithmetic, by every thread of one CTA: the fixed-point sums of a step pushed into s in ObsNormalize's push
// order -- the final-observation rows (acc_fin, nfin rows; none: skipped), the next observations (acc_all, n_all > 0
// rows), then the reset rows (acc_rst, n_rst rows; none or null: skipped).  count is s.count[0] before the fold; ld reads
// s's arrays; per_col(j) runs after column j.  stats1: mean1 / std1 / count[1] / had_fin take the state after the final
// rows, which the bootstrap values of the next step's truncated paths are computed from.  push = false: only count[0]
// advances.
template <class Ld, class PerCol>
__device__ __forceinline__ void norm_fold_stats(const NormStats& s, Ld&& ld, int O, long long count, int nfin,
                                                const long long* acc_all, const long long* acc_fin, long long n_all,
                                                bool stats1, bool push, const long long* acc_rst, long long n_rst,
                                                PerCol&& per_col) {
    for (int j = threadIdx.x; push && j < O; j += blockDim.x) {
        float mean = ld(s.mean + j), sumsq = ld(s.sumsq + j);
        long long c = count;
        if (nfin > 0) {
            norm_push(mean, sumsq, c, nfin, __ldcg(acc_fin + j), __ldcg(acc_fin + O + j));
            c += nfin;
            if (stats1) {
                s.mean1[j] = mean;
                s.std1[j] = norm_std(sumsq, c);
            }
        }
        norm_push(mean, sumsq, c, n_all, __ldcg(acc_all + j), __ldcg(acc_all + O + j));
        c += n_all;
        if (n_rst > 0) {
            norm_push(mean, sumsq, c, n_rst, __ldcg(acc_rst + j), __ldcg(acc_rst + O + j));
            c += n_rst;
        }
        s.mean[j] = mean;
        s.sumsq[j] = sumsq;
        s.std[j] = norm_std(sumsq, c);
        per_col(j);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        if (stats1) s.count[1] = count + nfin;
        s.count[0] = count + nfin + n_all + n_rst;
        if (stats1) *s.had_fin = nfin > 0 ? 1 : 0;
    }
}

// Executed by the last-arriving CTA of a launch: folds the launch's fixed-point sums into the running statistics
// (norm_fold_stats) and clears the sums, fin_count and the ticket.
__device__ void norm_fold(const NormState& ns, int O, long long n_all, bool stats1, bool push = true,
                          long long* acc_rst = nullptr, long long n_rst = 0) {
    __threadfence();
    const int nfin = *((volatile int*)ns.fin_count);
    const long long count = __ldcg(ns.count);    // (.cg: written by another CTA in an earlier launch)
    norm_fold_stats(NormStats{ns.mean, ns.sumsq, ns.std, ns.mean1, ns.std1, ns.count, ns.had_fin},
                    [](const float* a) { return __ldcg(a); }, O, count, nfin, ns.acc_all, ns.acc_fin, n_all, stats1,
                    push, acc_rst, n_rst, [&](int j) {
                        ns.acc_all[j] = 0; ns.acc_all[O + j] = 0;
                        ns.acc_fin[j] = 0; ns.acc_fin[O + j] = 0;
                        if (acc_rst) { acc_rst[j] = 0; acc_rst[O + j] = 0; }
                    });
    if (threadIdx.x == 0) {
        *ns.fin_count = 0;
        *ns.ticket = 0u;
    }
}

// x * 2^36 rounded to the nearest integer.  The scaling by a power of two is exact in fp32 as well (|x| <= 10 by the env
// spec), so one fp32 -> int64 conversion gives the same integer as the fp64 product did.
__device__ __forceinline__ long long to_fix(float x) { return __float2ll_rn(x * 68719476736.0f); }

// adds a tile's fixed-point sums of column j to the launch's accumulators: x and x^2 over all next-obs rows, and over the
// final-observation rows when there are any
__device__ __forceinline__ void push_fix_sums(const NormState& ns, int O, int j, long long sx, long long sxx, long long fx,
                                              long long fxx) {
    atomicAdd((unsigned long long*)(ns.acc_all + j), (unsigned long long)sx);
    atomicAdd((unsigned long long*)(ns.acc_all + O + j), (unsigned long long)sxx);
    if (fx != 0 || fxx != 0) {
        atomicAdd((unsigned long long*)(ns.acc_fin + j), (unsigned long long)fx);
        atomicAdd((unsigned long long*)(ns.acc_fin + O + j), (unsigned long long)fxx);
    }
}

// Called by every thread of every CTA of the launch: true in the CTA that arrives last at the ticket, after every CTA's
// global writes are visible to it.
__device__ __forceinline__ bool last_cta(unsigned int* ticket) {
    __shared__ int s_last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = (atomicAdd(ticket, 1u) == gridDim.x * gridDim.y - 1) ? 1 : 0;
    __syncthreads();
    return s_last;
}

// ObsNormalize of one value (Normalizer.normalize, normalizer.py:L122-139): clip((x - mean) / std, -5, 5)
__device__ __forceinline__ float norm_clip(float v, float mean, float std) {
    return fminf(fmaxf(__fdiv_rn(__fadd_rn(v, -mean), std), -5.f), 5.f);
}

// ---------------------------------------------------------------------------------------------
// reset of all envs (OnPolicyAdapter.rollout resets every epoch: onpolicy_adapter.py:L80) and the
// normaliser push of the reset observations (ObsNormalize.reset, wrapper.py:L243-261).
__global__ void __launch_bounds__(NTHREADS) env_reset_kernel(EnvSpec es, EnvState st, NormState ns, SauteSpec sa,
                                                             int N) {
    __shared__ float sNew[RT][KC + 1];
    const int env0 = blockIdx.x * RT;
    const int O = es.O;
    const int e = threadIdx.x >> 3, q = threadIdx.x & 7;
    const int env = env0 + e;
    const bool ok = env < N;
    uint32_t epi = 0;
    if (ok) epi = st.episode[env] + 1u;
    for (int c0 = 0; c0 < O; c0 += KC) {
        for (int j = c0 + q; j < min(O, c0 + KC); j += 8) {
            float v = 0.f;
            if (ok) {
                v = env_reset_value(es, es.env_id_offset + env, epi, j);
                st.s_raw[(size_t)env * O + j] = v;  // buffer 0: step 0 reads parity 0
            }
            sNew[e][j - c0] = v;
        }
        __syncthreads();
        if (es.obs_normalize) {
            const int j = c0 + threadIdx.x;
            if (threadIdx.x < KC && j < O) {
                long long sx = 0, sxx = 0;
                for (int r = 0; r < RT; ++r)
                    if (env0 + r < N) {
                        const float v = sNew[r][threadIdx.x];
                        sx += to_fix(v);
                        sxx += to_fix(__fmul_rn(v, v));
                    }
                push_fix_sums(ns, O, j, sx, sxx, 0, 0);
            }
        }
        __syncthreads();
    }
    if (ok && q == 0) {
        st.episode[env] = epi;
        st.ep_step[env] = 0;
        st.ep_ret[env] = 0.f;
        st.ep_cost[env] = 0.f;
        st.ep_len[env] = 0;
        if (sa.safety) sa.safety[env] = sa.init;   // buffer 0: step 0 reads parity 0
    }
    if (es.obs_normalize && last_cta(ns.ticket)) norm_fold(ns, O, N, true);
}

// Philox4x32-10 (fast-mode noise); counter = (env gid, global step, lane block, 0).
__device__ __forceinline__ void philox_round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
    const uint32_t n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
    c[0] = n0; c[1] = lo1; c[2] = n2; c[3] = lo0;
}
// both normals of action pair pr (actions 2 pr, 2 pr + 1): one Philox block serves two pairs, Box-Muller gives the pair's
// (cos, sin) values
__device__ float2 philox_normal2(uint32_t seed, uint32_t gid, uint32_t step, int pr) {
    uint32_t c[4] = {gid, step, (uint32_t)(pr >> 1), 0x0B200u};
    uint32_t k0 = seed, k1 = 0xCAFEF00Du;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        philox_round(c, k0, k1);
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    const int pair = pr & 1;
    const float u0 = ((float)(c[2 * pair] >> 8) + 0.5f) * (1.0f / 16777216.0f);
    const float u1 = ((float)(c[2 * pair + 1] >> 8) + 0.5f) * (1.0f / 16777216.0f);
    const float r = sqrtf(-2.0f * logf(u0));
    float sn, cs;
    sincosf(6.283185307179586f * u1, &sn, &cs);
    return make_float2(r * cs, r * sn);
}
// the normal of action a alone
__device__ float philox_normal(uint32_t seed, uint32_t gid, uint32_t step, int a) {
    const float2 n = philox_normal2(seed, gid, step, a >> 1);
    return (a & 1) ? n.y : n.x;
}

// Evaluation of a saved policy (Evaluator.evaluate, evaluator.py:L399-490) on N synthetic envs: env e runs episodes
// e, e + N, ... of num_episodes with the deterministic action, and accumulates each in fp64 like the reference's
// Python floats.  Results land in episode order.
struct EvalSpec {
    int* left;            // [N] episodes the env still has to run, the current one included (0: the env is idle)
    int* done_eps;        // [N] episodes it has finished
    double* ret;          // [N] return of the current episode
    double* cost;         // [N] its cost, discounted by crit^length
    int* len;             // [N] its length
    double* out_ret;      // [num_episodes] results in episode order
    double* out_cost;
    int* out_len;
    long long* acc_rst;   // [2][O] fixed-point sums of the reset rows of a step
    int* ctr;             // [3]: [0] envs running at the start of this step (0: evaluation done -- the done word),
                          //      [1] the same for the next step, [2] reset rows of this step
    double crit;          // cost_criteria
    double cost_limit;    // EarlyTerminated: an episode also ends once its discounted cost >= cost_limit
    int early;
    int explicit_reset;   // N == 1: the env is reset after every episode, as the reference calls env.reset();
                          // N > 1: the envs reset themselves, only an episode cut by the cost rule resets the env
    float* act_out;       // [N][A] the action of each running env in the last step it ran, or null
};

struct StepArgs {
    EnvSpec es;
    EnvState st;
    NormState ns;
    Slabs sl;
    SauteSpec sa;
    EarlySpec et;
    const float* theta;   // flat [actor | critic_r | critic_c]
    const float* eps;     // [N][A] noise of this step (parity mode) or null (Philox fast mode)
    uint32_t noise_seed;
    uint32_t global_step; // epoch * T + t, Philox counter
    int t, T, N;
    int is_tail;          // t == T: critics only (epoch-end bootstrap)
    int precision;        // 0 = fp32 FMA tiles of 32 envs, 1 = wgmma TF32 tiles of 128 envs, 2 = split-bf16 wgmma tiles (O <= 64)
    unsigned int* bar_ctr;    // persistent epoch kernel: grid-barrier arrival counter and release flag (zero at launch)
    unsigned int* bar_flag;
    long long* ring;          // persistent training kernel: 3 RING_SLOTs of normaliser sums (zero at launch)
    long long* dbg;           // optional clock64 stamps (persistent kernel), normally null
    float* acc;               // tensor-core tiles: accumulator images, one [128][TC_COLS] per CTA
    // external-env act step (EXT instantiations only): the sampled action after ActionScale onto [act_lo, act_hi]
    const float* act_lo;      // [A]
    const float* act_hi;      // [A]
    float* act_env;           // [N][A]
    // external-env act step replayed from a CUDA graph: the Philox counter is *epoch_dev * T + t (u32 wrap-around, as
    // the host computes global_step) instead of global_step.  Null: global_step is used.
    const unsigned* epoch_dev;
    EvalSpec ev;              // EVAL instantiations only
};

// Philox counter of an act step: a graph replay reads the epoch from the device, an eager launch passes it
__device__ __forceinline__ uint32_t act_global_step(const StepArgs& p) {
    return p.epoch_dev ? __ldg(p.epoch_dev) * (uint32_t)p.T + (uint32_t)p.t : p.global_step;
}

// ActionScale (wrapper.py:L510-512) from [-1, 1] onto [lo, hi] in the reference's fp32 order:
// lo + (hi - lo) * (a - (-1)) / (1 - (-1)).  No clipping: the env receives what the wrapper would hand it.
__device__ __forceinline__ float action_scale(float a, float lo, float hi) {
    return __fadd_rn(lo, __fdiv_rn(__fmul_rn(__fadd_rn(hi, -lo), __fadd_rn(a, 1.f)), 2.f));
}

// the sampled action a of env at step t into the act slab; EXT: also scaled onto the user env's box for env.step
template <bool EXT>
__device__ __forceinline__ void store_action(const StepArgs& p, int t, int env, int a, float act) {
    p.sl.act[((size_t)t * p.N + env) * p.es.A + a] = act;
    if constexpr (EXT) p.act_env[(size_t)env * p.es.A + a] = action_scale(act, __ldg(p.act_lo + a), __ldg(p.act_hi + a));
}

// A path cut at a step without termination (time limit): its critics bootstrap from the final observation.
__device__ __forceinline__ bool cut_path(unsigned f) { return (f & OSB_FLAG_TRUNCATED) && !(f & OSB_FLAG_TERMINATED); }

// Critic output v of env (net 1: reward critic, 2: cost critic).  boot_cut: v is V(final observation of step t - 1),
// stored where that path was cut; tail (t == T): v is the epoch-end bootstrap, stored unless the path ended at T - 1;
// otherwise v is the value at step t.
__device__ __forceinline__ void store_critic(const Slabs& sl, int net, int N, int t, int env, bool boot_cut, bool tail,
                                             float v) {
    if (boot_cut) {
        const size_t idx = (size_t)(t - 1) * N + env;
        if (cut_path(__ldcg(sl.flags + idx))) (net == 1 ? sl.boot_r : sl.boot_c)[idx] = v;
    } else if (tail) {
        const size_t idx = (size_t)(t - 1) * N + env;
        if (__ldcg(sl.flags + idx) == 0) (net == 1 ? sl.boot_r : sl.boot_c)[idx] = v;
    } else {
        (net == 1 ? sl.val_r : sl.val_c)[(size_t)t * N + env] = v;
    }
}

// normalise (or copy) a tile of raw observations into sX (chunk kc), zero padded.
// z = per-env safety state (Saute) appended as column O of the network input (rows are On = O + 1 wide then), or null;
// z_one: the final observations of finished episodes carry z = 1 (the state was reset before the augmentation).
__device__ __forceinline__ void load_obs_tile(const float* __restrict__ raw, int env0, int N, int O,
                                              int kc, const float* sMean, const float* sStd,
                                              bool normalize, float* sX, float* obs_out,
                                              const float* z = nullptr, bool z_one = false) {
    const int c0 = kc * KC;
    const int On = O + (z ? 1 : 0);
    for (int i = threadIdx.x; i < RT * KC; i += NTHREADS) {
        const int e = i / KC, k = i % KC;
        const int env = env0 + e, j = c0 + k;
        float v = 0.f;
        if (env < N && j < O) {
            v = raw[(size_t)env * O + j];
            if (normalize) v = norm_clip(v, sMean[j], sStd[j]);
            if (obs_out) obs_out[(size_t)env * On + j] = v;
        } else if (env < N && j == O && z) {
            v = z_one ? 1.f : __ldcg(z + env);
            if (obs_out) obs_out[(size_t)env * On + j] = v;
        }
        sX[e * LD + k] = v;
    }
}

// ActionScale (wrapper.py:L510-512) from [-1,1] onto the synthetic env's [-1,1] box, then the env's own clip
__device__ __forceinline__ float env_action(float a) {
    a = __fadd_rn(__fadd_rn(a, 1.f), -1.f);
    return fminf(fmaxf(a, -1.f), 1.f);
}
// reward 1 - mean_j s'_j^2 from sumsq = sum_j s'_j^2 (in the spec's summation tree), and the cost [s'_0 > threshold]
__device__ __forceinline__ float env_reward(float sumsq, int O) { return __fadd_rn(1.f, -__fdiv_rn(sumsq, (float)O)); }
__device__ __forceinline__ float env_cost(const EnvSpec& es, float s0n) { return (s0n > es.cost_threshold) ? 1.f : 0.f; }

// cost of this step (indicator on the next value of state dim 0) from the current raw state and the sampled action
__device__ __forceinline__ float env_step_cost(const EnvSpec& es, float s0, float act0, float bias0) {
    return env_cost(es, env_next_value(s0, env_action(act0), bias0));
}

// SauteAdapter.step (saute_adapter.py:L172-217) for one env: z <- (z - cost / budget) / gamma, reward override once
// z <= 0, z <- 1 when the episode ends.  Returns the reward to store (episode returns keep the original one).
__device__ __forceinline__ float saute_step(const SauteSpec& sa, int t, int N, int env, float rew, float cost, bool fin) {
    if (!sa.safety) return rew;
    float z = __ldcg(sa.safety + (size_t)(t & 1) * N + env);
    z = __fdiv_rn(__fadd_rn(z, -__fdiv_rn(cost, sa.budget)), sa.gamma);
    const float out = (z > 0.f) ? rew : sa.unsafe_reward;
    sa.safety[(size_t)((t + 1) & 1) * N + env] = fin ? 1.f : z;
    return out;
}

// Episode-end word of a synthetic env's step.  EP_EARLY: EarlyTerminated's cost limit ends the episode as a termination;
// EP_BOTH: it does so in the step the env's own episode ends, so the env auto-resets and then the adapter resets it.
enum : int { EP_FIN = 1, EP_TERM = 2, EP_TRUNC = 4, EP_EARLY = 8, EP_BOTH = 16 };

// the env's own episode end: time limit and hash-driven termination
__device__ __forceinline__ int episode_end(const EnvSpec& es, uint32_t gid, int ep_step, uint32_t gstep) {
    const bool trunc = ep_step + 1 >= es.max_episode_steps;
    const bool term = es.term_threshold != 0u && hash4(es.seed ^ 0xA5A5A5A5u, gid, gstep, 0xFFFFu) < es.term_threshold;
    return ((term || trunc) ? EP_FIN : 0) | (term ? EP_TERM : 0) | (trunc ? EP_TRUNC : 0);
}
// the word after the accumulated cost exceeded the limit
__device__ __forceinline__ int early_end(int fl) { return fl | ((fl & EP_FIN) ? EP_BOTH : 0) | EP_FIN | EP_TERM | EP_EARLY; }
// episode counter after an episode end (the reset observation's hash input)
__device__ __forceinline__ uint32_t next_episode(uint32_t epi, int fl) { return epi + ((fl & EP_BOTH) ? 2u : 1u); }

// Step t of one env into the reward / cost / flags slabs, and the episode statistics (_log_value, _log_metrics,
// _reset_log: onpolicy_adapter.py:L138-175): an episode that ends here leaves (EpRet, EpCost, EpLen) in epfin.
// rew_store goes to the slab, rew_acc into the episode return (Saute stores its own reward; the return keeps the env's).
__device__ __forceinline__ void record_step(const Slabs& sl, const EnvState& st, int T, int N, int t, int env,
                                            float rew_store, float rew_acc, float cst, bool term, bool trunc) {
    const size_t idx = (size_t)t * N + env;
    sl.rew[idx] = rew_store;
    sl.cost[idx] = cst;
    sl.flags[idx] = (uint8_t)((term ? OSB_FLAG_TERMINATED : 0u) | (trunc ? OSB_FLAG_TRUNCATED : 0u));
    const float er = __fadd_rn(st.ep_ret[env], rew_acc);
    const float ec = __fadd_rn(st.ep_cost[env], cst);
    const int el = st.ep_len[env] + 1;
    if (term || trunc) {
        const size_t TN = (size_t)T * N;
        sl.epfin[idx] = er;
        sl.epfin[TN + idx] = ec;
        sl.epfin[2 * TN + idx] = (float)el;
        st.ep_ret[env] = 0.f; st.ep_cost[env] = 0.f; st.ep_len[env] = 0;
    } else {
        st.ep_ret[env] = er; st.ep_cost[env] = ec; st.ep_len[env] = el;
    }
}

// The end of a synthetic env's step t: reward 1 - mean_j s'_j^2 (sumsq = sum_j s'_j^2 in the spec's summation tree; 0 on
// an EarlyTerminated end), cost = [s'_0 > cost_threshold], the Saute state, the step record and the env's counters.
// ep_step / epi / gstep are the values before the step, acc_cost the EarlyTerminated accumulator including this step.  They
// are references so that the tensor-core kernel's shared-memory copies are read where they are used, not held in registers
// across the divisions.
__device__ __forceinline__ void synthetic_step_end(const StepArgs& p, int N, int T, int O, int t, int env, int fl,
                                                   float sumsq, float s0n, const int& ep_step, const uint32_t& epi,
                                                   const uint32_t& gstep, const float& acc_cost) {
    const bool fin = fl & EP_FIN, early = fl & EP_EARLY;
    const float rew = early ? 0.f : env_reward(sumsq, O);
    const float cst = env_cost(p.es, s0n);
    record_step(p.sl, p.st, T, N, t, env, saute_step(p.sa, t, N, env, rew, cst, fin), rew, cst, fl & EP_TERM,
                fl & EP_TRUNC);
    if (p.et.cost_acc) p.et.cost_acc[env] = early ? 0.f : acc_cost;
    if (fin) {
        p.st.episode[env] = next_episode(epi, fl);
        p.st.ep_step[env] = 0;
    } else {
        p.st.ep_step[env] = ep_step + 1;
    }
    p.st.gstep[env] = gstep + 1u;
}

// ---------------------------------------------------------------------------------------------
// Evaluation of a saved policy (EVAL instantiations of the step kernels), after the actor forward of a tile of R envs;
// sMu[e * ld + a] holds the mean of env env0 + e.
//
// eval_action: the deterministic action in place (sample_action with eps = 0: the bits osb_policy_step gives without
// eps), into act_out for running envs and, EXT, scaled onto [act_lo, act_hi] into act_env for env.step.
template <int R, bool EXT>
__device__ void eval_action(const StepArgs& p, int env0, float* sMu, int ld, const float* log_std) {
    const int A = p.es.A, N = p.N;
    for (int i = threadIdx.x; i < R * A; i += NTHREADS) {
        const int e = i / A, a = i % A, env = env0 + e;
        const float sd = expf(__ldg(log_std + a));
        float term;
        const float act = sample_action(sMu[e * ld + a], sd, __fmul_rn(2.f, __fmul_rn(sd, sd)), logf(sd), 0.f, term);
        sMu[e * ld + a] = act;
        if (env < N) {
            if (p.ev.act_out && __ldcg(p.ev.left + env) > 0) p.ev.act_out[(size_t)env * A + a] = act;
            if constexpr (EXT) p.act_env[(size_t)env * A + a] = action_scale(act, __ldg(p.act_lo + a), __ldg(p.act_hi + a));
        }
    }
}

// The synthetic env's evaluation step t of the tile.  Per running env (one thread each): ActionScale, the transition
// into final_raw (scratch of this step), reward / cost, the fp64 episode sums, the Saute state, the EarlyTerminated rule
// and the episode end.  Then the normaliser sums of the rows the reference pushes in this step, in its order: the final
// observations of envs that ended, the next observations of every running env (an env that ended hands back its
// auto-reset observation), and the observations of the envs reset after the step.  sF / sE1 / sE2: R ints of shared
// scratch each.  eval_fold (one CTA, after every CTA's step) folds the sums into the statistics.
template <int R>
__device__ void eval_step(const StepArgs& p, int t, int env0, float* sMu, int ld, const float* log_std, int* sF,
                          uint32_t* sE1, uint32_t* sE2) {
    const EvalSpec& ev = p.ev;
    const int O = p.es.O, A = p.es.A, N = p.N, tid = threadIdx.x;
    eval_action<R, false>(p, env0, sMu, ld, log_std);
    __syncthreads();
    const float* s_cur = p.st.s_raw + (size_t)(t & 1) * N * O;
    float* s_nxt = p.st.s_raw + (size_t)((t + 1) & 1) * N * O;
    float* sn_all = p.st.final_raw + (size_t)(t & 1) * N * O;
    if (tid < R) {
        const int env = env0 + tid;
        int f = 0;
        if (env < N && ev.left[env] > 0) {
            const uint32_t gid = p.es.env_id_offset + env;
            const int ep_step = p.st.ep_step[env];
            const uint32_t epi = p.st.episode[env], gstep = p.st.gstep[env];
            const bool envfin = episode_end(p.es, gid, ep_step, gstep) & EP_FIN;
            const float* s = s_cur + (size_t)env * O;
            float* sn = sn_all + (size_t)env * O;
            // p_q = sum of s'_j^2 over j = q (mod 8), ascending; combined in the spec's tree
            float part[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            for (int j = 0; j < O; ++j) {
                const float v = env_next_value(s[j], env_action(sMu[tid * ld + (j % A)]), __ldg(p.st.bias + j));
                part[j & 7] = __fadd_rn(part[j & 7], __fmul_rn(v, v));
                sn[j] = v;
            }
            const float tot = __fadd_rn(__fadd_rn(__fadd_rn(part[0], part[1]), __fadd_rn(part[2], part[3])),
                                        __fadd_rn(__fadd_rn(part[4], part[5]), __fadd_rn(part[6], part[7])));
            const float rew = env_reward(tot, O);
            const float cst = env_cost(p.es, sn[0]);
            const int len = ev.len[env];
            const double r64 = ev.ret[env] + (double)rew;
            const double c64 = ev.cost[env] + pow(ev.crit, (double)len) * (double)cst;
            const bool done = envfin || (ev.early && c64 >= ev.cost_limit);
            saute_step(p.sa, t, N, env, rew, cst, done);      // z returns to 1 when the episode ends
            const int left = ev.left[env];
            const bool rst = done && left > 1 && (ev.explicit_reset || !envfin);
            uint32_t epi_n = envfin ? epi + 1u : epi;      // the env's own reset on its episode end
            const uint32_t epi_auto = epi_n;
            if (rst) ++epi_n;
            p.st.episode[env] = epi_n;
            p.st.ep_step[env] = (envfin || rst) ? 0 : ep_step + 1;
            p.st.gstep[env] = gstep + 1u;
            if (done) {
                const int k = ev.done_eps[env];
                const size_t out = (size_t)env + (size_t)k * N;
                ev.out_ret[out] = r64; ev.out_cost[out] = c64; ev.out_len[out] = len + 1;
                ev.done_eps[env] = k + 1;
                ev.left[env] = left - 1;
                ev.ret[env] = 0.0; ev.cost[env] = 0.0; ev.len[env] = 0;
            } else {
                ev.ret[env] = r64; ev.cost[env] = c64; ev.len[env] = len + 1;
            }
            for (int j = 0; j < O; ++j)
                s_nxt[(size_t)env * O + j] = rst ? env_reset_value(p.es, gid, epi_n, j)
                                                 : envfin ? env_reset_value(p.es, gid, epi_auto, j) : sn[j];
            f = 1 | (envfin ? 2 : 0) | (rst ? 4 : 0) | ((!done || left > 1) ? 8 : 0);
            sE1[tid] = epi_auto; sE2[tid] = epi_n;
        }
        sF[tid] = f;
    }
    __syncthreads();
    if (p.es.obs_normalize) {
        for (int j = tid; j < O; j += NTHREADS) {
            long long sx = 0, sxx = 0, fx = 0, fxx = 0, rx = 0, rxx = 0;
            for (int r = 0; r < R; ++r) {
                const int f = sF[r];
                if (!(f & 1)) continue;
                const uint32_t gid = p.es.env_id_offset + env0 + r;
                const float w = sn_all[(size_t)(env0 + r) * O + j];
                const float v = (f & 2) ? env_reset_value(p.es, gid, sE1[r], j) : w;
                sx += to_fix(v); sxx += to_fix(__fmul_rn(v, v));
                if (f & 2) { fx += to_fix(w); fxx += to_fix(__fmul_rn(w, w)); }
                if (f & 4) {
                    const float u = env_reset_value(p.es, gid, sE2[r], j);
                    rx += to_fix(u); rxx += to_fix(__fmul_rn(u, u));
                }
            }
            push_fix_sums(p.ns, O, j, sx, sxx, fx, fxx);
            if (rx != 0 || rxx != 0) {
                atomicAdd((unsigned long long*)(ev.acc_rst + j), (unsigned long long)rx);
                atomicAdd((unsigned long long*)(ev.acc_rst + O + j), (unsigned long long)rxx);
            }
        }
    }
    if (tid == 0) {
        int nfin = 0, nrst = 0, nnext = 0;
        for (int r = 0; r < R; ++r) {
            nfin += (sF[r] >> 1) & 1; nrst += (sF[r] >> 2) & 1; nnext += (sF[r] >> 3) & 1;
        }
        if (nfin) atomicAdd(p.ns.fin_count, nfin);
        if (nrst) atomicAdd(ev.ctr + 2, nrst);
        if (nnext) atomicAdd(ev.ctr + 1, nnext);
    }
}

// One CTA, after every CTA's eval_step of the step: pushes the step's rows into the statistics (final rows, next rows,
// reset rows: three pushes, as Normalizer.normalize is called three times) and advances the done word.
__device__ void eval_fold(const StepArgs& p) {
    const EvalSpec& ev = p.ev;
    __threadfence();
    const int nall = *((volatile int*)ev.ctr), nrst = *((volatile int*)(ev.ctr + 2));
    norm_fold(p.ns, p.es.O, nall, false, p.es.obs_normalize, ev.acc_rst, nrst);
    if (threadIdx.x == 0) {
        ev.ctr[0] = __ldcg(ev.ctr + 1);
        ev.ctr[1] = 0;
        ev.ctr[2] = 0;
    }
}

// Software grid barrier at the end of step t of a persistent (cooperative) launch: every CTA arrives, the last one runs
// on_last() (the step's fold into the running state) before it releases the others.  bar_ctr / bar_flag are zero at launch.
template <class F>
__device__ __forceinline__ void grid_step_barrier(const StepArgs& p, int t, int& s_last, F&& on_last) {
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = (atomicAdd(p.bar_ctr, 1u) == gridDim.x * gridDim.y * (unsigned)(t + 1) - 1u) ? 1 : 0;
    __syncthreads();
    if (s_last) {
        on_last();
        __threadfence();
        __syncthreads();
        if (threadIdx.x == 0) asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p.bar_flag), "r"((unsigned)(t + 1)) : "memory");
    } else if (threadIdx.x == 0) {
        unsigned v;
        do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p.bar_flag) : "memory"); } while (v < (unsigned)(t + 1));
    }
    __syncthreads();
}

// The same barrier without a last arriver's work: every CTA arrives and waits for the others.
__device__ __forceinline__ void grid_step_arrive_wait(const StepArgs& p, int t) {
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned all = gridDim.x * gridDim.y * (unsigned)(t + 1);
        unsigned v;
        asm volatile("atom.release.gpu.global.add.u32 %0, [%1], 1;" : "=r"(v) : "l"(p.bar_ctr) : "memory");
        ++v;
        while (v < all) asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p.bar_ctr) : "memory");
    }
    __syncthreads();
}

// EXT = true: the act half of a step on a user env (csrc: osb_ext_act).  The network part is the same; the actor CTAs
// hand the scaled action to the env through p.act_env instead of running the synthetic transition, and the normaliser is
// fed by the observe kernel after env.step.
// EVAL = true: a step of the evaluation of a saved policy (actor CTAs only, no slabs): eval_step on the synthetic env;
// EXT, the deterministic action into act_env for env.step (the observe half is ext_eval_observe_kernel).  A launch after
// every env has finished its episodes returns at once.
template <bool EXT, bool EVAL, int ACT>
__global__ void __launch_bounds__(NTHREADS) rollout_step_kernel(StepArgs p, NetSpec spec) {
    if constexpr (EVAL) {
        if (__ldcg(p.ev.ctr) == 0) return;
    }
    extern __shared__ __align__(16) float smem[];
    NetSmem W;
    float* base = carve_net_smem<false>(smem, W);
    float* sX = base;  base += RT * LD;
    float* sH1 = base; base += RT * LD;
    float* sH2 = base; base += RT * LD;
    float* sO = base;  base += RT * LDO;
    float* sMean = base; base += p.es.O;
    float* sStd = base;  base += p.es.O;
    float* sAct = base;  base += RT * OUTP;
    float* sNew = base;  base += RT * (KC + 1);
    float* sFin = base;  base += RT * (KC + 1);
    float* sRew = base;  base += RT;
    float* sCost = base; base += RT;
    int* sFlag = reinterpret_cast<int*>(base); base += RT;
    __shared__ int s_anyfin;

    const int net = p.is_tail ? (int)blockIdx.y + 1 : (int)blockIdx.y;
    const Hidden<ACT> af(spec, net);
    const int env0 = blockIdx.x * RT;
    const int O = p.es.O, A = p.es.A, N = p.N, t = p.t;
    const int On = O + (p.sa.safety ? 1 : 0);            // network input width (Saute: [obs | z])
    const float* z_cur = p.sa.safety ? p.sa.safety + (size_t)(t & 1) * N : nullptr;
    const int nchunks = (On + KC - 1) / KC;
    const NetLayout L = net_layout(net, On, A);
    const float* theta = p.theta + net_offset(net, On, A);
    const bool normalize = p.es.obs_normalize && p.ns.count[0] > 1;
    const float* s_cur = p.st.s_raw + (size_t)(t & 1) * N * O;
    float* s_nxt = p.st.s_raw + (size_t)((t + 1) & 1) * N * O;

    load_net_rest<false>(theta, L, W);
    load_w1_chunk(theta, L, 0, W);
    auto load_chunk_cur = [&](int kc) {
        load_w1_chunk(theta, L, kc, W);
        for (int j = threadIdx.x; j < O; j += NTHREADS) { sMean[j] = p.ns.mean[j]; sStd[j] = p.ns.std[j]; }
        load_obs_tile(s_cur, env0, N, O, kc, sMean, sStd, normalize, sX, nullptr, z_cur);
    };

    // ---- bootstrap values of paths that ended in the previous step (critic CTAs only) --------
    if (!EVAL && net != 0 && t > 0) {
        if (threadIdx.x == 0) s_anyfin = 0;
        __syncthreads();
        if (threadIdx.x < RT && env0 + threadIdx.x < N && cut_path(p.sl.flags[(size_t)(t - 1) * N + env0 + threadIdx.x]))
            s_anyfin = 1;
        __syncthreads();
        if (s_anyfin) {
            const bool norm1 = p.es.obs_normalize && p.ns.count[1] > 1;
            const float* fin = p.st.final_raw + (size_t)((t - 1) & 1) * N * O;
            auto load_chunk_fin = [&](int kc) {
                load_w1_chunk(theta, L, kc, W);
                for (int j = threadIdx.x; j < O; j += NTHREADS) { sMean[j] = p.ns.mean1[j]; sStd[j] = p.ns.std1[j]; }
                load_obs_tile(fin, env0, N, O, kc, sMean, sStd, norm1, sX, nullptr, z_cur, true);
            };
            for (int j = threadIdx.x; j < O; j += NTHREADS) { sMean[j] = p.ns.mean1[j]; sStd[j] = p.ns.std1[j]; }
            __syncthreads();
            load_obs_tile(fin, env0, N, O, 0, sMean, sStd, norm1, sX, nullptr, z_cur, true);
            __syncthreads();
            mlp_hidden<RT>(sX, sH1, sH2, W, nchunks, af, load_chunk_fin);
            mlp_out<RT>(sH2, sO, W, 1);
            if (threadIdx.x < RT && env0 + threadIdx.x < N)
                store_critic(p.sl, net, N, t, env0 + threadIdx.x, true, false, sO[threadIdx.x * LDO]);
            __syncthreads();
            if (nchunks > 1) { load_w1_chunk(theta, L, 0, W); }
        }
    }

    // ---- forward on the current observation ------------------------------------------------
    for (int j = threadIdx.x; j < O; j += NTHREADS) { sMean[j] = p.ns.mean[j]; sStd[j] = p.ns.std[j]; }
    __syncthreads();
    if (!EVAL && net == 0 && nchunks > 1) {
        // write the whole normalised observation row once (chunks > 0 are not revisited below)
        for (int kc = 1; kc < nchunks; ++kc)
            load_obs_tile(s_cur, env0, N, O, kc, sMean, sStd, normalize, sX,
                          p.sl.obs + (size_t)t * N * On, z_cur);
        __syncthreads();
    }
    load_obs_tile(s_cur, env0, N, O, 0, sMean, sStd, normalize, sX,
                  (!EVAL && net == 0) ? p.sl.obs + (size_t)t * N * On : nullptr, z_cur);
    __syncthreads();
    mlp_hidden<RT>(sX, sH1, sH2, W, nchunks, af, load_chunk_cur);
    mlp_out<RT>(sH2, sO, W, L.out);
    if constexpr (EVAL) {
        __syncthreads();
        if constexpr (EXT) {
            eval_action<RT, true>(p, env0, sO, LDO, theta + L.off_logstd);
        } else {
            eval_step<RT>(p, t, env0, sO, LDO, theta + L.off_logstd, sFlag, reinterpret_cast<uint32_t*>(sNew),
                          reinterpret_cast<uint32_t*>(sFin));
            if (last_cta(p.ns.ticket)) eval_fold(p);
        }
        return;
    }

    if (net != 0 && threadIdx.x < RT && env0 + threadIdx.x < N)
        store_critic(p.sl, net, N, t, env0 + threadIdx.x, false, p.is_tail, sO[threadIdx.x * LDO]);

    // ---- actor CTA: sample, log-prob ---------------------------------------------------------
    if (net == 0) {
        // thread -> (env e = tid / 8, lane q = tid % 8); action components a = q, q + 8
        const int e = threadIdx.x >> 3, q = threadIdx.x & 7;
        const int env = env0 + e;
        const bool ok = env < N;
        uint32_t gstep = p.global_step;
        if constexpr (EXT) gstep = act_global_step(p);
        float lp = 0.f;
        for (int a = q; a < A; a += 8) {
            const float mu = sO[e * LDO + a];
            const float sd = expf(__ldg(theta + L.off_logstd + a));
            float eps = 0.f;
            if (ok)
                eps = p.eps ? p.eps[(size_t)env * A + a]
                            : philox_normal(p.noise_seed, p.es.env_id_offset + env, gstep, a);
            float term;
            const float act = sample_action(mu, sd, __fmul_rn(2.f, __fmul_rn(sd, sd)), logf(sd), eps, term);
            lp += term;
            sAct[e * OUTP + a] = act;
            if (ok) store_action<EXT>(p, t, env, a, act);
        }
        lp += __shfl_xor_sync(0xffffffffu, lp, 1);
        lp += __shfl_xor_sync(0xffffffffu, lp, 2);
        lp += __shfl_xor_sync(0xffffffffu, lp, 4);
        if (ok && q == 0) p.sl.logp[(size_t)t * N + env] = lp;
    }
    if constexpr (EXT) return;
    __syncthreads();

    // ---- env transition ----------------------------------------------------------------------
    if (net == 0) {
        const int e = threadIdx.x >> 3, q = threadIdx.x & 7;
        const int env = env0 + e;
        const bool ok = env < N;
        const uint32_t gid = p.es.env_id_offset + env;
        int ep_step = 0, fl = 0; uint32_t epi = 0, gstep = 0;
        float acc_cost = 0.f;
        if (ok) {
            ep_step = p.st.ep_step[env]; epi = p.st.episode[env]; gstep = p.st.gstep[env];
            fl = episode_end(p.es, gid, ep_step, gstep);
            if (p.et.cost_acc) {
                acc_cost = __fadd_rn(p.et.cost_acc[env], env_step_cost(p.es, s_cur[(size_t)env * O], sAct[e * OUTP], __ldg(p.st.bias)));
                if (acc_cost > p.et.cost_limit) fl = early_end(fl);
            }
        }
        const bool fin = fl & EP_FIN;
        float part = 0.f, s0n = 0.f;
        float* finrow = p.st.final_raw + ((size_t)(t & 1) * N + (ok ? env : 0)) * O;
        for (int c0 = 0; c0 < O; c0 += KC) {
            for (int j = c0 + q; j < min(O, c0 + KC); j += 8) {
                float nv = 0.f, fv = 0.f;
                if (ok) {
                    const float a = env_action(sAct[e * OUTP + (j % A)]);
                    const float s = s_cur[(size_t)env * O + j];
                    const float sn = env_next_value(s, a, __ldg(p.st.bias + j));
                    part = __fadd_rn(part, __fmul_rn(sn, sn));
                    if (j == 0) s0n = sn;
                    fv = sn;
                    nv = fin ? env_reset_value(p.es, gid, next_episode(epi, fl), j) : sn;
                    s_nxt[(size_t)env * O + j] = nv;
                    if (fin) finrow[j] = sn;
                }
                sNew[e * (KC + 1) + (j - c0)] = nv;
                sFin[e * (KC + 1) + (j - c0)] = fin ? fv : 0.f;
            }
            if (c0 == 0 && q == 0) sFlag[e] = fin ? 1 : 0;
            __syncthreads();
            if (p.es.obs_normalize) {
                const int j = c0 + threadIdx.x;
                if (threadIdx.x < KC && j < O) {
                    long long sx = 0, sxx = 0, fx = 0, fxx = 0;
                    for (int r = 0; r < RT; ++r)
                        if (env0 + r < N) {
                            const float v = sNew[r * (KC + 1) + threadIdx.x];
                            sx += to_fix(v); sxx += to_fix(__fmul_rn(v, v));
                            if (sFlag[r]) {
                                const float w = sFin[r * (KC + 1) + threadIdx.x];
                                fx += to_fix(w); fxx += to_fix(__fmul_rn(w, w));
                            }
                        }
                    push_fix_sums(p.ns, O, j, sx, sxx, fx, fxx);
                }
            }
            __syncthreads();
        }
        // sum_j s'_j^2 in the fixed summation tree shared with the oracle
        part = __fadd_rn(part, __shfl_xor_sync(0xffffffffu, part, 1));
        part = __fadd_rn(part, __shfl_xor_sync(0xffffffffu, part, 2));
        part = __fadd_rn(part, __shfl_xor_sync(0xffffffffu, part, 4));
        if (ok && q == 0) synthetic_step_end(p, N, p.T, O, t, env, fl, part, s0n, ep_step, epi, gstep, acc_cost);
        if (p.es.obs_normalize && threadIdx.x == 0) {
            int nf = 0;
            for (int r = 0; r < RT; ++r) nf += (env0 + r < N) ? sFlag[r] : 0;
            if (nf) atomicAdd(p.ns.fin_count, nf);
        }
    }
    // every CTA (actor and critic) has now consumed the normaliser state of this step; the last
    // one to arrive folds the step's sums into it for the next launch.
    if (p.es.obs_normalize && !p.is_tail && last_cta(p.ns.ticket)) norm_fold(p.ns, O, N, true);
}

// ---------------------------------------------------------------------------------------------
// Tensor-core variant of the step kernel (train_cfgs.matmul_precision = tf32, O <= 64): tiles of 128
// envs, the forward of a network on the tensor-core tiles of csrc/tc_forward.cuh (X3 = false: tf32 (5e-3); X3 = true:
// split-bf16, fp32-level values / log-probs).  Everything around the forward (ObsNormalize, sampling, env transition,
// slab append, normaliser sums, ticket) is the arithmetic of rollout_step_kernel.
constexpr int RTC = TC_ROWS;
constexpr int RTA = 64;       // envs per actor tile of the persistent training kernel
constexpr int SNW = KC + 1;   // row stride of the next-state staging tiles

// the 4-byte-word region after the operand tiles (all offsets in words)
constexpr int TF_B1 = 0;                          // [64] layer biases
constexpr int TF_B2 = TF_B1 + 64;                 // [64]
constexpr int TF_B3 = TF_B2 + 64;                 // [16]
constexpr int TF_MEAN = TF_B3 + 16;               // [64] ObsNormalize mean
constexpr int TF_STD = TF_MEAN + 64;              // [64] ObsNormalize std
constexpr int TF_ACT = TF_STD + 64;               // [128][16] mu, then the sampled action
constexpr int TF_RAW = TF_ACT + RTC * OUTP;       // [128][65] raw current state of the tile (actor CTAs; kept by the obs staging)
constexpr int TF_SN = TF_RAW + RTC * SNW;         // [128][65] state after the transition, before any reset
constexpr int TF_ACC = TF_SN + RTC * SNW;         // long long [4][4][64] partial fixed-point sums
constexpr int TF_FLAG = TF_ACC + 2 * 4 * 4 * 64;  // [128] episode-end word (EP_*)
constexpr int TF_EPI = TF_FLAG + RTC;             // [128] episode counter
constexpr int TF_STEP = TF_EPI + RTC;             // [128] step inside the episode
constexpr int TF_GSTEP = TF_STEP + RTC;           // [128] total steps of the env (termination hash counter)
constexpr int TF_SD = TF_GSTEP + RTC;             // [3][16] sigma, 2 sigma^2, log sigma per action
constexpr int TF_EARLY = TF_SD + 48;              // [128] accumulated cost incl. this step (EarlyTerminated)
constexpr int TF_WORDS = TF_EARLY + RTC;
// persistent training kernel only: its own copy of the running statistics (NormStats)
constexpr int TF_NS = TF_WORDS;                   // [5][64] mean, sumsq, std, mean1, std1
constexpr int TF_NCNT = TF_NS + 5 * 64;           // long long [2] count, then int had_fin
constexpr int TF_WORDS_PERSIST = TF_NCNT + 6;
static_assert(TF_ACC % 2 == 0 && TF_NCNT % 2 == 0, "the fixed-point sums and counts need 8-byte alignment");

// The persistent training kernel's normaliser sums: a ring of three slots, step t adding into slot t % 3.  Slot layout
// in long longs: acc_all [2][O] at 0, acc_fin [2][O] at 128, fin_count (an int) at 256.
constexpr int RING_SLOT = 258;
__device__ __forceinline__ long long* ring_slot(long long* ring, int t) { return ring + (t % 3) * RING_SLOT; }

// PERSIST = true: ONE cooperative launch runs the whole epoch (steps 0 .. T, the last one being the critics' epoch-end
// bootstrap): the weight tiles, biases and the accumulator image allocation stay resident, every step ends in a grid barrier
// after which every CTA folds the step's normaliser sums into its own copy of the running statistics (RING below)
// (adapter/onpolicy_adapter.py:L58-136 is the loop this replaces).  Data written by other CTAs in earlier steps
// (raw states, flags, normaliser sums) is read with ld.global.cg.
// EXT = true: the act half of a step on a user env, as in rollout_step_kernel<true> (never persistent: Python runs
// env.step between the launches).
// EVAL = true: the evaluation of a saved policy, as in rollout_step_kernel<EXT, true>; PERSIST (synthetic env only): ONE
// cooperative launch runs every step until all envs have finished, the last CTA at each step's grid barrier running
// eval_fold.
template <bool X3, bool PERSIST, bool EXT, bool EVAL, int ACT>
__global__ void __launch_bounds__(NTHREADS, 1) rollout_step_tc_kernel(StepArgs p, NetSpec spec) {
    static_assert(!(EXT && PERSIST), "the external-env steps are one launch per step");
    if constexpr (EVAL) {
        if (__ldcg(p.ev.ctr) == 0) return;
    }
    using namespace umma;
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const uint32_t pad = (1024u - (smem_u32(smem_raw) & 1023u)) & 1023u;
    const uint32_t B0 = smem_u32(smem_raw) + pad;       // the X tile comes first (TcTiles::X == 0)
    float* fbase = reinterpret_cast<float*>(smem_raw + pad + TcTiles<X3>::FLOATS);
    float* sB1 = fbase + TF_B1;
    float* sB2 = fbase + TF_B2;
    float* sB3 = fbase + TF_B3;
    float* sMean = fbase + TF_MEAN;
    float* sStd = fbase + TF_STD;
    float* sAct = fbase + TF_ACT;
    float* sRaw = fbase + TF_RAW;
    float* sSn = fbase + TF_SN;
    long long* sAcc = reinterpret_cast<long long*>(fbase + TF_ACC);
    int* sFlag = reinterpret_cast<int*>(fbase + TF_FLAG);
    uint32_t* sEpi = reinterpret_cast<uint32_t*>(fbase + TF_EPI);
    int* sStep = reinterpret_cast<int*>(fbase + TF_STEP);
    uint32_t* sGstep = reinterpret_cast<uint32_t*>(fbase + TF_GSTEP);
    float* sSd = fbase + TF_SD;
    float* sEarlyAcc = fbase + TF_EARLY;
    // RING: the persistent training kernel.  Every CTA holds the running statistics in shared memory (sNs, loaded at
    // launch) and folds each step's sums from the ring into them after the step's barrier, so that the barrier is a
    // plain arrive / wait; the designated CTA clears the ring slot of step t - 2 in step t and writes sNs back to
    // NormState at the end.
    constexpr bool RING = PERSIST && !EVAL;
    const NormStats sNs{fbase + TF_NS, fbase + TF_NS + 64, fbase + TF_NS + 128, fbase + TF_NS + 192, fbase + TF_NS + 256,
                        reinterpret_cast<long long*>(fbase + TF_NCNT), reinterpret_cast<int*>(fbase + TF_NCNT + 4)};
    __shared__ uint64_t bar;
    __shared__ int s_last, s_anyfin;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int q = warp & 3, h = warp >> 2;
    const int O = p.es.O, A = p.es.A, N = p.N, T = p.T;
    // RING: a 1-D grid of ceil(N / RTA) actor CTAs on tiles of R = RTA envs, then ceil(N / RTC) CTAs per critic on tiles
    // of R = RTC envs (ring_grid).  Otherwise grid = (env tiles of RTC) x networks.
    const int n_act = (N + RTA - 1) / RTA, n_crit = (N + RTC - 1) / RTC, cb = (int)blockIdx.x - n_act;
    const int net = RING ? (cb < 0 ? 0 : 1 + cb / n_crit)
                         : PERSIST ? (int)blockIdx.y : (p.is_tail ? (int)blockIdx.y + 1 : (int)blockIdx.y);
    const int R = (RING && net == 0) ? RTA : RTC;
    const int env0 = RING ? (cb < 0 ? (int)blockIdx.x * RTA : (cb % n_crit) * RTC) : (int)blockIdx.x * RTC;
    const int On = O + (p.sa.safety ? 1 : 0);            // network input width (Saute: [obs | z]), <= 64 here
    const NetLayout L = net_layout(net, On, A);
    const float* theta = p.theta + net_offset(net, On, A);
    const int e_env = tid >> 1, e_half = tid & 1;       // actor CTAs: 2 threads per env in the transition
    const int my_env = env0 + e_env;
    const bool my_ok = (net == 0) && (!RING || e_env < R) && my_env < N;

    tc_stage_weights<X3>(B0, theta, L, On, sB1, sB2, sB3);
    if (net == 0 && tid < 16) {          // Normal(mu, sigma): sigma = exp(log_std) is state independent
        const float sd = (tid < A) ? expf(__ldg(theta + L.off_logstd + tid)) : 1.f;
        sSd[tid] = sd; sSd[16 + tid] = __fmul_rn(2.f, __fmul_rn(sd, sd)); sSd[32 + tid] = logf(sd);
    }
    if (tid == 0) { mbar_init(&bar, 1); mbar_init_fence(); s_anyfin = 0; }
    const bool designated = RING && blockIdx.x == gridDim.x - 1;   // a cost-critic CTA: off the actors' chain
    if constexpr (RING) {
        if (tid < O) {
            sNs.mean[tid] = __ldcg(p.ns.mean + tid); sNs.sumsq[tid] = __ldcg(p.ns.sumsq + tid);
            sNs.std[tid] = __ldcg(p.ns.std + tid);
            sNs.mean1[tid] = __ldcg(p.ns.mean1 + tid); sNs.std1[tid] = __ldcg(p.ns.std1 + tid);
        }
        if (tid == 0) { sNs.count[0] = __ldcg(p.ns.count); sNs.count[1] = __ldcg(p.ns.count + 1); *sNs.had_fin = __ldcg(p.ns.had_fin); }
    }
    __syncthreads();
    const Acc tm = acc_cta(p.acc, TC_COLS);
    const uint32_t lane_base = (uint32_t)(q * 32) << 16;
    uint32_t phase = 0;

    // development aid (tools/rollout_stage_times.py): clock64 stamps of thread 0 of the first actor and reward-critic CTA
    const bool dbg_on = PERSIST && p.dbg != nullptr && tid == 0 &&
                        (RING ? (blockIdx.x == 0 || cb == 0) : (blockIdx.x == 0 && blockIdx.y < 2));
    int dbg_n = 0;
#define RSTAMP(id) do { if (dbg_on && dbg_n < 250) { long long* d_ = p.dbg + (net ? 512 : 0); d_[1 + 2 * dbg_n] = (id); d_[2 + 2 * dbg_n] = clock64(); ++dbg_n; d_[0] = dbg_n; } } while (0)
    const int t_first = PERSIST ? 0 : p.t, t_last = PERSIST ? T : p.t;
#pragma unroll 1
    for (int t = t_first; t <= t_last; ++t) {
    const bool is_tail = t == T;
    if (PERSIST && is_tail && net == 0) break;          // the tail step is the critics' (no barrier follows it)
    if (EVAL && PERSIST && t > 0 && __ldcg(p.ev.ctr) == 0) break;   // every env has finished (uniform after the barrier)
    const float* eps_t = PERSIST ? (p.eps ? p.eps + (size_t)t * N * A : nullptr) : p.eps;
    const uint32_t gstep_t = PERSIST ? p.global_step + (uint32_t)t : p.global_step;
    const bool normalize = p.es.obs_normalize && (RING ? sNs.count[0] : __ldcg(p.ns.count)) > 1;
    const float* s_cur = p.st.s_raw + (size_t)(t & 1) * N * O;
    float* s_nxt = p.st.s_raw + (size_t)((t + 1) & 1) * N * O;
    if (PERSIST) { if (tid == 0) s_anyfin = 0; __syncthreads(); }
    // which envs of this tile finish in this step (time limit / hash-driven termination): known before the forward
    if (!EXT && !EVAL && net == 0 && tid < R) {
        const int env = env0 + tid;
        int fl = 0, ep_step = 0; uint32_t epi = 0, gstep = 0;
        if (env < N) {
            ep_step = p.st.ep_step[env]; epi = p.st.episode[env]; gstep = p.st.gstep[env];
            fl = episode_end(p.es, p.es.env_id_offset + env, ep_step, gstep);
        }
        sFlag[tid] = fl; sEpi[tid] = epi; sStep[tid] = ep_step; sGstep[tid] = gstep;
    }
    RSTAMP(1);

    // does this critic tile need bootstrap values for paths cut in the previous step?
    if (net != 0 && t > 0 && tid < RTC && env0 + tid < N && cut_path(__ldcg(p.sl.flags + (size_t)(t - 1) * N + env0 + tid)))
        s_anyfin = 1;
    __syncthreads();
    const int first_pass = (net != 0 && t > 0 && s_anyfin) ? 0 : 1;

    // pass 0: final observations of the previous step (critics, rare); pass 1: current observation
#pragma unroll 1
    for (int pass = first_pass; pass < 2; ++pass) {
        const float* raw = pass ? s_cur : p.st.final_raw + (size_t)((t - 1) & 1) * N * O;
        const float* gmean = RING ? (pass ? sNs.mean : sNs.mean1) : (pass ? p.ns.mean : p.ns.mean1);
        const float* gstd = RING ? (pass ? sNs.std : sNs.std1) : (pass ? p.ns.std : p.ns.std1);
        const bool norm_on = pass ? normalize : (p.es.obs_normalize && (RING ? sNs.count[1] : __ldcg(p.ns.count + 1)) > 1);
        float* obs_out = (!EVAL && pass && net == 0) ? p.sl.obs + (size_t)t * N * On : nullptr;
        const bool own_state = !EVAL && PERSIST && pass && net == 0 && t > t_first;
        if (tid < 64) {
            sMean[tid] = (tid < O) ? (RING ? gmean[tid] : __ldcg(gmean + tid)) : 0.f;
            sStd[tid] = (tid < O) ? (RING ? gstd[tid] : __ldcg(gstd + tid)) : 1.f;
        }
        __syncthreads();
        if ((O & 3) == 0 && On == O) {   // 128-bit row loads, all 8 in flight per thread
            const int kq = tid & 15, k4 = kq << 2;
            float4 xv[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int env = (!RING || 16 * j < R) ? env0 + (tid >> 4) + 16 * j : N;   // rows past the tile: not loaded
                if (own_state) {          // persistent kernel, actor CTA: the state this CTA wrote in the previous step is still in smem
                    const float* r = sRaw + ((tid >> 4) + 16 * j) * SNW + k4;
                    xv[j] = (env < N && k4 < O) ? make_float4(r[0], r[1], r[2], r[3]) : make_float4(0.f, 0.f, 0.f, 0.f);
                } else
                xv[j] = (env < N && k4 < O) ? __ldcg(reinterpret_cast<const float4*>(raw + (size_t)env * O + k4))
                                            : make_float4(0.f, 0.f, 0.f, 0.f);
            }
            const float m0 = sMean[k4], m1 = sMean[k4 + 1], m2 = sMean[k4 + 2], m3 = sMean[k4 + 3];
            const float s0 = sStd[k4], s1 = sStd[k4 + 1], s2 = sStd[k4 + 2], s3 = sStd[k4 + 3];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                if constexpr (RING) {
                    if (16 * j >= R) break;
                }
                const int e = (tid >> 4) + 16 * j;
                const int env = env0 + e;
                float4 v = xv[j];
                if (pass && net == 0 && k4 < O) { float* r = sRaw + e * SNW + k4; r[0] = v.x; r[1] = v.y; r[2] = v.z; r[3] = v.w; }
                if (env < N && k4 < O) {
                    if (norm_on) {
                        v.x = norm_clip(v.x, m0, s0);
                        v.y = norm_clip(v.y, m1, s1);
                        v.z = norm_clip(v.z, m2, s2);
                        v.w = norm_clip(v.w, m3, s3);
                    }
                    if (obs_out) *reinterpret_cast<float4*>(obs_out + (size_t)env * O + k4) = v;
                }
                if constexpr (X3) {
                    uint32_t w0[2], w1[2], w2[2];
                    x3::split2(v.x, v.y, w0[0], w1[0], w2[0]);
                    x3::split2(v.z, v.w, w0[1], w1[1], w2[1]);
                    const uint32_t o = B0 + x3::off128(e, k4);
                    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(o), "r"(w0[0]), "r"(w0[1]) : "memory");
                    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(o + TcTiles<true>::SUB), "r"(w1[0]), "r"(w1[1]) : "memory");
                    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(o + 2 * TcTiles<true>::SUB), "r"(w2[0]), "r"(w2[1]) : "memory");
                } else {
                asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(tile_addr(B0, e, k4, RTC)),
                             "f"(tf32r(v.x)), "f"(tf32r(v.y)), "f"(tf32r(v.z)), "f"(tf32r(v.w))
                             : "memory");
                }
            }
        } else {
            const int k = tid & 63;
            const float mk = sMean[k], sk = sStd[k];
#pragma unroll 1
            for (int j0 = 0; j0 < 32; j0 += 8) {   // 8 rows at a time, their loads all in flight
                if constexpr (RING) {
                    if (4 * j0 >= R) break;                       // rows past the actor tile
                }
                float xv[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    const int e = (tid >> 6) + 4 * (j0 + u), env = env0 + e;
                    xv[u] = (env < N && k < O) ? (own_state ? sRaw[e * SNW + k] : __ldcg(raw + (size_t)env * O + k)) : 0.f;
                }
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    const int e = (tid >> 6) + 4 * (j0 + u), env = env0 + e;
                    float v = xv[u];
                    if (env < N && k < O) {
                        if (pass && net == 0) sRaw[e * SNW + k] = v;
                        if (norm_on) v = norm_clip(v, mk, sk);
                        if (obs_out) obs_out[(size_t)env * On + k] = v;
                    }
                    if constexpr (X3) x3::store1_x3(B0, TcTiles<true>::SUB, x3::off128(e, k), v);
                    else sts(tile_addr(B0, e, k, RTC), tf32r(v));
                }
            }
        }
        if (On != O) {          // Saute: column O of the tile = the safety state (1 on final observations)
            __syncthreads();    // the staging loop above zero-filled that column
            if (tid < R) {
                const int env = env0 + tid;
                float z = 0.f;
                if (env < N) {
                    z = pass ? __ldcg(p.sa.safety + (size_t)(t & 1) * N + env) : 1.f;
                    if (obs_out) obs_out[(size_t)env * On + O] = z;
                }
                if constexpr (X3) x3::store1_x3(B0, TcTiles<true>::SUB, x3::off128(tid, O), z);
                else sts(tile_addr(B0, tid, O, RTC), tf32r(z));
            }
        }
        fence_async_smem();
        __syncthreads();
        RSTAMP(2);
        auto stamp = [&](int l) {   // bf16x3: stamps 3-5, one per layer
            if (X3) RSTAMP(2 + l);
        };
        // bf16x3 actor tiles of RTA = 64 envs: one m64 block per layer.  tf32 runs its 128-row forward on them too, rows
        // past the tile computing values nobody reads.
        const Hidden<ACT, TcTanh<X3>> af(spec, net);
        if constexpr (X3 && RING) {
            if (net == 0) tc_forward<X3, RTA>(B0, tm, &bar, phase, sB1, sB2, 1, af, TcNop{}, stamp);
            else tc_forward<X3>(B0, tm, &bar, phase, sB1, sB2, 1, af, TcNop{}, stamp);
        } else {
            tc_forward<X3>(B0, tm, &bar, phase, sB1, sB2, 1, af, TcNop{}, stamp);
        }
        if (h == 0) {
            float o16[16];
            acc_ld16(tm, lane_base + TC_C_OUT, o16);
            const int e = 32 * q + lane;
            const int env = env0 + e;
            if (net != 0) {
                if (env < N) store_critic(p.sl, net, N, t, env, pass == 0, is_tail, o16[0] + sB3[0]);
            } else {
#pragma unroll
                for (int a = 0; a < 16; ++a) sAct[e * OUTP + a] = o16[a] + sB3[a];   // mu
            }
        }
        __syncthreads();
    }
    if constexpr (EVAL) {
        if constexpr (EXT) {
            eval_action<RTC, true>(p, env0, sAct, OUTP, theta + L.off_logstd);
            return;
        } else {
            eval_step<RTC>(p, t, env0, sAct, OUTP, theta + L.off_logstd, sFlag, sEpi, reinterpret_cast<uint32_t*>(sStep));
            if constexpr (PERSIST) {
                grid_step_barrier(p, t, s_last, [&] { eval_fold(p); });
                continue;
            } else {
                if (last_cta(p.ns.ticket)) eval_fold(p);
                return;
            }
        }
    }

    RSTAMP(6);
    if (net == 0) {
        // ---- sample + log-prob.  A <= 8: thread -> (env e = 64 g + tid / 4, action pair pr = tid % 4): one Philox block
        //      yields both normals of the pair (Box-Muller cos / sin); the log-prob terms are summed in the tree
        //      ((t0+t1)+(t2+t3)) + ((t4+t5)+(t6+t7)) of rollout_step_kernel.  A > 8: one action per lane as there. -----------
        if (A <= 8) {
            const int pr = tid & 3, a0 = 2 * pr, a1 = a0 + 1;
#pragma unroll 1
            for (int g = 0; 64 * g < R; ++g) {
                const int e = 64 * g + (tid >> 2);
                const int env = env0 + e;
                const bool ok = env < N;
                float2 n = make_float2(0.f, 0.f);
                if (ok && a0 < A) {
                    if (eps_t) { n.x = eps_t[(size_t)env * A + a0]; n.y = (a1 < A) ? eps_t[(size_t)env * A + a1] : 0.f; }
                    else n = philox_normal2(p.noise_seed, p.es.env_id_offset + env, EXT ? act_global_step(p) : gstep_t, pr);
                }
                float lp = 0.f;
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    const int a = a0 + u;
                    if (a < A) {
                        float term;
                        const float act = sample_action(sAct[e * OUTP + a], sSd[a], sSd[16 + a], sSd[32 + a], u ? n.y : n.x, term);
                        lp += term;
                        sAct[e * OUTP + a] = act;
                        if (ok) store_action<EXT>(p, t, env, a, act);
                    }
                }
                lp += __shfl_xor_sync(0xffffffffu, lp, 1);
                lp += __shfl_xor_sync(0xffffffffu, lp, 2);
                if (ok && pr == 0) p.sl.logp[(size_t)t * N + env] = lp;
            }
        } else {
            const int qq = tid & 7;
#pragma unroll 1
            for (int g = 0; 32 * g < R; ++g) {
                const int e = 32 * g + (tid >> 3);
                const int env = env0 + e;
                const bool ok = env < N;
                float lp = 0.f;
                for (int a = qq; a < A; a += 8) {
                    float eps = 0.f;
                    if (ok)
                        eps = eps_t ? eps_t[(size_t)env * A + a]
                                    : philox_normal(p.noise_seed, p.es.env_id_offset + env, EXT ? act_global_step(p) : gstep_t, a);
                    float term;
                    const float act = sample_action(sAct[e * OUTP + a], sSd[a], sSd[16 + a], sSd[32 + a], eps, term);
                    lp += term;
                    sAct[e * OUTP + a] = act;
                    if (ok) store_action<EXT>(p, t, env, a, act);
                }
                lp += __shfl_xor_sync(0xffffffffu, lp, 1);
                lp += __shfl_xor_sync(0xffffffffu, lp, 2);
                lp += __shfl_xor_sync(0xffffffffu, lp, 4);
                if (ok && qq == 0) p.sl.logp[(size_t)t * N + env] = lp;
            }
        }
        if constexpr (EXT) return;
        __syncthreads();
        if (p.et.cost_acc) {      // EarlyTerminated: the step's cost is known from state dim 0 -> finish flags before the transition
            if (tid < R && env0 + tid < N) {
                const int env = env0 + tid;
                const float acc = __fadd_rn(p.et.cost_acc[env], env_step_cost(p.es, sRaw[tid * SNW], sAct[tid * OUTP], __ldg(p.st.bias)));
                if (acc > p.et.cost_limit) sFlag[tid] = early_end(sFlag[tid]);
                sEarlyAcc[tid] = acc;
            }
            __syncthreads();
        }
        RSTAMP(7);
        // ---- env transition + normaliser sums, elementwise: thread -> (dim j = tid % 64, env quarter g = tid / 64 of the
        //      tile's R envs).
        //      The raw state comes from shared memory (kept by the obs staging), the next state goes out in whole
        //      rows (coalesced), the fixed-point column sums accumulate in registers. ---------------------------------------
        {
            const int j = tid & 63, g = tid >> 6, eq = R >> 2;
            long long sx = 0, sxx = 0, fx = 0, fxx = 0;
            if (j < O) {
                const int ja = j % A;
                const float bj = __ldg(p.st.bias + j);
#pragma unroll 4
                for (int e = eq * g; e < eq * g + eq; ++e) {
                    const int env = env0 + e;
                    if (env < N) {
                        const float a = env_action(sAct[e * OUTP + ja]);
                        const float sn = env_next_value(sRaw[e * SNW + j], a, bj);
                        const int fl = sFlag[e];
                        float nv = sn;
                        if (fl & EP_FIN) {
                            nv = env_reset_value(p.es, p.es.env_id_offset + env, next_episode(sEpi[e], fl), j);
                            p.st.final_raw[((size_t)(t & 1) * N + env) * O + j] = sn;
                            fx += to_fix(sn); fxx += to_fix(__fmul_rn(sn, sn));
                        }
                        s_nxt[(size_t)env * O + j] = nv;
                        if (PERSIST) sRaw[e * SNW + j] = nv;            // next step's obs staging of this CTA reads it back from here
                        sSn[e * SNW + j] = sn;
                        sx += to_fix(nv); sxx += to_fix(__fmul_rn(nv, nv));
                    }
                }
            }
            if (p.es.obs_normalize) {
                sAcc[(g * 4 + 0) * 64 + j] = sx; sAcc[(g * 4 + 1) * 64 + j] = sxx;
                sAcc[(g * 4 + 2) * 64 + j] = fx; sAcc[(g * 4 + 3) * 64 + j] = fxx;
            }
        }
        __syncthreads();
        RSTAMP(8);
        // ---- reward / cost / flags / episode bookkeeping: 2 threads per env.  Thread `e_half` owns the partial sums
        //      p_q, q = 4*e_half .. 4*e_half+3 (dims j = q mod 8): the summation tree is the one of the spec
        //      ((p0+p1)+(p2+p3)) + ((p4+p5)+(p6+p7)). ------------------------------------------------------------------
        {
            const int env = my_env;
            const bool ok = my_ok;
            float part[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
            for (int jb = 4 * e_half; jb < O; jb += 8) {
#pragma unroll
                for (int qi = 0; qi < 4; ++qi) {
                    const int j = jb + qi;
                    if (j < O) { const float sn = sSn[e_env * SNW + j]; part[qi] = __fadd_rn(part[qi], __fmul_rn(sn, sn)); }
                }
            }
            float tot = __fadd_rn(__fadd_rn(part[0], part[1]), __fadd_rn(part[2], part[3]));
            tot = __fadd_rn(tot, __shfl_xor_sync(0xffffffffu, tot, 1));
            if (ok && e_half == 0)
                synthetic_step_end(p, N, T, O, t, env, sFlag[e_env], tot, sSn[e_env * SNW], sStep[e_env], sEpi[e_env], sGstep[e_env],
                                   sEarlyAcc[e_env]);
        }
        if (p.es.obs_normalize) {
            NormState ns = p.ns;
            if constexpr (RING) {
                long long* slot = ring_slot(p.ring, t);
                ns.acc_all = slot; ns.acc_fin = slot + 128; ns.fin_count = reinterpret_cast<int*>(slot + 256);
            }
            if (tid < O) {
                long long a0 = 0, a1 = 0, a2 = 0, a3 = 0;
                for (int gg = 0; gg < 4; ++gg) {
                    a0 += sAcc[(gg * 4 + 0) * 64 + tid]; a1 += sAcc[(gg * 4 + 1) * 64 + tid];
                    a2 += sAcc[(gg * 4 + 2) * 64 + tid]; a3 += sAcc[(gg * 4 + 3) * 64 + tid];
                }
                push_fix_sums(ns, O, tid, a0, a1, a2, a3);
            }
            if (tid == 64) {
                int nfin = 0;
                for (int r = 0; r < R; ++r) nfin += (env0 + r < N) ? (sFlag[r] & EP_FIN) : 0;
                if (nfin) atomicAdd(ns.fin_count, nfin);
            }
        }
    }
    RSTAMP(9);
    if constexpr (RING) {
        if (!is_tail) {
            if (designated) {   // slot (t + 1) % 3 held step t - 2's sums, which every CTA folded before barrier t - 1
                long long* slot = ring_slot(p.ring, t + 1);
                for (int i = tid; i < RING_SLOT; i += NTHREADS) slot[i] = 0;
            }
            grid_step_arrive_wait(p, t);
            RSTAMP(10);
            if (p.es.obs_normalize) {
                const long long* slot = ring_slot(p.ring, t);
                norm_fold_stats(sNs, [](const float* a) { return *a; }, O, sNs.count[0], __ldcg(reinterpret_cast<const int*>(slot + 256)),
                                slot, slot + 128, N, true, true, nullptr, 0, [](int) {});
                __syncthreads();
                RSTAMP(11);
            }
        }
    } else if (!EXT && p.es.obs_normalize && !is_tail && last_cta(p.ns.ticket)) {
        norm_fold(p.ns, O, N, true);
    }
    }   // step loop
#undef RSTAMP
    __syncthreads();
    if (designated) {   // the host, checkpoints and the next epoch read the running statistics from NormState
        if (tid < O) {
            p.ns.mean[tid] = sNs.mean[tid]; p.ns.sumsq[tid] = sNs.sumsq[tid]; p.ns.std[tid] = sNs.std[tid];
            p.ns.mean1[tid] = sNs.mean1[tid]; p.ns.std1[tid] = sNs.std1[tid];
        }
        if (tid == 0) { p.ns.count[0] = sNs.count[0]; p.ns.count[1] = sNs.count[1]; *p.ns.had_fin = *sNs.had_fin; }
    }
}

// 1024: the alignment pad in front of the operand tiles.  ring: the persistent training kernel (its NormStats copy).
static size_t rollout_tc_smem_bytes(bool x3, bool ring) {
    return 1024 + (x3 ? TcTiles<true>::FLOATS : TcTiles<false>::FLOATS) + (ring ? TF_WORDS_PERSIST : TF_WORDS) * sizeof(float) + 64;
}

// ---------------------------------------------------------------------------------------------
// External envs (a user CMDP stepped in PyTorch): the observe half of a step, after env.step, and the ingest of the
// reset observations at epoch start (onpolicy_adapter.py:L80).  Elementwise over tiles of XT envs: slab append, episode
// bookkeeping (onpolicy_adapter.py:L138-175), next / final observations into the parity buffers the act kernels read,
// and ObsNormalize (wrapper.py:L231-241: final rows first -> mean1 / std1, then all rows).
//
// The observations of a user env have no bound, so the fixed-point sums of the synthetic path do not apply: each tile
// writes fp64 (mean, M2) per column of its rows, and the last CTA (ticket) combines them in tile order (Chan et al.) --
// no floating-point atomics, the same result on every run.  ext_tile_moments and ext_fold_push below are that push for
// the training observe, the evaluation observe and the reset rows alike.
constexpr int XT = 32;

struct ExtObs {
    const float* next_obs;      // [N][O] raw observation after the step (rows that finished are already reset)
    const float* rew;           // [N]
    const float* cost;          // [N]
    const uint8_t* term;        // [N]
    const uint8_t* trunc;       // [N]
    const float* final_obs;     // [N][O] or null
    const uint8_t* final_mask;  // [N] rows of final_obs that hold a final observation, or null
    double* part;               // the push's workspace (ext_tile_moments)
    int* nonfinite;             // [1] set to 1 when an observation is not finite
};

__device__ __forceinline__ void chan_combine(double& n, double& m, double& q, double nk, double mk, double qk) {
    if (nk == 0.0) return;
    if (n == 0.0) { n = nk; m = mk; q = qk; return; }
    const double nn = n + nk, d = mk - m;
    m += d * nk / nn;
    q += qk + d * d * n * nk / nn;
    n = nn;
}

// The tile half of the fp64 ObsNormalize push, for the CTA's tile of rows envs from env0.  Per column, two passes over
// the rows (ascending) give (mean, M2) of set A -- rows r of a with inA[r], every row when ALL -- and of set B -- rows r
// of b with inB[r], none without FIN; a mean over no rows is 0.  part: [tiles][4][O] (A mean, A M2, B mean, B M2), then
// [tiles][2] (A rows, B rows).  moments = false writes the row counts only.  Returns whether this CTA is the last on
// the ticket.
template <bool ALL, bool FIN>
__device__ __forceinline__ bool ext_tile_moments(double* part, const float* a, const int* inA, const float* b,
                                                 const int* inB, int O, int env0, int rows, bool moments,
                                                 unsigned int* ticket) {
    const int tid = threadIdx.x, tile = blockIdx.x, ntiles = gridDim.x;
    int na = ALL ? rows : 0, nb = 0;
    for (int r = 0; r < rows; ++r) {
        if constexpr (!ALL) na += inA[r];
        if constexpr (FIN) nb += inB[r];
    }
    double* P = part + (size_t)tile * 4 * O;
    for (int j = tid; moments && j < O; j += NTHREADS) {
        double s = 0.0, sf = 0.0;
        for (int r = 0; r < rows; ++r) {
            const size_t g = (size_t)(env0 + r) * O + j;
            if (ALL || inA[r]) s += (double)a[g];
            if (FIN && inB[r]) sf += (double)b[g];
        }
        const double m = na ? s / na : 0.0, mf = nb ? sf / nb : 0.0;
        double q = 0.0, qf = 0.0;
        for (int r = 0; r < rows; ++r) {
            const size_t g = (size_t)(env0 + r) * O + j;
            if (ALL || inA[r]) { const double d = (double)a[g] - m; q += d * d; }
            if (FIN && inB[r]) { const double df = (double)b[g] - mf; qf += df * df; }
        }
        P[j] = m; P[O + j] = q; P[2 * O + j] = mf; P[3 * O + j] = qf;
    }
    double* cnt = part + (size_t)ntiles * 4 * O;
    if (tid == 0) { cnt[2 * tile] = (double)na; cnt[2 * tile + 1] = (double)nb; }
    return last_cta(ticket);
}

// The last CTA's half: combine the tiles in tile order and push set B, then set A, into ns (norm_fold's sequence); a
// set with no rows is not pushed, and with no row in either the statistics are untouched.  Then count[0] and the
// ticket.  ALL (the training observe): set A is all N envs, its tile counts follow from N, and the set-B push is also
// kept as mean1 / std1 with count[1] and had_fin, for the truncation bootstraps of the next act launch.
template <bool ALL, bool FIN>
__device__ __forceinline__ void ext_fold_push(const double* part, NormState ns, int O, int N, bool moments) {
    __shared__ int s_na, s_nb;
    const int tid = threadIdx.x, ntiles = gridDim.x;
    __threadfence();
    const double* cnt = part + (size_t)ntiles * 4 * O;
    if (tid == 0) {
        int a = 0, b = 0;
        for (int k = 0; k < ntiles; ++k) {
            if constexpr (!ALL) a += (int)__ldcg(cnt + 2 * k);
            if constexpr (FIN) b += (int)__ldcg(cnt + 2 * k + 1);
        }
        s_na = a; s_nb = b;
    }
    __syncthreads();
    const int na = ALL ? N : s_na, nb = FIN ? s_nb : 0;
    const long long count = __ldcg(ns.count);
    for (int j = tid; moments && (na > 0 || nb > 0) && j < O; j += NTHREADS) {
        double n = 0.0, m = 0.0, q = 0.0, nF = 0.0, mF = 0.0, qF = 0.0;
        for (int k = 0; k < ntiles; ++k) {
            const double* Pk = part + (size_t)k * 4 * O;
            chan_combine(n, m, q, ALL ? (double)min(XT, N - k * XT) : __ldcg(cnt + 2 * k), __ldcg(Pk + j),
                         __ldcg(Pk + O + j));
            if constexpr (FIN)
                chan_combine(nF, mF, qF, __ldcg(cnt + 2 * k + 1), __ldcg(Pk + 2 * O + j), __ldcg(Pk + 3 * O + j));
        }
        float mean = __ldcg(ns.mean + j), sumsq = __ldcg(ns.sumsq + j);
        long long c = count;
        if (nb > 0) {
            norm_push_moments(mean, sumsq, c, nb, mF, qF);
            c += nb;
            if constexpr (ALL) {
                ns.mean1[j] = mean;
                ns.std1[j] = norm_std(sumsq, c);
            }
        }
        if (na > 0) {
            norm_push_moments(mean, sumsq, c, na, m, q);
            c += na;
        }
        ns.mean[j] = mean;
        ns.sumsq[j] = sumsq;
        ns.std[j] = norm_std(sumsq, c);
    }
    __syncthreads();
    if (tid == 0) {
        if constexpr (ALL) {
            ns.count[1] = count + nb;
            *ns.had_fin = nb > 0 ? 1 : 0;
        }
        ns.count[0] = count + nb + na;
        *ns.ticket = 0u;
    }
}

// EARLY: EarlyTerminatedAdapter.step on top of the step (early_terminated_adapter.py:L77-87), one thread per env.  The
// env's raw cost goes into the accumulator; once it exceeds cost_limit the step stores reward 0 (in the slab and in the
// episode return), terminated = 1 and truncated as the env reported it, the accumulator is cleared, and trig[env] = 1
// asks the host to reset the env (ext_reset_rows_kernel then ingests the reset observation).  An ordinary episode end
// leaves the accumulator alone.  trig_total, when not null, receives the number of triggered envs (zeroed by the host
// before the launch).  The observation rows are those env.step returned, so ObsNormalize pushes the env's own final rows
// and then every next row, a triggered env that did not end contributing its pre-reset state.
//
// WRAP: the step of an env behind TimeLimit / AutoReset (wrapper.py), after ext_wrapper_step_kernel and the reset of the
// done envs.  The launcher passes the step's own rows as both next_obs and final_obs, the done mask as final_mask and
// the wrapper's truncated as trunc; the next row of a done env comes from reset_obs instead.  So a done env's final row
// is its step row, and set A of the push is the next rows as they land in the state buffer: AutoReset's reset row sits
// inside ObsNormalize, in the same batch as every other env's next row.
template <bool EARLY, bool WRAP = false>
__device__ __forceinline__ void ext_observe_step(ExtObs x, EnvState st, NormState ns, Slabs sl, int O, int N, int T, int t,
                                                 int obs_normalize, int is_reset, EarlySpec et, uint8_t* trig,
                                                 int* trig_total, const float* reset_obs = nullptr) {
    __shared__ int sFin[XT];
    __shared__ int s_bad;
    const int tid = threadIdx.x, env0 = blockIdx.x * XT, rows = min(XT, N - env0);
    if (tid == 0) s_bad = 0;
    if (tid < XT) {
        const int env = env0 + tid;
        int fin = 0;
        if (tid < rows) {
            if (is_reset) {
                st.ep_ret[env] = 0.f; st.ep_cost[env] = 0.f; st.ep_len[env] = 0;
            } else {
                fin = (x.final_obs && x.final_mask && x.final_mask[env]) ? 1 : 0;
                if constexpr (EARLY) {
                    const float acc = __fadd_rn(et.cost_acc[env], x.cost[env]);
                    const bool hit = acc > et.cost_limit;
                    et.cost_acc[env] = hit ? 0.f : acc;
                    trig[env] = hit ? 1 : 0;
                    if (hit && trig_total) atomicAdd(trig_total, 1);
                    const float r = hit ? 0.f : x.rew[env];
                    record_step(sl, st, T, N, t, env, r, r, x.cost[env], hit || x.term[env] != 0, x.trunc[env] != 0);
                } else {
                    const float r = x.rew[env];
                    record_step(sl, st, T, N, t, env, r, r, x.cost[env], x.term[env] != 0, x.trunc[env] != 0);
                }
            }
        }
        sFin[tid] = fin;
    }
    __syncthreads();

    // step t reads parity t & 1, so the reset observation goes to buffer 0 and the next one of step t to (t + 1) & 1
    float* s_nxt = st.s_raw + (size_t)(is_reset ? 0 : ((t + 1) & 1)) * N * O;
    float* fin_out = st.final_raw + (size_t)(t & 1) * N * O;
    bool bad = false;
    for (int i = tid; i < rows * O; i += NTHREADS) {
        const int r = i / O;
        const size_t g = (size_t)env0 * O + i;
        if constexpr (WRAP) {
            const float f = x.next_obs[g];
            bad |= !isfinite(f);
            float v = f;
            if (sFin[r]) {
                fin_out[g] = f;
                v = reset_obs[g];
                bad |= !isfinite(v);
            }
            s_nxt[g] = v;
        } else {
            const float v = x.next_obs[g];
            bad |= !isfinite(v);
            s_nxt[g] = v;
            if (sFin[r]) {
                const float f = x.final_obs[g];
                bad |= !isfinite(f);
                fin_out[g] = f;
            }
        }
    }
    if (bad) s_bad = 1;
    if (!obs_normalize) {
        __syncthreads();
        if (tid == 0 && s_bad) *x.nonfinite = 1;
        return;
    }
    if constexpr (WRAP) __syncthreads();       // set A is read back from the state buffer the tile just wrote
    // set A: every next row; set B: the final rows
    const bool last = ext_tile_moments<true, true>(x.part, WRAP ? s_nxt : x.next_obs, nullptr, x.final_obs, sFin, O, env0,
                                                   rows, true, ns.ticket);
    if (tid == 0 && s_bad) *x.nonfinite = 1;
    if (last) ext_fold_push<true, true>(x.part, ns, O, N, true);
}

__global__ void __launch_bounds__(NTHREADS) ext_observe_kernel(ExtObs x, EnvState st, NormState ns, Slabs sl, int O, int N,
                                                               int T, int t, int obs_normalize, int is_reset) {
    ext_observe_step<false>(x, st, ns, sl, O, N, T, t, obs_normalize, is_reset, EarlySpec{nullptr, 0.f}, nullptr, nullptr);
}

__global__ void __launch_bounds__(NTHREADS) ext_observe_early_kernel(ExtObs x, EnvState st, NormState ns, Slabs sl,
                                                                     int O, int N, int T, int t, int obs_normalize,
                                                                     EarlySpec et, uint8_t* trig, int* trig_total) {
    ext_observe_step<true>(x, st, ns, sl, O, N, T, t, obs_normalize, 0, et, trig, trig_total);
}

__global__ void __launch_bounds__(NTHREADS) ext_observe_wrapped_kernel(ExtObs x, EnvState st, NormState ns, Slabs sl,
                                                                       int O, int N, int T, int t, int obs_normalize,
                                                                       const float* __restrict__ reset_obs) {
    ext_observe_step<false, true>(x, st, ns, sl, O, N, T, t, obs_normalize, 0, EarlySpec{nullptr, 0.f}, nullptr, nullptr,
                                  reset_obs);
}

// TimeLimit and AutoReset (wrapper.py) around env.step for the envs of a wrapped user env, one thread per env.  steps[env]
// is TimeLimit's _time: incremented by the step, cleared where the env is done (AutoReset's reset goes through
// TimeLimit.reset).  With time_limit > 0 the step's truncated is steps >= time_limit, replacing the env's own flag;
// with 0 (no TimeLimit) it is the env's flag.  done[env] = terminated | truncated: the envs to reset before the observe
// launch.  done_total, when not null, receives the number of done envs (zeroed by the host before the launch).
__global__ void __launch_bounds__(256) ext_wrapper_step_kernel(const uint8_t* __restrict__ term,
                                                               const uint8_t* __restrict__ env_trunc, int* steps,
                                                               uint8_t* trunc, uint8_t* done, int* done_total, int N,
                                                               int time_limit) {
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env >= N) return;
    const int k = steps[env] + 1;
    const bool tr = time_limit > 0 ? k >= time_limit : env_trunc[env] != 0;
    const bool d = tr || term[env] != 0;
    steps[env] = d ? 0 : k;
    trunc[env] = tr ? 1 : 0;
    done[env] = d ? 1 : 0;
    if (d && done_total) atomicAdd(done_total, 1);
}

// The reset observations of the envs the cost rule cut at step t (rows of obs where mask is set; the others are ignored)
// into the state buffer step t + 1 reads, and their ObsNormalize push (ObsNormalize.reset, wrapper.py:L243-261) after the
// step's own pushes, the masked rows as set A of the fp64 push, so the row count stays on the device.  No masked row:
// the statistics are untouched.  mean1 / std1 / had_fin keep the values of the step's final-row push, which the next
// act launch's truncation bootstraps read.
__global__ void __launch_bounds__(NTHREADS, 1) ext_reset_rows_kernel(const float* __restrict__ obs,
                                                                  const uint8_t* __restrict__ mask, float* s_nxt,
                                                                  NormState ns, double* part, int* nonfinite, int O,
                                                                  int N, int obs_normalize) {
    __shared__ int sM[XT];
    __shared__ int s_bad;
    const int tid = threadIdx.x, env0 = blockIdx.x * XT, rows = min(XT, N - env0);
    if (tid == 0) s_bad = 0;
    if (tid < XT) sM[tid] = (tid < rows && mask[env0 + tid] != 0) ? 1 : 0;
    __syncthreads();
    bool bad = false;
    for (int i = tid; i < rows * O; i += NTHREADS) {
        if (sM[i / O]) {
            const size_t g = (size_t)env0 * O + i;
            const float v = obs[g];
            bad |= !isfinite(v);
            s_nxt[g] = v;
        }
    }
    if (bad) s_bad = 1;
    if (!obs_normalize) {
        __syncthreads();
        if (tid == 0 && s_bad) *nonfinite = 1;
        return;
    }
    const bool last = ext_tile_moments<false, false>(part, obs, sM, nullptr, nullptr, O, env0, rows, true, ns.ticket);
    if (tid == 0 && s_bad) *nonfinite = 1;
    if (last) ext_fold_push<false, false>(part, ns, O, N, true);
}

// Evaluation of a saved policy on a user env (Evaluator.evaluate with a registered env), the observe half of step t after
// env.step; is_reset: the ingest of env.reset()'s observations (before step t + 1; t = -1 for the first reset).  Per env
// still running (left > 0), one thread each: the fp64 episode sums, the EarlyTerminated rule, the Saute state, the
// episode end and the results, as eval_step does for the synthetic env.  The next observations go to the state buffer
// step t + 1 reads.  ObsNormalize pushes the final observations of the running envs that report one, then the next
// observations of every running env (reset: the observations of every env with episodes left), through the fp64 push
// (ext_tile_moments / ext_fold_push).  The last CTA
// also advances the done word ctr[0]; ctr[2] counts the envs to reset now (N == 1: every episode end with episodes left),
// and a reset ingest clears it.  RST: rst[env] (one byte per env, written on every launch) is 1 where the cost rule ended
// a running env's episode that the env itself did not end, and the env has episodes left: the envs the caller resets
// through reset_envs(mask) before ext_reset_rows_kernel ingests their rows.
//
// WRAP (with RST): an env that declares the TimeLimit / AutoReset wrappers, which the evaluation never auto-resets
// (evaluator.py: TimeLimit(time_limit) only, the loop resets).  tl_steps[env] is TimeLimit's _time, cleared at each
// episode end; with tl_limit > 0 a step truncates at tl_steps >= tl_limit instead of by the env's flag.  rst[env] is 1
// for every episode end with episodes left, and the launcher passes no final rows: a step's rows are the env's own.
template <bool RST, bool WRAP = false>
__device__ __forceinline__ void ext_eval_observe_step(ExtObs x, EnvState st, NormState ns, SauteSpec sa, EvalSpec ev,
                                                      int O, int N, int t, int obs_normalize, int is_reset,
                                                      uint8_t* rst_out, int* tl_steps = nullptr, int tl_limit = 0) {
    __shared__ int sRun[XT], sFin[XT];
    __shared__ int s_bad;
    const int tid = threadIdx.x, env0 = blockIdx.x * XT, rows = min(XT, N - env0);
    if (tid == 0) s_bad = 0;
    if (tid < XT) {
        const int env = env0 + tid;
        int run = 0, fin = 0, nxt = 0, rst = 0, cut = 0;
        if (tid < rows && ev.left[env] > 0) {
            run = 1;
            if (!is_reset) {
                fin = (x.final_obs && x.final_mask && x.final_mask[env]) ? 1 : 0;
                const float rew = x.rew[env], cst = x.cost[env];
                const int len = ev.len[env];
                const double r64 = ev.ret[env] + (double)rew;
                const double c64 = ev.cost[env] + pow(ev.crit, (double)len) * (double)cst;
                bool env_done;
                if constexpr (WRAP) {
                    const int k = tl_steps[env] + 1;
                    env_done = x.term[env] != 0 || (tl_limit > 0 ? k >= tl_limit : x.trunc[env] != 0);
                    tl_steps[env] = k;
                } else {
                    env_done = x.term[env] != 0 || x.trunc[env] != 0;
                }
                const bool done = env_done || (ev.early && c64 >= ev.cost_limit);
                if (sa.safety) saute_step(sa, t, N, env, rew, cst, done);
                const int left = ev.left[env];
                if constexpr (WRAP) {
                    cut = (done && left > 1) ? 1 : 0;
                    if (done) tl_steps[env] = 0;
                } else if constexpr (RST) {
                    cut = (done && !env_done && left > 1) ? 1 : 0;
                }
                if (done) {
                    const int k = ev.done_eps[env];
                    const size_t out = (size_t)env + (size_t)k * N;
                    ev.out_ret[out] = r64; ev.out_cost[out] = c64; ev.out_len[out] = len + 1;
                    ev.done_eps[env] = k + 1;
                    ev.left[env] = left - 1;
                    ev.ret[env] = 0.0; ev.cost[env] = 0.0; ev.len[env] = 0;
                } else {
                    ev.ret[env] = r64; ev.cost[env] = c64; ev.len[env] = len + 1;
                }
                nxt = (!done || left > 1) ? 1 : 0;
                rst = (done && left > 1 && ev.explicit_reset) ? 1 : 0;
            }
        }
        sRun[tid] = run; sFin[tid] = fin;
        if constexpr (RST) {
            if (tid < rows) rst_out[env] = (uint8_t)cut;
        }
        if (!is_reset) {
            if (nxt) atomicAdd(ev.ctr + 1, 1);
            if (rst) atomicAdd(ev.ctr + 2, 1);
        }
    }
    __syncthreads();
    float* s_nxt = st.s_raw + (size_t)((t + 1) & 1) * N * O;
    bool bad = false;
    for (int i = tid; i < rows * O; i += NTHREADS) {
        const size_t g = (size_t)env0 * O + i;
        const float v = x.next_obs[g];
        bad |= sRun[i / O] && !isfinite(v);
        s_nxt[g] = v;
        if (sFin[i / O]) bad |= !isfinite(x.final_obs[g]);
    }
    if (bad) s_bad = 1;
    // set A: the running rows; set B: their final rows.  Without obs_normalize only the row counts go to count[0].
    const bool last = ext_tile_moments<false, true>(x.part, x.next_obs, sRun, x.final_obs, sFin, O, env0, rows,
                                                    obs_normalize, ns.ticket);
    if (tid == 0 && s_bad) *x.nonfinite = 1;
    if (!last) return;
    ext_fold_push<false, true>(x.part, ns, O, N, obs_normalize);
    if (tid == 0) {
        if (is_reset) {
            ev.ctr[2] = 0;
        } else {
            ev.ctr[0] = __ldcg(ev.ctr + 1);
            ev.ctr[1] = 0;
        }
    }
}

__global__ void __launch_bounds__(NTHREADS) ext_eval_observe_kernel(ExtObs x, EnvState st, NormState ns, SauteSpec sa,
                                                                    EvalSpec ev, int O, int N, int t, int obs_normalize,
                                                                    int is_reset) {
    ext_eval_observe_step<false>(x, st, ns, sa, ev, O, N, t, obs_normalize, is_reset, nullptr);
}

__global__ void __launch_bounds__(NTHREADS) ext_eval_observe_rst_kernel(ExtObs x, EnvState st, NormState ns,
                                                                        SauteSpec sa, EvalSpec ev, int O, int N, int t,
                                                                        int obs_normalize, uint8_t* rst) {
    ext_eval_observe_step<true>(x, st, ns, sa, ev, O, N, t, obs_normalize, 0, rst);
}

__global__ void __launch_bounds__(NTHREADS) ext_eval_observe_wrapped_kernel(ExtObs x, EnvState st, NormState ns,
                                                                            SauteSpec sa, EvalSpec ev, int O, int N,
                                                                            int t, int obs_normalize, uint8_t* rst,
                                                                            int* tl_steps, int tl_limit) {
    ext_eval_observe_step<true, true>(x, st, ns, sa, ev, O, N, t, obs_normalize, 0, rst, tl_steps, tl_limit);
}

// Window of the last <= W finished episodes in (step, env) append order: Logger deque semantics
// (common/logger.py:L253-282 with window_lens; adapter/onpolicy_adapter.py:L159-175).
// ring[3][W] holds (EpRet, EpCost, EpLen); meta[0] = number of valid entries, meta[1] = head.
// Single CTA of 1024 threads: find the first row (from the end) after which >= W episodes finished,
// then append rows in order with a block-wide ordered compaction (exclusive scan of counts).
__global__ void __launch_bounds__(1024) episode_window_kernel(const uint8_t* __restrict__ flags,
                                                              const float* __restrict__ epfin,
                                                              int T, int N, int W,
                                                              float* __restrict__ ring,
                                                              int* __restrict__ meta) {
    __shared__ int s_cnt, s_total, s_warp[32], s_base;
    const size_t TN = (size_t)T * N;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int seg = (N + 1023) / 1024;          // contiguous envs per thread
    const int lo = min(N, tid * seg), hi = min(N, lo + seg);
    if (tid == 0) s_total = 0;
    int first_row = T;
    for (int t = T - 1; t >= 0; --t) {
        if (tid == 0) s_cnt = 0;
        __syncthreads();
        int cnt = 0;
        for (int i = lo; i < hi; ++i) cnt += flags[(size_t)t * N + i] != 0;
        if (cnt) atomicAdd(&s_cnt, cnt);
        __syncthreads();
        first_row = t;
        if (tid == 0) s_total += s_cnt;
        __syncthreads();
        if (s_total >= W) break;
    }
    __syncthreads();
    const int total_new = s_total;
    if (total_new == 0) return;
    const int head0 = meta[1], count0 = meta[0];
    const int skip = total_new > W ? total_new - W : 0;   // only the last W appended entries survive
    if (tid == 0) s_base = 0;
    __syncthreads();
    for (int t = first_row; t < T; ++t) {
        int cnt = 0;
        for (int i = lo; i < hi; ++i) cnt += flags[(size_t)t * N + i] != 0;
        // block exclusive scan of cnt
        int incl = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        if (lane == 31) s_warp[wid] = incl;
        __syncthreads();
        if (wid == 0) {
            int w = s_warp[lane], wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, wi, o);
                if (lane >= o) wi += v;
            }
            s_warp[lane] = wi - w;   // exclusive warp offsets
            if (lane == 31) s_cnt = wi;  // row total
        }
        __syncthreads();
        int seq = s_base + s_warp[wid] + incl - cnt;   // sequence index of my first entry
        for (int i = lo; i < hi; ++i) {
            const size_t idx = (size_t)t * N + i;
            if (flags[idx] != 0) {
                if (seq >= skip) {
                    const int pos = (head0 + (seq - skip)) % W;
                    ring[0 * W + pos] = epfin[idx];
                    ring[1 * W + pos] = epfin[TN + idx];
                    ring[2 * W + pos] = epfin[2 * TN + idx];
                }
                ++seq;
            }
        }
        __syncthreads();
        if (tid == 0) s_base += s_cnt;
        __syncthreads();
    }
    if (tid == 0) {
        const int kept = total_new - skip;
        meta[1] = (head0 + kept) % W;
        meta[0] = min(W, count0 + kept);
    }
}

// window_sums[4] = {sum EpRet, sum EpCost, sum EpLen, count} over the ring (fp64).
__global__ void window_sums_kernel(const float* __restrict__ ring, const int* __restrict__ meta,
                                   int W, double* __restrict__ window_sums) {
    if (threadIdx.x != 0) return;
    const int count = meta[0];
    double s[3] = {0, 0, 0};
    for (int q = 0; q < 3; ++q)
        for (int i = 0; i < count; ++i) s[q] += (double)ring[q * W + i];
    window_sums[0] = s[0]; window_sums[1] = s[1]; window_sums[2] = s[2];
    window_sums[3] = (double)count;
}

}  // namespace osb

using namespace osb;

static SauteSpec g_saute = {nullptr, 1.f, 1.f, 0.f, 1.f};
static EarlySpec g_early = {nullptr, 0.f};

static size_t rollout_smem_bytes(int O) {   // O = network input width
    size_t f = NETSMEM_FLOATS_FWD + 3 * RT * LD + RT * LDO + 2 * (size_t)O + RT * OUTP +
               2 * RT * (KC + 1) + 3 * RT;
    return f * sizeof(float);
}

static int launch_env_reset(const EnvSpec& es, const EnvState& st, const NormState& ns, int N, cudaStream_t stream) {
    env_reset_kernel<<<(N + RT - 1) / RT, NTHREADS, 0, stream>>>(es, st, ns, g_saute, N);
    OSB_LAUNCH_CHECK();
    return OSB_OK;
}

extern "C" {

// Opaque-struct-free C ABI: the caller passes plain device pointers.
int osb_env_reset(int O, int A, int max_episode_steps, unsigned seed, unsigned term_threshold,
                  unsigned env_id_offset, float cost_threshold, int obs_normalize, int N,
                  float* s_raw, float* final_raw, int* ep_step, unsigned* episode, unsigned* gstep,
                  float* ep_ret, float* ep_cost, int* ep_len, const float* bias,
                  float* norm_mean, float* norm_sumsq, float* norm_std, float* norm_mean1,
                  float* norm_std1, long long* norm_count, long long* acc_all, long long* acc_fin,
                  int* fin_count, int* had_fin, unsigned* ticket, void* stream) {
    OSB_CHECK_ARG(O > 0 && A > 0 && A <= OUTP && N > 0, "bad dims (need 0 < A <= 16)");
    EnvSpec es{O, A, max_episode_steps, seed, term_threshold, env_id_offset, cost_threshold, obs_normalize};
    EnvState st{s_raw, final_raw, ep_step, episode, gstep, ep_ret, ep_cost, ep_len, bias};
    NormState ns{norm_mean, norm_sumsq, norm_std, norm_mean1, norm_std1, norm_count, acc_all,
                 acc_fin, fin_count, had_fin, ticket};
    return launch_env_reset(es, st, ns, N, (cudaStream_t)stream);
}

static long long* g_rollout_dbg = nullptr;

}  // extern "C"

// StepArgs of the synthetic env's step and epoch entries, which share this argument list
static StepArgs synthetic_step_args(int O, int A, int max_episode_steps, unsigned seed, unsigned term_threshold,
                                    unsigned env_id_offset, float cost_threshold, int obs_normalize, int N, int T,
                                    float* s_raw, float* final_raw, int* ep_step, unsigned* episode, unsigned* gstep,
                                    float* ep_ret, float* ep_cost, int* ep_len, const float* bias, float* norm_mean,
                                    float* norm_sumsq, float* norm_std, float* norm_mean1, float* norm_std1,
                                    long long* norm_count, long long* acc_all, long long* acc_fin, int* fin_count,
                                    int* had_fin, unsigned* ticket, float* obs, float* act, float* logp, float* rew,
                                    float* cost, float* val_r, float* val_c, float* boot_r, float* boot_c,
                                    unsigned char* flags, float* epfin, const float* theta, unsigned noise_seed,
                                    int precision) {
    StepArgs p{};
    p.es = EnvSpec{O, A, max_episode_steps, seed, term_threshold, env_id_offset, cost_threshold, obs_normalize};
    p.st = EnvState{s_raw, final_raw, ep_step, episode, gstep, ep_ret, ep_cost, ep_len, bias};
    p.ns = NormState{norm_mean, norm_sumsq, norm_std, norm_mean1, norm_std1, norm_count, acc_all,
                     acc_fin, fin_count, had_fin, ticket};
    p.sl = Slabs{obs, act, logp, rew, cost, val_r, val_c, boot_r, boot_c, flags, epfin};
    p.sa = g_saute; p.et = g_early;
    p.theta = theta; p.noise_seed = noise_seed; p.T = T; p.N = N; p.precision = precision;
    return p;
}

// The one-time host actions of an act launch on an external env -- kernel attributes and the accumulator image -- call
// cudaFuncSetAttribute / cudaMalloc, which CUDA-graph capture does not allow.  osb_ext_prepare performs them before a
// capture; a launch on a capturing stream that would still need one fails here instead of breaking the capture.
static int ext_refuse_if_capturing(cudaStream_t stream, const char* what) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    OSB_CUDA(cudaStreamIsCapturing(stream, &cs));
    if (cs == cudaStreamCaptureStatusNone) return OSB_OK;
    char msg[256];
    snprintf(msg, sizeof(msg), "osb_ext_act / osb_eval_ext_act on a capturing stream needs %s: call osb_ext_prepare / "
             "osb_eval_ext_prepare before the capture", what);
    osb_set_error(msg);
    return OSB_ERR_UNSUPPORTED;
}

// CTAs of the persistent training kernel: ceil(N / RTA) actor tiles, then ceil(N / RTC) tiles per critic
static int ring_grid(int N) { return (N + RTA - 1) / RTA + 2 * ((N + RTC - 1) / RTC); }
// one [128][TC_COLS] image per CTA, enough for every grid (ring_grid(N) >= 3 ceil(N / RTC))
static size_t rollout_tc_acc_bytes(int N) { return (size_t)ring_grid(N) * 128 * TC_COLS * sizeof(float); }

static int sm_count() {
    static int n_sm = 0;
    if (!n_sm) { int dev = 0; OSB_CUDA(cudaGetDevice(&dev)); OSB_CUDA(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev)); }
    return n_sm;
}

// tf32 / bf16x3 with a network input of <= 64 columns run on the tensor-core tiles, everything else on the fp32 tiles
static bool tc_tiles(const StepArgs& p) {
    return (p.precision == 1 || p.precision == 2) && p.es.O + (p.sa.safety ? 1 : 0) <= 64;
}
// the persistent kernels need every CTA resident: training ring_grid(N), evaluation one actor CTA per RTC envs
static bool persistent_fits(const StepArgs& p, bool eval) {
    return tc_tiles(p) && (eval ? (p.N + RTC - 1) / RTC : ring_grid(p.N)) <= sm_count();
}

// the persistent kernels' grid-barrier arrival counter and release flag (64 bytes), then the training kernel's ring of
// normaliser sums (3 RING_SLOTs)
static unsigned int* g_grid_bar = nullptr;
constexpr size_t GRID_BAR_BYTES = 64 + 3 * RING_SLOT * sizeof(long long);

// One launch of the step kernels: a training step (EVAL = false: grid = env tiles x the actor and both critics, the
// epoch-end tail only the critics) or an evaluation step (grid = env tiles x the actor); on the synthetic env or, EXT,
// the act half of a step on a user env.  persistent (synthetic env, persistent_fits): ONE cooperative launch runs every
// step.  prepare_only: perform the host actions (attributes, accumulator image) and launch nothing (osb_ext_prepare).
template <bool EXT, bool EVAL>
static int launch_rollout(StepArgs& p, cudaStream_t stream, bool persistent = false, bool prepare_only = false) {
    const int nets = EVAL ? 1 : (p.is_tail ? 2 : 3);
    const NetSpec spec = net_spec();
    // the evaluation steps run the actor alone; the tail step only the critics
    const int act = EVAL ? spec.act[0] : launch_act(spec, p.is_tail ? 6 : 7);
    return with_act<!EVAL>(act, [&](auto a) {
        if (tc_tiles(p)) {
            const bool x3 = p.precision == 2;
            const size_t smem_tc = rollout_tc_smem_bytes(x3, persistent && !EVAL);
            static bool attr_tc = false;
            if (!attr_tc) {
                if constexpr (EXT) {
                    if (int rc = ext_refuse_if_capturing(stream, "the tensor-core kernel attributes")) return rc;
                }
                // {tf32, bf16x3} x {one step, persistent}; EXT launches only the one-step pair
                const void* kernels[] = {(const void*)rollout_step_tc_kernel<false, false, EXT, EVAL, a.value>,
                                         (const void*)rollout_step_tc_kernel<true, false, EXT, EVAL, a.value>,
                                         (const void*)rollout_step_tc_kernel<false, true, false, EVAL, a.value>,
                                         (const void*)rollout_step_tc_kernel<true, true, false, EVAL, a.value>};
                for (int i = 0; i < (EXT ? 2 : 4); ++i)
                    OSB_CUDA(cudaFuncSetAttribute(kernels[i], cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                  (int)rollout_tc_smem_bytes(i & 1, i >= 2 && !EVAL)));
                attr_tc = true;
            }
            if constexpr (EXT) {
                if (acc_scratch_capacity(ACC_ROLLOUT) < rollout_tc_acc_bytes(p.N))
                    if (int rc = ext_refuse_if_capturing(stream, "a larger accumulator image")) return rc;
            }
            p.acc = acc_scratch(ACC_ROLLOUT, rollout_tc_acc_bytes(p.N));
            if (!p.acc) return OSB_ERR_CUDA;
            if (prepare_only) return OSB_OK;
            const dim3 grid_tc = (persistent && !EVAL) ? dim3(ring_grid(p.N)) : dim3((p.N + RTC - 1) / RTC, nets);
            if (persistent) {
                // every CTA resident: the step barrier is a software grid barrier
                if (!g_grid_bar) OSB_CUDA(cudaMalloc(&g_grid_bar, GRID_BAR_BYTES));
                p.bar_ctr = g_grid_bar; p.bar_flag = g_grid_bar + 1;
                p.ring = reinterpret_cast<long long*>(g_grid_bar + 16);
                OSB_CUDA(cudaMemsetAsync(p.bar_ctr, 0, EVAL ? 2 * sizeof(unsigned int) : GRID_BAR_BYTES, stream));
                NetSpec sp = spec;
                void* args[] = {&p, &sp};
                osb_count_launch();
                OSB_CUDA(cudaLaunchCooperativeKernel(x3 ? (void*)rollout_step_tc_kernel<true, true, false, EVAL, a.value>
                                                        : (void*)rollout_step_tc_kernel<false, true, false, EVAL, a.value>,
                                                     grid_tc, dim3(NTHREADS), args, smem_tc, stream));
                return OSB_OK;
            }
            if (x3) rollout_step_tc_kernel<true, false, EXT, EVAL, a.value><<<grid_tc, NTHREADS, smem_tc, stream>>>(p, spec);
            else rollout_step_tc_kernel<false, false, EXT, EVAL, a.value><<<grid_tc, NTHREADS, smem_tc, stream>>>(p, spec);
            OSB_LAUNCH_CHECK();
            return OSB_OK;
        }
        const int On = p.es.O + (p.sa.safety ? 1 : 0);
        const size_t smem = rollout_smem_bytes(On);
        static size_t attr = 0;
        if (smem > attr) {
            if constexpr (EXT) {
                if (int rc = ext_refuse_if_capturing(stream, "a larger shared-memory attribute")) return rc;
            }
            OSB_CUDA(cudaFuncSetAttribute(rollout_step_kernel<EXT, EVAL, a.value>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            attr = smem;
        }
        if (prepare_only) return OSB_OK;
        rollout_step_kernel<EXT, EVAL, a.value><<<dim3((p.N + RT - 1) / RT, nets), NTHREADS, smem, stream>>>(p, spec);
        OSB_LAUNCH_CHECK();
        return OSB_OK;
    });
}

extern "C" {

// Saute / Simmer mode of the following osb_env_reset / osb_rollout_* calls (process-wide until changed): safety = [2][N]
// device floats (the safety state z by step parity), or NULL for the plain OnPolicyAdapter semantics.  The networks then
// take O + 1 inputs ([normalised obs | z]) and the obs slab rows are O + 1 wide.  saute_adapter.py:L135-217.
int osb_rollout_set_saute(float* safety, float safety_budget, float saute_gamma, float unsafe_reward, float safety_init) {
    OSB_CHECK_ARG(safety == nullptr || (safety_budget > 0.f && saute_gamma > 0.f), "safety_budget and saute_gamma must be positive");
    g_saute = SauteSpec{safety, safety_budget, saute_gamma, unsafe_reward, safety_init};
    return OSB_OK;
}

// EarlyTerminated mode of the following osb_rollout_* calls (process-wide until changed): cost_acc = [N] device floats
// (per-env accumulated cost, persistent across episodes and epochs) or NULL.  early_terminated_adapter.py:L56-98.
int osb_rollout_set_early_termination(float* cost_acc, float cost_limit) {
    g_early = EarlySpec{cost_acc, cost_limit};
    return OSB_OK;
}

// development aid: clock64 stamps of the persistent rollout kernel go to buf (1024 long long), NULL turns it off
int osb_rollout_debug_buffer(long long* buf) { g_rollout_dbg = buf; return OSB_OK; }

int osb_rollout_step(int O, int A, int max_episode_steps, unsigned seed, unsigned term_threshold,
                     unsigned env_id_offset, float cost_threshold, int obs_normalize, int N, int T,
                     int t, float* s_raw, float* final_raw, int* ep_step, unsigned* episode,
                     unsigned* gstep, float* ep_ret, float* ep_cost, int* ep_len, const float* bias,
                     float* norm_mean, float* norm_sumsq, float* norm_std, float* norm_mean1,
                     float* norm_std1, long long* norm_count, long long* acc_all,
                     long long* acc_fin, int* fin_count, int* had_fin, unsigned* ticket,
                     float* obs, float* act, float* logp, float* rew, float* cost, float* val_r,
                     float* val_c, float* boot_r, float* boot_c, unsigned char* flags, float* epfin,
                     const float* theta, const float* eps, unsigned noise_seed,
                     unsigned global_step, int precision, void* stream) {
    OSB_CHECK_ARG(O > 0 && A > 0 && A <= OUTP && N > 0 && T > 0, "bad dims (need 0 < A <= 16)");
    OSB_CHECK_ARG(t >= 0 && t <= T, "step index out of range");
    StepArgs p = synthetic_step_args(O, A, max_episode_steps, seed, term_threshold, env_id_offset, cost_threshold,
                                     obs_normalize, N, T, s_raw, final_raw, ep_step, episode, gstep, ep_ret, ep_cost,
                                     ep_len, bias, norm_mean, norm_sumsq, norm_std, norm_mean1, norm_std1, norm_count,
                                     acc_all, acc_fin, fin_count, had_fin, ticket, obs, act, logp, rew, cost, val_r,
                                     val_c, boot_r, boot_c, flags, epfin, theta, noise_seed, precision);
    p.eps = eps; p.global_step = global_step;
    p.t = t; p.is_tail = (t == T) ? 1 : 0;
    return launch_rollout<false, false>(p, (cudaStream_t)stream);
}

int osb_rollout_epoch(int O, int A, int max_episode_steps, unsigned seed, unsigned term_threshold,
                      unsigned env_id_offset, float cost_threshold, int obs_normalize, int N, int T,
                      float* s_raw, float* final_raw, int* ep_step, unsigned* episode,
                      unsigned* gstep, float* ep_ret, float* ep_cost, int* ep_len, const float* bias,
                      float* norm_mean, float* norm_sumsq, float* norm_std, float* norm_mean1,
                      float* norm_std1, long long* norm_count, long long* acc_all,
                      long long* acc_fin, int* fin_count, int* had_fin, unsigned* ticket,
                      float* obs, float* act, float* logp, float* rew, float* cost, float* val_r,
                      float* val_c, float* boot_r, float* boot_c, unsigned char* flags, float* epfin,
                      const float* theta, const float* eps_all, unsigned noise_seed,
                      unsigned epoch_index, int W, float* ring, int* meta, double* window_sums,
                      int precision, void* stream) {
    OSB_CHECK_ARG(O > 0 && A > 0 && A <= OUTP && N > 0 && T > 0, "bad dims (need 0 < A <= 16)");
    cudaStream_t s = (cudaStream_t)stream;
    StepArgs p = synthetic_step_args(O, A, max_episode_steps, seed, term_threshold, env_id_offset, cost_threshold,
                                     obs_normalize, N, T, s_raw, final_raw, ep_step, episode, gstep, ep_ret, ep_cost,
                                     ep_len, bias, norm_mean, norm_sumsq, norm_std, norm_mean1, norm_std1, norm_count,
                                     acc_all, acc_fin, fin_count, had_fin, ticket, obs, act, logp, rew, cost, val_r,
                                     val_c, boot_r, boot_c, flags, epfin, theta, noise_seed, precision);
    int rc = launch_env_reset(p.es, p.st, p.ns, N, s);
    if (rc) return rc;
    p.dbg = g_rollout_dbg;
    // tensor-core modes with every CTA resident: one persistent launch per epoch.  OSB_ROLLOUT_PER_STEP=1 keeps one
    // launch per step, the persistent kernel's reference.
    if (persistent_fits(p, false) && !getenv("OSB_ROLLOUT_PER_STEP")) {
        p.t = 0; p.is_tail = 0; p.eps = eps_all; p.global_step = epoch_index * (unsigned)T;
        rc = launch_rollout<false, false>(p, s, true);
        if (rc) return rc;
        return osb_episode_window(flags, epfin, T, N, W, ring, meta, window_sums, stream);
    }
    for (int t = 0; t <= T; ++t) {
        p.t = t; p.is_tail = (t == T) ? 1 : 0;
        p.eps = (eps_all && t < T) ? eps_all + (size_t)t * N * A : nullptr;
        p.global_step = epoch_index * (unsigned)T + (unsigned)t;
        rc = launch_rollout<false, false>(p, s);
        if (rc) return rc;
    }
    return osb_episode_window(flags, epfin, T, N, W, ring, meta, window_sums, stream);
}

int osb_episode_window(const unsigned char* flags, const float* epfin, int T, int N, int W,
                       float* ring, int* meta, double* window_sums, void* stream) {
    OSB_CHECK_ARG(flags && epfin && ring && meta && window_sums && W > 0, "bad argument");
    cudaStream_t s = (cudaStream_t)stream;
    episode_window_kernel<<<1, 1024, 0, s>>>(flags, epfin, T, N, W, ring, meta);
    OSB_LAUNCH_CHECK();
    window_sums_kernel<<<1, 32, 0, s>>>(ring, meta, W, window_sums);
    OSB_LAUNCH_CHECK();
    return OSB_OK;
}

}  // extern "C"

static StepArgs ext_step_args(int O, int A, int obs_normalize, int N, int precision);

extern "C" {

int osb_eval_synthetic(int O, int A, int max_episode_steps, unsigned seed, unsigned term_threshold, float cost_threshold,
                       int obs_normalize, int N, int num_episodes, float* s_raw, float* final_raw, int* ep_step,
                       unsigned* episode, unsigned* gstep, float* ep_ret, float* ep_cost, int* ep_len, const float* bias,
                       float* norm_mean, float* norm_sumsq, float* norm_std, float* norm_mean1, float* norm_std1,
                       long long* norm_count, long long* acc_all, long long* acc_fin, int* fin_count, int* had_fin,
                       unsigned* ticket, float* safety, float safety_budget, float saute_gamma, int early,
                       double cost_limit, double cost_criteria, int* left, int* done_eps, double* ret, double* cost,
                       int* len, long long* acc_rst, int* ctr, double* out_ret, double* out_cost, int* out_len,
                       float* act_out, const float* theta, int precision, int per_step, void* stream) {
    OSB_CHECK_ARG(O > 0 && A > 0 && A <= OUTP && N > 0 && num_episodes >= N && max_episode_steps > 0,
                  "bad dims (need 0 < A <= 16, 0 < N <= num_episodes, max_episode_steps > 0)");
    OSB_CHECK_ARG(precision >= 0 && precision <= 2, "precision must be 0, 1 or 2");
    OSB_CHECK_ARG(safety == nullptr || (safety_budget > 0.f && saute_gamma > 0.f), "safety_budget and saute_gamma must be positive");
    OSB_CHECK_ARG(left && done_eps && ret && cost && len && acc_rst && ctr && out_ret && out_cost && out_len && theta,
                  "bad argument");
    cudaStream_t s = (cudaStream_t)stream;
    // every episode ends by its time limit, so no env runs more than this many steps
    const long long steps = (long long)((num_episodes + N - 1) / N) * max_episode_steps;
    OSB_CHECK_ARG(steps < (1ll << 30), "too many steps per env");
    StepArgs p = synthetic_step_args(O, A, max_episode_steps, seed, term_threshold, 0u, cost_threshold, obs_normalize,
                                     N, (int)steps, s_raw, final_raw, ep_step, episode, gstep, ep_ret, ep_cost, ep_len,
                                     bias, norm_mean, norm_sumsq, norm_std, norm_mean1, norm_std1, norm_count, acc_all,
                                     acc_fin, fin_count, had_fin, ticket, nullptr, nullptr, nullptr, nullptr, nullptr,
                                     nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, theta, 0u, precision);
    // the safety state z starts every episode at 1, Saute and Simmer alike; the reward is never replaced
    p.sa = SauteSpec{safety, safety ? safety_budget : 1.f, safety ? saute_gamma : 1.f, 0.f, 1.f};
    p.et = EarlySpec{nullptr, 0.f};
    p.ev = EvalSpec{left, done_eps, ret, cost, len, out_ret, out_cost, out_len, acc_rst, ctr, cost_criteria, cost_limit,
                    early, N == 1 ? 1 : 0, act_out};
    // every env's first episode starts from a reset, its observations pushed as one batch (a vector env's reset)
    env_reset_kernel<<<(N + RT - 1) / RT, NTHREADS, 0, s>>>(p.es, p.st, p.ns, p.sa, N);
    OSB_LAUNCH_CHECK();
    if (!per_step && persistent_fits(p, true)) {   // p.T bounds the persistent kernel's steps
        p.t = 0;
        return launch_rollout<false, true>(p, s, true);
    }
    static int* h_done = nullptr;
    if (!h_done) OSB_CUDA(cudaMallocHost(&h_done, sizeof(int)));
    constexpr int CHECK_EVERY = 16;     // the done word is read after every 16 launches; later launches return at once
    for (long long t = 0; t < steps; ++t) {
        p.t = (int)(t & 1);     // the parity of the state buffers (T = the step bound keeps every launch a full step)
        if (int rc = launch_rollout<false, true>(p, s)) return rc;
        if ((t + 1) % CHECK_EVERY == 0 && t + 1 < steps) {
            OSB_CUDA(cudaMemcpyAsync(h_done, ctr, sizeof(int), cudaMemcpyDeviceToHost, s));
            OSB_CUDA(cudaStreamSynchronize(s));
            if (*h_done == 0) break;
        }
    }
    return OSB_OK;
}

// the workspace of the fp64 ObsNormalize push (ext_tile_moments): the training and evaluation observe launches and the
// reset rows of either take the same
int osb_ext_workspace_doubles(int O, int N) { return ((N + XT - 1) / XT) * (4 * O + 2); }
int osb_eval_ext_workspace_doubles(int O, int N) { return osb_ext_workspace_doubles(O, N); }

int osb_eval_ext_act(int O, int A, int obs_normalize, int N, int t, const float* s_raw, const float* norm_mean,
                     const float* norm_std, const long long* norm_count, const float* safety, const float* theta,
                     const float* act_lo, const float* act_hi, float* act_env, const int* left, const int* ctr,
                     float* act_out, int precision, void* stream) {
    OSB_CHECK_ARG(O > 0 && A > 0 && A <= OUTP && N > 0 && t >= 0, "bad dims (need 0 < A <= 16) / step index");
    OSB_CHECK_ARG(precision >= 0 && precision <= 2, "precision must be 0, 1 or 2");
    OSB_CHECK_ARG(s_raw && norm_mean && norm_std && norm_count && theta && act_lo && act_hi && act_env && left && ctr,
                  "bad argument");
    StepArgs p = ext_step_args(O, A, obs_normalize, N, precision);
    p.st.s_raw = const_cast<float*>(s_raw);
    p.ns.mean = const_cast<float*>(norm_mean); p.ns.std = const_cast<float*>(norm_std);
    p.ns.count = const_cast<long long*>(norm_count);
    p.sa.safety = const_cast<float*>(safety);
    p.theta = theta; p.t = t & 1; p.T = 2;
    p.act_lo = act_lo; p.act_hi = act_hi; p.act_env = act_env;
    p.ev.left = const_cast<int*>(left); p.ev.ctr = const_cast<int*>(ctr); p.ev.act_out = act_out;
    return launch_rollout<true, true>(p, (cudaStream_t)stream);
}

// osb_eval_ext_observe, and with rst osb_eval_ext_observe_rst
static int eval_ext_observe(int O, int N, int t, int obs_normalize, int is_reset, const float* next_obs, const float* rew,
                            const float* cost, const unsigned char* terminated, const unsigned char* truncated,
                            const float* final_obs, const unsigned char* final_mask, float* s_raw, float* norm_mean,
                            float* norm_sumsq, float* norm_std, long long* norm_count, unsigned* ticket, float* safety,
                            float safety_budget, float saute_gamma, int early, double cost_limit, double cost_criteria,
                            int* left, int* done_eps, double* ret, double* cost_acc, int* len, int* ctr,
                            double* out_ret, double* out_cost, int* out_len, double* workspace, int* nonfinite,
                            unsigned char* rst, int* tl_steps, int tl_limit, void* stream) {
    OSB_CHECK_ARG(O > 0 && N > 0 && t >= -1, "bad dims / step index");
    OSB_CHECK_ARG(next_obs && s_raw && norm_mean && norm_sumsq && norm_std && norm_count && ticket && left && ctr &&
                  workspace && nonfinite, "bad argument");
    OSB_CHECK_ARG(is_reset || (rew && cost && terminated && truncated && done_eps && ret && cost_acc && len && out_ret &&
                               out_cost && out_len), "bad argument");
    OSB_CHECK_ARG(safety == nullptr || (safety_budget > 0.f && saute_gamma > 0.f), "safety_budget and saute_gamma must be positive");
    ExtObs x{next_obs, rew, cost, terminated, truncated, final_obs, final_mask, workspace, nonfinite};
    EnvState st{s_raw, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    NormState ns{norm_mean, norm_sumsq, norm_std, nullptr, nullptr, norm_count, nullptr, nullptr, nullptr, nullptr, ticket};
    SauteSpec sa{safety, safety ? safety_budget : 1.f, safety ? saute_gamma : 1.f, 0.f, 1.f};
    EvalSpec ev{left, done_eps, ret, cost_acc, len, out_ret, out_cost, out_len, nullptr, ctr, cost_criteria, cost_limit,
                early, N == 1 ? 1 : 0, nullptr};
    const int grid = (N + XT - 1) / XT;
    if (tl_steps)
        ext_eval_observe_wrapped_kernel<<<grid, NTHREADS, 0, (cudaStream_t)stream>>>(x, st, ns, sa, ev, O, N, t,
                                                                                     obs_normalize, rst, tl_steps,
                                                                                     tl_limit);
    else if (rst)
        ext_eval_observe_rst_kernel<<<grid, NTHREADS, 0, (cudaStream_t)stream>>>(x, st, ns, sa, ev, O, N, t,
                                                                                 obs_normalize, rst);
    else
        ext_eval_observe_kernel<<<grid, NTHREADS, 0, (cudaStream_t)stream>>>(x, st, ns, sa, ev, O, N, t, obs_normalize,
                                                                             is_reset);
    OSB_LAUNCH_CHECK();
    return OSB_OK;
}

int osb_eval_ext_observe(int O, int N, int t, int obs_normalize, int is_reset, const float* next_obs, const float* rew,
                         const float* cost, const unsigned char* terminated, const unsigned char* truncated,
                         const float* final_obs, const unsigned char* final_mask, float* s_raw, float* norm_mean,
                         float* norm_sumsq, float* norm_std, long long* norm_count, unsigned* ticket, float* safety,
                         float safety_budget, float saute_gamma, int early, double cost_limit, double cost_criteria,
                         int* left, int* done_eps, double* ret, double* cost_acc, int* len, int* ctr, double* out_ret,
                         double* out_cost, int* out_len, double* workspace, int* nonfinite, void* stream) {
    return eval_ext_observe(O, N, t, obs_normalize, is_reset, next_obs, rew, cost, terminated, truncated, final_obs,
                            final_mask, s_raw, norm_mean, norm_sumsq, norm_std, norm_count, ticket, safety,
                            safety_budget, saute_gamma, early, cost_limit, cost_criteria, left, done_eps, ret, cost_acc,
                            len, ctr, out_ret, out_cost, out_len, workspace, nonfinite, nullptr, nullptr, 0, stream);
}

// osb_eval_ext_observe of a step (no reset ingest) that also writes rst[N], the envs the cost rule cut with episodes left
int osb_eval_ext_observe_rst(int O, int N, int t, int obs_normalize, const float* next_obs, const float* rew,
                             const float* cost, const unsigned char* terminated, const unsigned char* truncated,
                             const float* final_obs, const unsigned char* final_mask, float* s_raw, float* norm_mean,
                             float* norm_sumsq, float* norm_std, long long* norm_count, unsigned* ticket, float* safety,
                             float safety_budget, float saute_gamma, int early, double cost_limit,
                             double cost_criteria, int* left, int* done_eps, double* ret, double* cost_acc, int* len,
                             int* ctr, double* out_ret, double* out_cost, int* out_len, double* workspace,
                             int* nonfinite, unsigned char* rst, void* stream) {
    OSB_CHECK_ARG(t >= 0, "bad dims / step index");
    OSB_CHECK_ARG(rst, "bad argument");
    return eval_ext_observe(O, N, t, obs_normalize, 0, next_obs, rew, cost, terminated, truncated, final_obs,
                            final_mask, s_raw, norm_mean, norm_sumsq, norm_std, norm_count, ticket, safety,
                            safety_budget, saute_gamma, early, cost_limit, cost_criteria, left, done_eps, ret, cost_acc,
                            len, ctr, out_ret, out_cost, out_len, workspace, nonfinite, rst, nullptr, 0, stream);
}

// osb_eval_ext_observe_rst of a step on an env behind TimeLimit / AutoReset: tl_steps[N] is the TimeLimit step counter
// (time_limit > 0) and rst[N] flags every episode end with episodes left; final_obs / final_mask are not read.
int osb_eval_ext_observe_wrapped(int O, int N, int t, int obs_normalize, const float* next_obs, const float* rew,
                                 const float* cost, const unsigned char* terminated, const unsigned char* truncated,
                                 float* s_raw, float* norm_mean, float* norm_sumsq, float* norm_std,
                                 long long* norm_count, unsigned* ticket, float* safety, float safety_budget,
                                 float saute_gamma, int early, double cost_limit, double cost_criteria, int* left,
                                 int* done_eps, double* ret, double* cost_acc, int* len, int* ctr, double* out_ret,
                                 double* out_cost, int* out_len, double* workspace, int* nonfinite, unsigned char* rst,
                                 int* tl_steps, int time_limit, void* stream) {
    OSB_CHECK_ARG(t >= 0 && time_limit >= 0, "bad dims / step index / time limit");
    OSB_CHECK_ARG(rst && tl_steps, "bad argument");
    return eval_ext_observe(O, N, t, obs_normalize, 0, next_obs, rew, cost, terminated, truncated, nullptr, nullptr,
                            s_raw, norm_mean, norm_sumsq, norm_std, norm_count, ticket, safety, safety_budget,
                            saute_gamma, early, cost_limit, cost_criteria, left, done_eps, ret, cost_acc, len, ctr,
                            out_ret, out_cost, out_len, workspace, nonfinite, rst, tl_steps, time_limit, stream);
}

// ---- external envs ---------------------------------------------------------------------------
static int launch_observe(const ExtObs& x, EnvState st, NormState ns, Slabs sl, int O, int N, int T, int t,
                          int obs_normalize, int is_reset, void* stream) {
    ext_observe_kernel<<<(N + XT - 1) / XT, NTHREADS, 0, (cudaStream_t)stream>>>(x, st, ns, sl, O, N, T, t, obs_normalize,
                                                                                 is_reset);
    OSB_LAUNCH_CHECK();
    return OSB_OK;
}

int osb_ext_reset_ingest(int O, int N, int obs_normalize, const float* obs, float* s_raw, float* ep_ret, float* ep_cost,
                         int* ep_len, float* norm_mean, float* norm_sumsq, float* norm_std, float* norm_mean1,
                         float* norm_std1, long long* norm_count, int* had_fin, unsigned* ticket, double* workspace,
                         int* nonfinite, void* stream) {
    OSB_CHECK_ARG(O > 0 && N > 0 && obs && s_raw && ep_ret && ep_cost && ep_len && workspace && nonfinite, "bad argument");
    ExtObs x{obs, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, workspace, nonfinite};
    EnvState st{s_raw, nullptr, nullptr, nullptr, nullptr, ep_ret, ep_cost, ep_len, nullptr};
    NormState ns{norm_mean, norm_sumsq, norm_std, norm_mean1, norm_std1, norm_count, nullptr, nullptr, nullptr, had_fin, ticket};
    Slabs sl{};
    return launch_observe(x, st, ns, sl, O, N, 1, 0, obs_normalize, 1, stream);
}

int osb_ext_observe(int O, int N, int T, int t, int obs_normalize, const float* next_obs, const float* rew,
                    const float* cost, const unsigned char* terminated, const unsigned char* truncated,
                    const float* final_obs, const unsigned char* final_mask, float* s_raw, float* final_raw,
                    float* ep_ret, float* ep_cost, int* ep_len, float* norm_mean, float* norm_sumsq, float* norm_std,
                    float* norm_mean1, float* norm_std1, long long* norm_count, int* had_fin, unsigned* ticket,
                    float* rew_slab, float* cost_slab, unsigned char* flags, float* epfin, double* workspace,
                    int* nonfinite, void* stream) {
    OSB_CHECK_ARG(O > 0 && N > 0 && T > 0 && t >= 0 && t < T, "bad dims / step index");
    OSB_CHECK_ARG(next_obs && rew && cost && terminated && truncated && s_raw && final_raw && rew_slab && cost_slab &&
                  flags && epfin && workspace && nonfinite, "bad argument");
    ExtObs x{next_obs, rew, cost, terminated, truncated, final_obs, final_mask, workspace, nonfinite};
    EnvState st{s_raw, final_raw, nullptr, nullptr, nullptr, ep_ret, ep_cost, ep_len, nullptr};
    NormState ns{norm_mean, norm_sumsq, norm_std, norm_mean1, norm_std1, norm_count, nullptr, nullptr, nullptr, had_fin, ticket};
    Slabs sl{nullptr, nullptr, nullptr, rew_slab, cost_slab, nullptr, nullptr, nullptr, nullptr, flags, epfin};
    return launch_observe(x, st, ns, sl, O, N, T, t, obs_normalize, 0, stream);
}

int osb_ext_observe_early(int O, int N, int T, int t, int obs_normalize, const float* next_obs, const float* rew,
                          const float* cost, const unsigned char* terminated, const unsigned char* truncated,
                          const float* final_obs, const unsigned char* final_mask, float* s_raw, float* final_raw,
                          float* ep_ret, float* ep_cost, int* ep_len, float* norm_mean, float* norm_sumsq,
                          float* norm_std, float* norm_mean1, float* norm_std1, long long* norm_count, int* had_fin,
                          unsigned* ticket, float* rew_slab, float* cost_slab, unsigned char* flags, float* epfin,
                          double* workspace, int* nonfinite, float* cost_acc, float cost_limit, unsigned char* trig,
                          int* trig_total, void* stream) {
    OSB_CHECK_ARG(O > 0 && N > 0 && T > 0 && t >= 0 && t < T, "bad dims / step index");
    OSB_CHECK_ARG(next_obs && rew && cost && terminated && truncated && s_raw && final_raw && rew_slab && cost_slab &&
                  flags && epfin && workspace && nonfinite && cost_acc && trig, "bad argument");
    cudaStream_t s = (cudaStream_t)stream;
    if (trig_total) OSB_CUDA(cudaMemsetAsync(trig_total, 0, sizeof(int), s));
    ExtObs x{next_obs, rew, cost, terminated, truncated, final_obs, final_mask, workspace, nonfinite};
    EnvState st{s_raw, final_raw, nullptr, nullptr, nullptr, ep_ret, ep_cost, ep_len, nullptr};
    NormState ns{norm_mean, norm_sumsq, norm_std, norm_mean1, norm_std1, norm_count, nullptr, nullptr, nullptr, had_fin, ticket};
    Slabs sl{nullptr, nullptr, nullptr, rew_slab, cost_slab, nullptr, nullptr, nullptr, nullptr, flags, epfin};
    ext_observe_early_kernel<<<(N + XT - 1) / XT, NTHREADS, 0, s>>>(x, st, ns, sl, O, N, T, t, obs_normalize,
                                                                    EarlySpec{cost_acc, cost_limit}, trig, trig_total);
    OSB_LAUNCH_CHECK();
    return OSB_OK;
}

int osb_ext_wrapper_step(int N, int time_limit, const unsigned char* terminated, const unsigned char* truncated,
                         int* steps, unsigned char* trunc_out, unsigned char* done, int* done_total, void* stream) {
    OSB_CHECK_ARG(N > 0 && time_limit >= 0, "bad dims / time limit");
    OSB_CHECK_ARG(terminated && truncated && steps && trunc_out && done, "bad argument");
    cudaStream_t s = (cudaStream_t)stream;
    if (done_total) OSB_CUDA(cudaMemsetAsync(done_total, 0, sizeof(int), s));
    ext_wrapper_step_kernel<<<(N + 255) / 256, 256, 0, s>>>(terminated, truncated, steps, trunc_out, done, done_total, N,
                                                            time_limit);
    OSB_LAUNCH_CHECK();
    return OSB_OK;
}

int osb_ext_observe_wrapped(int O, int N, int T, int t, int obs_normalize, const float* step_obs, const float* rew,
                            const float* cost, const unsigned char* terminated, const unsigned char* truncated,
                            const float* reset_obs, const unsigned char* done, float* s_raw, float* final_raw,
                            float* ep_ret, float* ep_cost, int* ep_len, float* norm_mean, float* norm_sumsq,
                            float* norm_std, float* norm_mean1, float* norm_std1, long long* norm_count, int* had_fin,
                            unsigned* ticket, float* rew_slab, float* cost_slab, unsigned char* flags, float* epfin,
                            double* workspace, int* nonfinite, void* stream) {
    OSB_CHECK_ARG(O > 0 && N > 0 && T > 0 && t >= 0 && t < T, "bad dims / step index");
    OSB_CHECK_ARG(step_obs && rew && cost && terminated && truncated && done && s_raw && final_raw && rew_slab &&
                  cost_slab && flags && epfin && workspace && nonfinite, "bad argument");
    // the step's rows are the final rows of the done envs: set B of the push, and final_raw for the bootstraps
    ExtObs x{step_obs, rew, cost, terminated, truncated, step_obs, done, workspace, nonfinite};
    EnvState st{s_raw, final_raw, nullptr, nullptr, nullptr, ep_ret, ep_cost, ep_len, nullptr};
    NormState ns{norm_mean, norm_sumsq, norm_std, norm_mean1, norm_std1, norm_count, nullptr, nullptr, nullptr, had_fin, ticket};
    Slabs sl{nullptr, nullptr, nullptr, rew_slab, cost_slab, nullptr, nullptr, nullptr, nullptr, flags, epfin};
    ext_observe_wrapped_kernel<<<(N + XT - 1) / XT, NTHREADS, 0, (cudaStream_t)stream>>>(x, st, ns, sl, O, N, T, t,
                                                                                         obs_normalize, reset_obs);
    OSB_LAUNCH_CHECK();
    return OSB_OK;
}

int osb_ext_reset_rows(int O, int N, int t, int obs_normalize, const unsigned char* mask, const float* obs, float* s_raw,
                       float* norm_mean, float* norm_sumsq, float* norm_std, long long* norm_count, unsigned* ticket,
                       double* workspace, int* nonfinite, void* stream) {
    OSB_CHECK_ARG(O > 0 && N > 0 && t >= 0, "bad dims / step index");
    OSB_CHECK_ARG(mask && obs && s_raw && norm_mean && norm_sumsq && norm_std && norm_count && ticket && workspace &&
                  nonfinite, "bad argument");
    NormState ns{norm_mean, norm_sumsq, norm_std, nullptr, nullptr, norm_count, nullptr, nullptr, nullptr, nullptr, ticket};
    ext_reset_rows_kernel<<<(N + XT - 1) / XT, NTHREADS, 0, (cudaStream_t)stream>>>(
        obs, mask, s_raw + (size_t)((t + 1) & 1) * N * O, ns, workspace, nonfinite, O, N, obs_normalize);
    OSB_LAUNCH_CHECK();
    return OSB_OK;
}

}  // extern "C"

// StepArgs of the external-env act step: a user env, so no synthetic env, Saute or EarlyTerminated state
static StepArgs ext_step_args(int O, int A, int obs_normalize, int N, int precision) {
    StepArgs p{};
    p.es = EnvSpec{O, A, 0, 0u, 0u, 0u, 0.f, obs_normalize};
    p.sa = SauteSpec{nullptr, 1.f, 1.f, 0.f, 1.f};
    p.et = EarlySpec{nullptr, 0.f};
    p.N = N; p.precision = precision;
    return p;
}

// one act launch of the external-env path; epoch_dev non-null: the Philox counter is read on the device
static int ext_act(int O, int A, int obs_normalize, int N, int T, int t, unsigned env_id_offset, float* s_raw,
                   float* final_raw, float* norm_mean, float* norm_std, float* norm_mean1, float* norm_std1,
                   long long* norm_count, float* obs, float* act, float* logp, float* val_r, float* val_c,
                   float* boot_r, float* boot_c, unsigned char* flags, const float* theta, const float* eps,
                   unsigned noise_seed, unsigned global_step, const unsigned* epoch_dev, const float* act_lo,
                   const float* act_hi, float* act_env, int precision, void* stream) {
    OSB_CHECK_ARG(O > 0 && A > 0 && A <= OUTP && N > 0 && T > 0, "bad dims (need 0 < A <= 16)");
    OSB_CHECK_ARG(t >= 0 && t <= T, "step index out of range");
    OSB_CHECK_ARG(t == T || (act_lo && act_hi && act_env), "act_lo / act_hi / act_env are required for t < T");
    StepArgs p = ext_step_args(O, A, obs_normalize, N, precision);
    p.es.env_id_offset = env_id_offset;
    p.st.s_raw = s_raw; p.st.final_raw = final_raw;
    p.ns.mean = norm_mean; p.ns.std = norm_std; p.ns.mean1 = norm_mean1; p.ns.std1 = norm_std1; p.ns.count = norm_count;
    p.sl = Slabs{obs, act, logp, nullptr, nullptr, val_r, val_c, boot_r, boot_c, flags, nullptr};
    p.theta = theta; p.eps = eps; p.noise_seed = noise_seed; p.global_step = global_step;
    p.t = t; p.T = T; p.is_tail = (t == T) ? 1 : 0;
    p.act_lo = act_lo; p.act_hi = act_hi; p.act_env = act_env;
    p.epoch_dev = epoch_dev;
    return launch_rollout<true, false>(p, (cudaStream_t)stream);
}

static __global__ void ext_epoch_advance_kernel(unsigned* epoch_dev) { *epoch_dev += 1u; }

extern "C" {

int osb_ext_act(int O, int A, int obs_normalize, int N, int T, int t, unsigned env_id_offset, float* s_raw,
                float* final_raw, float* norm_mean, float* norm_std, float* norm_mean1, float* norm_std1,
                long long* norm_count, float* obs, float* act, float* logp, float* val_r, float* val_c, float* boot_r,
                float* boot_c, unsigned char* flags, const float* theta, const float* eps, unsigned noise_seed,
                unsigned global_step, const float* act_lo, const float* act_hi, float* act_env, int precision,
                void* stream) {
    return ext_act(O, A, obs_normalize, N, T, t, env_id_offset, s_raw, final_raw, norm_mean, norm_std, norm_mean1,
                   norm_std1, norm_count, obs, act, logp, val_r, val_c, boot_r, boot_c, flags, theta, eps, noise_seed,
                   global_step, nullptr, act_lo, act_hi, act_env, precision, stream);
}

int osb_ext_act_graph(int O, int A, int obs_normalize, int N, int T, int t, unsigned env_id_offset, float* s_raw,
                      float* final_raw, float* norm_mean, float* norm_std, float* norm_mean1, float* norm_std1,
                      long long* norm_count, float* obs, float* act, float* logp, float* val_r, float* val_c,
                      float* boot_r, float* boot_c, unsigned char* flags, const float* theta, const float* eps,
                      unsigned noise_seed, const unsigned* epoch_dev, const float* act_lo, const float* act_hi,
                      float* act_env, int precision, void* stream) {
    OSB_CHECK_ARG(epoch_dev, "epoch_dev is required");
    return ext_act(O, A, obs_normalize, N, T, t, env_id_offset, s_raw, final_raw, norm_mean, norm_std, norm_mean1,
                   norm_std1, norm_count, obs, act, logp, val_r, val_c, boot_r, boot_c, flags, theta, eps, noise_seed,
                   0u, epoch_dev, act_lo, act_hi, act_env, precision, stream);
}

int osb_ext_epoch_advance(unsigned* epoch_dev, void* stream) {
    OSB_CHECK_ARG(epoch_dev, "epoch_dev is required");
    ext_epoch_advance_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(epoch_dev);
    OSB_LAUNCH_CHECK();
    return OSB_OK;
}

int osb_ext_prepare(int O, int A, int N, int precision) {
    OSB_CHECK_ARG(O > 0 && A > 0 && A <= OUTP && N > 0, "bad dims (need 0 < A <= 16)");
    StepArgs p = ext_step_args(O, A, 0, N, precision);
    return launch_rollout<true, false>(p, nullptr, false, true);
}

// On: the network input width (O, + 1 with the Saute column); the host actions depend on nothing else of the state
int osb_eval_ext_prepare(int On, int A, int N, int precision) {
    OSB_CHECK_ARG(On > 0 && A > 0 && A <= OUTP && N > 0, "bad dims (need 0 < A <= 16)");
    OSB_CHECK_ARG(precision >= 0 && precision <= 2, "precision must be 0, 1 or 2");
    StepArgs p = ext_step_args(On, A, 0, N, precision);
    return launch_rollout<true, true>(p, nullptr, false, true);
}

}  // extern "C"
