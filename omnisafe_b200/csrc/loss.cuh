// Per-sample arithmetic of the learner, shared by the fp32 (update.cu), tf32 (update_tc.cu, eval_tc.cu) and
// bf16x3 (update_x3.cu, eval_tc.cu) kernels: the loss kinds, the minibatch sample order, the actor loss of the
// update with its gradients, and the statistics of the full-batch evaluation.  The kernels differ in how they
// stage a sample's inputs and how they reduce the results; what they compute per sample is defined here once.
//
//   PPO._loss_pi                            algorithms/on_policy/base/ppo.py:L35-87
//   PPOLag._compute_adv_surrogate           naive_lagrange/ppo_lag.py:L82-102
//   PolicyGradient._loss_pi (plain ratio)   base/policy_gradient.py:L551-588
//   CPO._loss_pi_cost                       second_order/cpo.py:L182-212
//   FOCOPS._loss_pi                         first_order/focops.py:L62-108
//   P3O._loss_pi                            penalty_function/p3o.py:L48-91
//   KL early-stop evaluation                base/policy_gradient.py:L383-397
#pragma once
#include "common.cuh"

namespace osb {

// loss_kind of the C ABI (engine.py LOSS_*)
enum LossKind {
    LOSS_PPO_CLIP = 0,
    LOSS_RATIO = 1,
    LOSS_FOCOPS = 2,   // two passes
    LOSS_COST = 3,
    LOSS_FVP = 4,      // dOUT supplied: backward half of the tensor-core Fisher-vector products
    LOSS_P3O = 5,      // two passes
    LOSS_DMU = 6,      // dOUT = dmu (actor) or dV (critic) supplied per row: J^T dOUT of the MLP (losses written in
                       // PyTorch); compiled only into the DMU instantiations of the stepwise kernels
};

// FOCOPS and P3O need a minibatch mean before any gradient: a forward-only pass 1 feeds pass1_gate().
__host__ __device__ __forceinline__ bool loss_two_pass(int kind) { return kind == LOSS_FOCOPS || kind == LOSS_P3O; }

// Only PPO._loss_pi and FOCOPS._loss_pi carry the entropy bonus.  EXT = false: the kernel is compiled without the
// two-pass kinds.
template <bool EXT = true>
__host__ __device__ __forceinline__ bool loss_has_entropy(int kind) {
    return kind == LOSS_PPO_CLIP || (EXT && (kind == LOSS_FOCOPS || kind == LOSS_P3O));
}

// The rollout slabs (row = t*N + i) and the samples of one launch: the window [mb_start, mb_start + mb_count)
// of a sample order over [0, total).
struct Batch {
    const float* obs;     // [rows][O]
    const float* act;     // [rows][A]
    const float* logp;    // [rows]
    const float* adv_r;   // [rows] raw advantages (standardised on the fly with `moments`)
    const float* adv_c;   // [rows]
    const float* tv_r;    // [rows] critic targets
    const float* tv_c;    // [rows]
    const float* moments; // [4] mean_r, std_r + 1e-8, mean_c, 1; null: 0, 1, 0
    const int* perm;      // [total] slab rows in minibatch order (parity mode: the reference's DataLoader order), or null
    long long total;      // number of samples the order ranges over
    unsigned perm_seed;   // Feistel key (perm == null)
    long long mb_start;
    int mb_count;
    int identity_stride;  // > 0: row = k * identity_stride (full-batch passes, fvp_sample_freq)
};

// Keyed bijection on [0, n): 4-round Feistel on the enclosing power-of-four domain + cycle walking.
__device__ __forceinline__ unsigned long long feistel_perm(unsigned long long k, unsigned long long n, unsigned seed) {
    int bits = 2;
    while ((1ull << bits) < n) bits += 2;
    const int half = bits >> 1;
    const unsigned mask = (1u << half) - 1u;
    unsigned long long x = k;
    do {
        unsigned l = (unsigned)(x >> half) & mask, r = (unsigned)x & mask;
#pragma unroll
        for (int round = 0; round < 4; ++round) {
            const unsigned f = mix32(r ^ (seed + 0x9E3779B9u * (unsigned)(round + 1))) & mask;
            const unsigned nl = r;
            r = l ^ f;
            l = nl;
        }
        x = ((unsigned long long)l << half) | r;
    } while (x >= n);
    return x;
}

// Slab row of sample k of the order.
__device__ __forceinline__ long long sample_row(const Batch& b, long long k) {
    if (b.identity_stride > 0) return k * b.identity_stride;
    return b.perm ? (long long)b.perm[k] : (long long)feistel_perm((unsigned long long)k, (unsigned long long)b.total, b.perm_seed);
}

struct LossParams {
    int kind;                       // LossKind of the actor
    float clip;                     // PPO clip
    float entropy_coef;
    float focops_lam, focops_eta;   // P3O: kappa, Jc - limit
    const float* lagrange;          // device scalar lambda or null (0): adv = (adv_r - lambda adv_c) / (1 + lambda)
    const float* mu_old;            // [rows][A] old-policy mean (FOCOPS)
    const float* logstd_old;        // [A] old-policy log_std (FOCOPS)
    const float* pass1;             // two-pass kinds: the pass1_gate() scalar in pass 2, null in pass 1
};

// Advantage standardisation and Lagrangian mix, per thread.  The update multiplies by the reciprocals, the
// evaluation divides (its results feed the line search and the KL early stop bit for bit).
struct AdvNorm {
    float m_r, s_r, m_c, lam;
    float inv_sr, inv_1lam;
};
__device__ __forceinline__ AdvNorm adv_norm(const float* moments, const float* lagrange) {
    AdvNorm n;
    n.lam = (lagrange != nullptr) ? __ldg(lagrange) : 0.f;
    n.m_r = 0.f; n.s_r = 1.f; n.m_c = 0.f;
    if (moments) { n.m_r = __ldg(moments + 0); n.s_r = __ldg(moments + 1); n.m_c = __ldg(moments + 2); }
    n.inv_sr = 1.f / n.s_r;
    n.inv_1lam = 1.f / (1.f + n.lam);
    return n;
}

// Per-CTA policy constants in shared memory, 16 floats per field, staged once per CTA (thread i: action i):
//   update      pol = log sigma | sigma | 1 / sigma^2        old = log sigma_old | 1 / sigma_old^2  (FOCOPS)
//   evaluation  pol = log sigma | sigma | log sigma_old | sigma_old
__device__ __forceinline__ void stage_policy(float* pol, int i, float log_std) {
    const float sd = expf(log_std);
    pol[i] = log_std; pol[16 + i] = sd; pol[32 + i] = 1.f / (sd * sd);
}
__device__ __forceinline__ void stage_policy_old(float* old, int i, float log_std_old) {
    const float so = expf(log_std_old);
    old[i] = log_std_old; old[16 + i] = 1.f / (so * so);
}
__device__ __forceinline__ void stage_eval_policy(float* pol, int i, float log_std, float log_std_old) {
    pol[i] = log_std; pol[16 + i] = expf(log_std); pol[32 + i] = log_std_old; pol[48 + i] = expf(log_std_old);
}

// Actor loss of one sample.
//   st = {loss, ratio, slot 2, count, slot 4}: the sample's statistics are added to it (slot 0: the loss without the
//   entropy bonus, which entropy_bonus_sum adds to slot 5, and without the P3O penalty; slot 2: FOCOPS KL, P3O
//   ratio * adv_c in pass 1 and the penalty term in pass 2; slot 4: FOCOPS mask 1{KL <= eta}).
//   grad(a, dL/dmu_a, dL/dlog_std_a) receives the gradients of every action a < A, already divided by the minibatch
//   size (inv_b).  The caller stores or accumulates them right there, in the same straight-line code as the products,
//   so fused multiply-adds form as in a hand-inlined loss.
//   mu, act: the sample's mean (bias included) and action, entries a < A.  mu_old(a): the sample's old mean, called
//   only by FOCOPS inside its KL loop, so a caller that reads it from global memory keeps no registers for it.
//   [a_lo, a_hi): the actions whose gradients are formed (default all), and stats: whether st is added to.  Everything
//   else, logp_new over every action included, is computed in full, so callers that split the actions of a sample among
//   threads get the same bits in each, and one of them keeps the statistics.
// EXT = false compiles only PPO-clip, ratio and cost surrogate.
template <bool EXT, int AP, class MuOld, class Grad>
__device__ __forceinline__ void actor_sample_loss(const LossParams& lp, const AdvNorm& an, int A, float inv_b,
                                                  const float (&mu)[AP], const float (&act)[AP], MuOld&& mu_old,
                                                  float logp_old, float adv_r_raw, float adv_c_raw, const float* pol,
                                                  const float* old, float (&st)[5], Grad&& grad, int a_lo = 0,
                                                  int a_hi = AP, bool stats = true) {
    float logp_new = 0.f, diff[AP];
#pragma unroll
    for (int a = 0; a < AP; ++a) {
        diff[a] = 0.f;
        if (a < A) {
            const float d = act[a] - mu[a];
            diff[a] = d;
            logp_new += -(d * d) * (0.5f * pol[32 + a]) - pol[a] - 0.9189385332046727f;
        }
    }
    const float ratio = expf(logp_new - logp_old);
    const float adv_r = (adv_r_raw - an.m_r) * an.inv_sr;
    const float adv_c = adv_c_raw - an.m_c;
    const float adv = (adv_r - an.lam * adv_c) * an.inv_1lam;
    float loss, dlogp;
    if (lp.kind == LOSS_PPO_CLIP || (EXT && lp.kind == LOSS_P3O)) {
        const float rc = fminf(fmaxf(ratio, 1.f - lp.clip), 1.f + lp.clip);
        const float s1 = ratio * adv, s2 = rc * adv;
        loss = -fminf(s1, s2);
        dlogp = (s1 <= s2) ? -adv * ratio * inv_b : 0.f;
        if (EXT && lp.kind == LOSS_P3O) {
            // + kappa * relu(mean_j(ratio_j adv_c_j) + Jc - limit); the gate (kappa when the minibatch mean makes the
            // relu active) comes from pass 1.  Slot 0 stays the PPO part, as the reference logs Loss/Loss_pi.
            const bool pass2 = lp.pass1 != nullptr;
            const float gate = pass2 ? __ldg(lp.pass1) : 0.f;
            dlogp += gate * adv_c * ratio * inv_b;
            if (stats) st[2] += pass2 ? gate * (ratio * adv_c + lp.focops_eta) : ratio * adv_c;   // Loss/Loss_pi_cost
        }
    } else if (lp.kind == LOSS_RATIO) {
        loss = -ratio * adv; dlogp = -adv * ratio * inv_b;
    } else if (lp.kind == LOSS_COST) {
        loss = ratio * adv_c; dlogp = adv_c * ratio * inv_b;
    }
    const bool focops = EXT && lp.kind == LOSS_FOCOPS;
    float dmask = 0.f, dmo[AP];
#pragma unroll
    for (int a = 0; a < AP; ++a) dmo[a] = 0.f;
    if (focops) {
        // The reference forms (kl[b,1] - ratio[b] adv[b] / lam) * mask[b,1] and takes the mean of the [b,b] matrix
        // (first_order/focops.py:L85-89), i.e.
        //   loss = mean_i(mask_i kl_i) - mean_i(mask_i) * mean_j(ratio_j adv_j) / lam ;
        // mean_i(mask_i) of this minibatch comes from pass 1.
        float kl = 0.f;
#pragma unroll
        for (int a = 0; a < AP; ++a)
            if (a < A) {
                const float sn = pol[16 + a];
                dmo[a] = mu[a] - mu_old(a);
                kl += (old[a] - pol[a]) + (sn * sn + dmo[a] * dmo[a]) * (0.5f * old[16 + a]) - 0.5f;
            }
        dmask = (kl <= lp.focops_eta) ? 1.f : 0.f;
        const float mbar = lp.pass1 ? __ldg(lp.pass1) : dmask;
        loss = kl * dmask - mbar * ratio * adv / lp.focops_lam;
        dlogp = -mbar * adv * ratio / lp.focops_lam * inv_b;
        if (stats) { st[2] += kl; st[4] += dmask; }
    }
    if (stats) { st[0] += loss; st[1] += ratio; st[3] += 1.f; }
#pragma unroll
    for (int a = 0; a < AP; ++a) {
        if (a < A && a >= a_lo && a < a_hi) {
            const float iv = pol[32 + a];
            float dm = dlogp * diff[a] * iv;                    // d logp / d mu
            float dl = dlogp * (diff[a] * diff[a] * iv - 1.f);  // d logp / d log_std
            if (focops) {
                const float sn = pol[16 + a];
                dm += dmask * inv_b * dmo[a] * old[16 + a];
                dl += dmask * inv_b * (sn * sn * old[16 + a] - 1.f);
            }
            grad(a, dm, dl);
        }
    }
}

// Slot 5 of the actor's statistics: the entropy bonus -entropy_coef * mean entropy summed over the CTA's `count` samples
// (Loss/Loss_pi is logged after loss -= entropy_coef * entropy.mean(), base/ppo.py:L76-84, first_order/focops.py:
// L108-116).  Every sample's entropy is 0.5 + 0.5 log 2 pi + mean_a log sigma_a, so a CTA forms it once, where it adds
// the bonus's gradient -entropy_coef / A to every log_std.  pol: the update layout of stage_policy's comment, still
// holding the sigma of the minibatch.  Logging only.
template <bool EXT = true>
__device__ __forceinline__ float entropy_bonus_sum(const LossParams& lp, int A, const float* pol, float count) {
    if (!loss_has_entropy<EXT>(lp.kind)) return 0.f;
    float ls = 0.f;
    for (int a = 0; a < A; ++a) ls += pol[a];
    return -lp.entropy_coef * (1.4189385332046727f + ls / (float)A) * count;
}

// Full-batch evaluation of one sample, added to acc = {sum_a KL(old || new), ratio * adv, ratio * adv_c, ratio,
// count, ratio * adv_r} (fp32 per sample, fp64 sums).  pol: the evaluation layout of stage_policy's comment.
template <int AP>
__device__ __forceinline__ void eval_sample(const AdvNorm& an, int A, const float (&mu)[AP], const float (&act)[AP],
                                            const float (&mu_old)[AP], float logp_old, float adv_r_raw, float adv_c_raw,
                                            const float* pol, double (&acc)[6]) {
    float logp_new = 0.f, kl = 0.f;
#pragma unroll
    for (int a = 0; a < AP; ++a)
        if (a < A) {
            const float sd = pol[16 + a], so = pol[48 + a];
            const float d = act[a] - mu[a];
            logp_new += -(d * d) / (2.f * sd * sd) - pol[a] - 0.9189385332046727f;
            // KL(old || new) per dimension (torch.distributions.kl._kl_normal_normal)
            const float vr = (so / sd) * (so / sd);
            const float t1 = (mu_old[a] - mu[a]) / sd;
            kl += 0.5f * (vr + t1 * t1 - 1.f - logf(vr));
        }
    const float ratio = expf(logp_new - logp_old);
    const float adv_r = (adv_r_raw - an.m_r) / an.s_r, adv_c = adv_c_raw - an.m_c;
    const float adv = (adv_r - an.lam * adv_c) / (1.f + an.lam);
    acc[0] += (double)kl; acc[1] += (double)(ratio * adv); acc[2] += (double)(ratio * adv_c);
    acc[3] += (double)ratio; acc[4] += 1.0; acc[5] += (double)(ratio * adv_r);
}

// ---- host side (csrc/loss.cu) ------------------------------------------------------------------------------------
// After pass 1 of a two-pass kind: reduces the actor rows of stats_part ([nblocks][3][8]) in fixed order into a device
// scalar that this function owns, and points lp.pass1 at it for pass 2.
//   FOCOPS: mean_i mask_i                                                     (slot 4 / slot 3)
//   P3O:    kappa if mean_i(ratio_i adv_c_i) + (Jc - limit) > 0 else 0        (slot 2 / slot 3; F.relu gate)
int pass1_gate(const float* stats_part, int nblocks, const int* stop_flag, LossParams& lp, cudaStream_t stream);
// out[8] <- fixed-order sums of the evaluation partials part[nblocks][8] (slots 6 and 7 zero).
int eval_reduce(const double* part, int nblocks, double* out, cudaStream_t stream);
// LOSS_DMU launches of the tensor-core kernels (csrc/update_tc.cu, csrc/update_x3.cu) behind osb_actor_dmu_backward:
// rows obs[rows][O] in order, dmu[rows][A]; gpart: osb_tc_grid_blocks(rows, 1) rows of P_actor floats.
int dmu_backward_tc(const float* theta_actor, int O, int A, const float* obs, const float* dmu, int rows, float* gpart,
                    float* stats_scratch, cudaStream_t stream);
int dmu_backward_x3(const float* theta_actor, int O, int A, const float* obs, const float* dmu, int rows, float* gpart,
                    float* stats_scratch, cudaStream_t stream);
// The backward halves of osb_fvp_partials_tc / osb_fvp_partials_x3 (csrc/fvp_tc.cu): the actor backward of the LOSS_FVP
// kind with dOUT = dmu / sigma^2 / (rows * A) over rows 0, stride, 2 stride, ... of obs [total][O], dmu [total][A];
// gpart: osb_tc_grid_blocks(rows, 1) rows of P_actor floats, rows = ceil(total / stride).
int fvp_backward_tc(const float* theta_actor, const float* vec, int O, int A, const float* obs, long long total, int stride,
                    const float* dmu, float* gpart, float* stats_scratch, cudaStream_t stream);
int fvp_backward_x3(const float* theta_actor, const float* vec, int O, int A, const float* obs, long long total, int stride,
                    const float* dmu, float* gpart, float* stats_scratch, cudaStream_t stream);
// ... and behind osb_critic_dv_backward: critic `net` (1, 2) of the flat theta, dv[rows] = dL/dV, value[rows] (or
// null) <- V; gpart: osb_tc_grid_blocks(rows, 1 << net) rows of P floats (the critic's segment written).
int dv_backward_tc(const float* theta, int O, int A, int net, const float* obs, const float* dv, float* value, int rows,
                   float* gpart, float* stats_scratch, cudaStream_t stream);
int dv_backward_x3(const float* theta, int O, int A, int net, const float* obs, const float* dv, float* value, int rows,
                   float* gpart, float* stats_scratch, cudaStream_t stream);

}  // namespace osb
