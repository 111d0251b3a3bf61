// Network optimiser arithmetic (torch.optim.Adam single-tensor path, betas 0.9 / 0.999, eps 1e-8, no weight decay;
// clip_grad_norm_; the logged minibatch means, policy_gradient.py:L429-443), shared by the stepwise, cooperative and
// NVLink optimiser kernels (csrc/optim.cu) and the persistent bf16x3 update kernel (csrc/update_x3.cu), so that a
// trained parameter is the same bits on every path.  The roundings are torch's: explicit __f*_rn where torch rounds
// each tensor op, fp64 scalars for the bias corrections.
#pragma once
#include "common.cuh"

namespace osb {

// Per-step scalars of Adam step t (1-based) at rate lr: step_size = lr / (1 - 0.9^t), bc2_sqrt = sqrt(1 - 0.999^t).
struct AdamScalars {
    float step_size, bc2_sqrt;
};
__device__ __forceinline__ AdamScalars adam_scalars(float lr, int t) {
    const double bc1 = 1.0 - pow(0.9, (double)t), bc2 = 1.0 - pow(0.999, (double)t);
    return {(float)((double)lr / bc1), (float)sqrt(bc2)};
}

// One Adam step of one parameter th with gradient g: updates m and v, returns the new parameter.
__device__ __forceinline__ float adam_update(float g, float th, float& m, float& v, AdamScalars s) {
    m = __fadd_rn(m, __fmul_rn(0.1f, __fadd_rn(g, -m)));                       // exp_avg.lerp_(grad, 1 - beta1)
    v = __fadd_rn(__fmul_rn(v, 0.999f), __fmul_rn(__fmul_rn(0.001f, g), g));   // mul_(beta2).addcmul_(g, g, 1 - beta2)
    const float denom = __fadd_rn(__fdiv_rn(sqrtf(v), s.bc2_sqrt), 1e-8f);
    return __fadd_rn(th, __fmul_rn(-s.step_size, __fdiv_rn(m, denom)));
}

// clip_grad_norm_ coefficient of a gradient with squared norm sumsq (max_norm > 0).
__device__ __forceinline__ float clip_coef(float sumsq, float max_norm) {
    return fminf(max_norm / (sqrtf(sumsq) + 1e-6f), 1.0f);
}

// One minibatch step into train_stats[net] ({loss, ratio, kl, steps, entropy bonus}): the means of the summed loss
// statistics over `count` samples, the critics' logged loss with its regulariser critic_norm_coef * sum theta^2 (t2).
__device__ __forceinline__ void fold_minibatch_stats(float* train_stats, int net, float loss, float ratio, float kl,
                                                     float count, float ent, float critic_norm_coef, float t2) {
    const float inv = count > 0.f ? 1.f / count : 0.f;
    float* ts = train_stats + net * 8;
    ts[0] += loss * inv + ((net != 0) ? critic_norm_coef * t2 : 0.f);
    ts[1] += ratio * inv;
    ts[2] += kl * inv;
    ts[3] += 1.f;
    ts[4] += ent * inv;   // actor: mean entropy bonus (csrc/loss.cuh entropy_bonus_sum)
}

}  // namespace osb
