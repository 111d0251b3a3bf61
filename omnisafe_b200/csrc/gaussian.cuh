// Diagonal-Gaussian policy arithmetic (GaussianLearningActor, models/actor/gaussian_learning_actor.py:L64-139, on
// torch.distributions.Normal), shared by the rollout step kernels (csrc/rollout.cu) and the policy-step kernels
// (csrc/policy.cu), so that a sampled action and its log-prob are the same bits wherever they are computed.
#pragma once
#include "common.cuh"

namespace osb {

// The log_prob term of one action component x under Normal(mu, sigma), in Normal.log_prob's order:
// -((x - loc)^2) / (2 var) - log(scale) - log(sqrt(2 pi)).  two_var = 2 sigma^2, log_sd = log sigma.
__device__ __forceinline__ float gaussian_log_prob(float x, float mu, float two_var, float log_sd) {
    const float d = __fadd_rn(x, -mu);
    const float term = __fdiv_rn(-__fmul_rn(d, d), two_var);
    return __fadd_rn(__fadd_rn(term, -log_sd), -0.9189385332046727f);
}

// One action component of Normal(mu, sigma): the action rsample gives (loc + eps * scale) and, in `term`, its log_prob
// term (gaussian_log_prob).  eps = 0 gives the mean (predict(obs, deterministic=True)).
__device__ __forceinline__ float sample_action(float mu, float sd, float two_var, float log_sd, float eps, float& term) {
    const float act = __fadd_rn(mu, __fmul_rn(sd, eps));
    term = gaussian_log_prob(act, mu, two_var, log_sd);
    return act;
}

}  // namespace osb
