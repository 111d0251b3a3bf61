// The fp32 state update of a running Normalizer (omnisafe/common/normalizer.py:L126-138), shared by ObsNormalize
// (rollout.cu) and Reward / CostNormalize (scalar_norm.cu).
#pragma once
#include <cuda_runtime.h>

namespace osb {

// Chan / Golub / LeVeque batched update as Normalizer._push writes it (normalizer.py:L126-135): n rows of batch mean
// mraw and sum of squared deviations m2 (rounded to fp32 as the reference's batch statistics are) merged into the
// fp32 state of count_old rows.
__device__ __forceinline__ void norm_push_moments(float& mean, float& sumsq, long long count_old, long long n,
                                                  double mraw, double m2) {
    const float mean_raw = (float)mraw, sumq_raw = (float)m2;
    const long long count = count_old + n;
    const float delta = __fadd_rn(mean_raw, -mean);
    mean = __fadd_rn(mean, __fdiv_rn(__fmul_rn(delta, (float)n), (float)count));
    const float d2 = __fmul_rn(delta, delta);
    const float corr = __fdiv_rn(__fmul_rn(__fmul_rn(d2, (float)count_old), (float)n), (float)count);
    sumsq = __fadd_rn(sumsq, __fadd_rn(sumq_raw, corr));
}

// std = max(sqrt(sumsq / (count - 1)), 1e-2) (normalizer.py:L136-138)
__device__ __forceinline__ float norm_std(float sumsq, long long count) {
    const float var = __fdiv_rn(sumsq, (float)(count - 1));
    return fmaxf(sqrtf(var), 1e-2f);
}

}  // namespace osb
