// The two small reductions behind the learner kernels of every arithmetic mode (csrc/loss.cuh): the pass-1 gate of
// the two-pass losses and the fixed-order sum of the evaluation partials.
#include "loss.cuh"

namespace osb {

// stats_part rows of the actor (network 0); slot 3 counts the samples
__global__ void pass1_gate_kernel(const float* __restrict__ stats_part, int nblocks, float* __restrict__ out,
                                  const int* __restrict__ stop_flag, int kind, float kappa, float jc_minus_limit) {
    if (threadIdx.x != 0 || (stop_flag && *stop_flag)) return;
    const int slot = (kind == LOSS_P3O) ? 2 : 4;
    float m = 0.f, n = 0.f;
    for (int b = 0; b < nblocks; ++b) { m += stats_part[((size_t)b * 3) * 8 + slot]; n += stats_part[((size_t)b * 3) * 8 + 3]; }
    const float mean = n > 0.f ? m / n : 0.f;
    out[0] = (kind == LOSS_P3O) ? ((mean + jc_minus_limit > 0.f) ? kappa : 0.f) : mean;
}

// 32 groups x 8 statistics: group g sums CTAs g, g+32, ... ; the 32 group sums fold in a fixed order
__global__ void eval_reduce_kernel(const double* __restrict__ part, int nblocks, double* __restrict__ out) {
    __shared__ double sh[32][8];
    const int q = threadIdx.x & 7, g = threadIdx.x >> 3;
    double s = 0.0;
    for (int b = g; b < nblocks; b += 32) s += part[(size_t)b * 8 + q];
    sh[g][q] = s;
    __syncthreads();
    if (threadIdx.x < 8) {
        double t = 0.0;
        for (int i = 0; i < 32; ++i) t += sh[i][threadIdx.x];
        out[threadIdx.x] = (threadIdx.x < 6) ? t : 0.0;
    }
}

int pass1_gate(const float* stats_part, int nblocks, const int* stop_flag, LossParams& lp, cudaStream_t stream) {
    static float* d_gate = nullptr;
    if (!d_gate) OSB_CUDA(cudaMalloc(&d_gate, sizeof(float)));
    pass1_gate_kernel<<<1, 32, 0, stream>>>(stats_part, nblocks, d_gate, stop_flag, lp.kind, lp.focops_lam, lp.focops_eta);
    OSB_LAUNCH_CHECK();
    lp.pass1 = d_gate;
    return OSB_OK;
}

int eval_reduce(const double* part, int nblocks, double* out, cudaStream_t stream) {
    eval_reduce_kernel<<<1, 256, 0, stream>>>(part, nblocks, out);
    OSB_LAUNCH_CHECK();
    return OSB_OK;
}

}  // namespace osb
