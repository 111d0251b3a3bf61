// RewardNormalize / CostNormalize (omnisafe/envs/wrapper.py:L280-423) for the slab layout.
//
// The reference pushes the N rewards (costs) of every vector step into a Normalizer(shape=(), clip=5)
// (common/normalizer.py:L88-139) and stores the normalised value in the buffer.  The policy never sees
// rewards during a rollout, so the whole epoch can be normalised AFTER the fused rollout, straight on
// the time-major slab [T][N], with exactly the reference's sequence of statistics:
//   1. row_moments_kernel : per step t the batch mean and sum of squared deviations (two passes, fixed
//                           order, fp64 accumulation rounded to the reference's fp32 values);
//   2. row_chan_kernel    : ONE thread replays the T Chan/Golub/LeVeque merges in fp32 (the running
//                           state is inherently sequential: T steps, a few hundred ns each);
//   3. row_apply_kernel   : x <- clamp((x - mean_t) / std_t, -clip, clip) with the statistics valid
//                           right after step t's push (count <= 1: passthrough, normalizer.py:L104).
#include "common.cuh"
#include "normalizer.cuh"

namespace osb {

constexpr int SN_THREADS = 256;

__device__ double sn_block_sum(double v, double* red) {
    v = warp_sum(v);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) red[w] = v;
    __syncthreads();
    double s = 0.0;
    for (int i = 0; i < SN_THREADS / 32; ++i) s += red[i];   // fixed order, every thread the same value
    return s;
}

// moments[t] = {mean_raw, sumq_raw} of row t
__global__ void __launch_bounds__(SN_THREADS) row_moments_kernel(const float* __restrict__ x, int N,
                                                                 float* __restrict__ moments) {
    __shared__ double red[SN_THREADS / 32];
    const float* row = x + (size_t)blockIdx.x * N;
    double s = 0.0;
    for (int i = threadIdx.x; i < N; i += SN_THREADS) s += (double)row[i];
    const float mean_raw = (float)(sn_block_sum(s, red) / (double)N);
    double q = 0.0;
    for (int i = threadIdx.x; i < N; i += SN_THREADS) {
        const float d = __fadd_rn(row[i], -mean_raw);
        q += (double)__fmul_rn(d, d);
    }
    const float sumq_raw = (float)sn_block_sum(q, red);
    if (threadIdx.x == 0) { moments[2 * blockIdx.x] = mean_raw; moments[2 * blockIdx.x + 1] = sumq_raw; }
}

// state = {mean, sumsq, std}; count[0] = samples seen.  row_stats[t] = {mean_t, std_t}, std_t < 0 marks
// "count <= 1 after this push" (the reference returns the data unchanged then).
__global__ void row_chan_kernel(const float* __restrict__ moments, int T, int N, float* __restrict__ state,
                                long long* __restrict__ count, float* __restrict__ row_stats) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    float mean = state[0], sumsq = state[1], stdv = state[2];
    long long c = count[0];
    for (int t = 0; t < T; ++t) {
        const float mean_raw = moments[2 * t], sumq_raw = moments[2 * t + 1];
        if (c == 0) {                     // Normalizer._first (normalizer.py:L117-125)
            mean = mean_raw; sumsq = sumq_raw; c = N;
        } else {
            norm_push_moments(mean, sumsq, c, N, mean_raw, sumq_raw);   // fp32 -> fp64 -> fp32 is exact
            c += N;
        }
        stdv = norm_std(sumsq, c);        // c == 1: inf/nan -> unused
        row_stats[2 * t] = mean;
        row_stats[2 * t + 1] = (c <= 1) ? -1.f : stdv;
    }
    state[0] = mean; state[1] = sumsq; state[2] = stdv;
    count[0] = c;
}

__global__ void __launch_bounds__(SN_THREADS) row_apply_kernel(float* __restrict__ x, int T, int N, float clip,
                                                               const float* __restrict__ row_stats) {
    const size_t total = (size_t)T * N;
    for (size_t i = (size_t)blockIdx.x * SN_THREADS + threadIdx.x; i < total; i += (size_t)gridDim.x * SN_THREADS) {
        const int t = (int)(i / N);
        const float m = __ldg(row_stats + 2 * t), s = __ldg(row_stats + 2 * t + 1);
        if (s > 0.f) x[i] = fminf(fmaxf(__fdiv_rn(__fadd_rn(x[i], -m), s), -clip), clip);
    }
}

}  // namespace osb

using namespace osb;

extern "C" {

// In-place RewardNormalize / CostNormalize of one epoch's slab x[T][N] (time-major).  state: 3 floats
// {mean, sumsq, std} + count[1] (int64), both persistent across epochs; workspace: 4 * T floats.
int osb_scalar_normalize_rows(float* x, int T, int N, float clip, float* state, long long* count,
                              float* workspace, void* stream) {
    OSB_CHECK_ARG(x && state && count && workspace && T > 0 && N > 0 && clip > 0.f, "bad argument");
    cudaStream_t s = (cudaStream_t)stream;
    float* moments = workspace;
    float* row_stats = workspace + 2 * (size_t)T;
    row_moments_kernel<<<T, SN_THREADS, 0, s>>>(x, N, moments);
    OSB_LAUNCH_CHECK();
    row_chan_kernel<<<1, 32, 0, s>>>(moments, T, N, state, count, row_stats);
    OSB_LAUNCH_CHECK();
    const size_t total = (size_t)T * N;
    int blocks = (int)((total + SN_THREADS - 1) / SN_THREADS);
    if (blocks > 8 * grid_sms()) blocks = 8 * grid_sms();
    row_apply_kernel<<<blocks, SN_THREADS, 0, s>>>(x, T, N, clip, row_stats);
    OSB_LAUNCH_CHECK();
    return OSB_OK;
}

}  // extern "C"
