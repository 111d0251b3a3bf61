// Tile-level MLP building blocks (fp32 FMA path, exact-fp32 "parity" arithmetic).
//
// The actor / reward-critic / cost-critic are three independent Linear-Act-Linear-Act-Linear
// trunks (omnisafe/utils/model.py:L73-111, models/actor/gaussian_learning_actor.py:L29-62,
// models/critic/v_critic.py:L27-73).  A CTA of 256 threads owns a tile of MT samples; activations
// and one network's weights live in shared memory and every layer is a register-tiled GEMM.
//
// Flat parameter order per network = the reference's named_parameters() order
// (omnisafe/utils/tools.py:L35-129):
//   actor : log_std[A], W1[H][O], b1[H], W2[H][H], b2[H], W3[A][H], b3[A]
//   critic:             W1[H][O], b1[H], W2[H][H], b2[H], W3[1][H], b3[1]
#pragma once
#include "activation.cuh"
#include "common.cuh"

namespace osb {

constexpr int HID = 64;      // hidden width (both layers); the configs use [64, 64]
constexpr int KC = 64;       // obs chunk width (layer-1 K is processed in chunks of 64)
constexpr int LD = 68;       // smem row stride in floats: 16 B aligned rows, LD/4 odd
constexpr int OUTP = 16;     // padded output width (A <= 16)
constexpr int LDO = 20;      // smem row stride of the [*, OUTP] tiles
constexpr int NTHREADS = 256;

struct NetLayout {
    int O, A, out;   // obs dim, act dim, output width of this net (A or 1)
    int off_logstd;  // -1 for critics
    int off_w1, off_b1, off_w2, off_b2, off_w3, off_b3, size;
};

__host__ __device__ inline NetLayout actor_layout(int O, int A) {
    NetLayout l;
    l.O = O; l.A = A; l.out = A;
    l.off_logstd = 0;
    l.off_w1 = A;
    l.off_b1 = l.off_w1 + HID * O;
    l.off_w2 = l.off_b1 + HID;
    l.off_b2 = l.off_w2 + HID * HID;
    l.off_w3 = l.off_b2 + HID;
    l.off_b3 = l.off_w3 + A * HID;
    l.size = l.off_b3 + A;
    return l;
}
__host__ __device__ inline NetLayout critic_layout(int O, int A) {
    NetLayout l;
    l.O = O; l.A = A; l.out = 1;
    l.off_logstd = -1;
    l.off_w1 = 0;
    l.off_b1 = HID * O;
    l.off_w2 = l.off_b1 + HID;
    l.off_b2 = l.off_w2 + HID * HID;
    l.off_w3 = l.off_b2 + HID;
    l.off_b3 = l.off_w3 + HID;
    l.size = l.off_b3 + 1;
    return l;
}
// net 0 = actor, 1 = reward critic, 2 = cost critic; flat theta = [actor | critic_r | critic_c]
__host__ __device__ inline NetLayout net_layout(int net, int O, int A) {
    return net == 0 ? actor_layout(O, A) : critic_layout(O, A);
}
__host__ __device__ inline int net_offset(int net, int O, int A) {
    const int sa = actor_layout(O, A).size, sc = critic_layout(O, A).size;
    return net == 0 ? 0 : (net == 1 ? sa : sa + sc);
}

// Shared-memory image of one network's weights.
struct NetSmem {
    float* w1;   // [HID][LD]  chunk kc of W1 (zero padded beyond O)
    float* w2;   // [HID][LD]
    float* w2t;  // [HID][LD]  W2 transposed (only filled when NEED_T)
    float* w3;   // [OUTP][LD] rows >= out are zero
    float* w3t;  // [HID][LDO] W3 transposed, cols >= out zero (only when NEED_T)
    float* b1;   // [HID]
    float* b2;   // [HID]
    float* b3;   // [OUTP]
};
constexpr int NETSMEM_FLOATS_FWD = 2 * HID * LD + OUTP * LD + 2 * HID + OUTP;
constexpr int NETSMEM_FLOATS_BWD = NETSMEM_FLOATS_FWD + HID * LD + HID * LDO;

template <bool NEED_T>
__device__ __forceinline__ float* carve_net_smem(float* base, NetSmem& s) {
    s.w1 = base; base += HID * LD;
    s.w2 = base; base += HID * LD;
    s.w3 = base; base += OUTP * LD;
    s.b1 = base; base += HID;
    s.b2 = base; base += HID;
    s.b3 = base; base += OUTP;
    if (NEED_T) {
        s.w2t = base; base += HID * LD;
        s.w3t = base; base += HID * LDO;
    } else {
        s.w2t = nullptr; s.w3t = nullptr;
    }
    return base;
}

// Loads W1 chunk `kc` (columns [kc*KC, kc*KC+KC) of W1[H][O]) zero padded.
__device__ __forceinline__ void load_w1_chunk(const float* __restrict__ theta, const NetLayout& L,
                                              int kc, NetSmem& s) {
    const int c0 = kc * KC;
    for (int i = threadIdx.x; i < HID * KC; i += NTHREADS) {
        const int n = i / KC, k = i % KC;
        const int col = c0 + k;
        s.w1[n * LD + k] = (col < L.O) ? __ldg(theta + L.off_w1 + n * L.O + col) : 0.f;
    }
}

template <bool NEED_T>
__device__ __forceinline__ void load_net_rest(const float* __restrict__ theta, const NetLayout& L,
                                              NetSmem& s) {
    for (int i = threadIdx.x; i < HID * HID; i += NTHREADS) {
        const int n = i / HID, k = i % HID;
        const float w = __ldg(theta + L.off_w2 + i);
        s.w2[n * LD + k] = w;
        if (NEED_T) s.w2t[k * LD + n] = w;
    }
    for (int i = threadIdx.x; i < OUTP * HID; i += NTHREADS) {
        const int o = i / HID, k = i % HID;
        const float w = (o < L.out) ? __ldg(theta + L.off_w3 + o * HID + k) : 0.f;
        s.w3[o * LD + k] = w;
        if (NEED_T) s.w3t[k * LDO + o] = w;
    }
    if (threadIdx.x < HID) {
        s.b1[threadIdx.x] = __ldg(theta + L.off_b1 + threadIdx.x);
        s.b2[threadIdx.x] = __ldg(theta + L.off_b2 + threadIdx.x);
    }
    if (threadIdx.x < OUTP)
        s.b3[threadIdx.x] = (threadIdx.x < L.out) ? __ldg(theta + L.off_b3 + threadIdx.x) : 0.f;
}

// C[m][n] = sum_k A[m][k] * B[n][k]   (m < MT, n < 64, k < K; K % 4 == 0)
// thread (tm = tid/16, tn = tid%16) owns rows tm+16i, cols tn+16j.
template <int MT, int LDA, int LDB>
__device__ __forceinline__ void gemm_nt(const float* __restrict__ A, const float* __restrict__ B,
                                        int K, float (&acc)[MT / 16][4]) {
    constexpr int MI = MT / 16;
    const int tm = threadIdx.x >> 4, tn = threadIdx.x & 15;
#pragma unroll
    for (int i = 0; i < MI; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
#pragma unroll 2
    for (int k = 0; k < K; k += 4) {
        float4 a[MI], b[4];
#pragma unroll
        for (int i = 0; i < MI; ++i)
            a[i] = *reinterpret_cast<const float4*>(A + (tm + 16 * i) * LDA + k);
#pragma unroll
        for (int j = 0; j < 4; ++j)
            b[j] = *reinterpret_cast<const float4*>(B + (tn + 16 * j) * LDB + k);
#pragma unroll
        for (int i = 0; i < MI; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                float c = acc[i][j];
                c = fmaf(a[i].x, b[j].x, c);
                c = fmaf(a[i].y, b[j].y, c);
                c = fmaf(a[i].z, b[j].z, c);
                c = fmaf(a[i].w, b[j].w, c);
                acc[i][j] = c;
            }
    }
}

// G[j][k] = sum_s P[s][j] * Q[s][k]   (j < 64, k < 64, s < MT)
// thread (tj = tid/16, tk = tid%16) owns j in [4tj, 4tj+4), k in [4tk, 4tk+4).
template <int MT, int LDP, int LDQ>
__device__ __forceinline__ void gemm_tn(const float* __restrict__ P, const float* __restrict__ Q,
                                        float (&acc)[4][4]) {
    const int j0 = (threadIdx.x >> 4) * 4, k0 = (threadIdx.x & 15) * 4;
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;
#pragma unroll 4
    for (int s = 0; s < MT; ++s) {
        const float4 p = *reinterpret_cast<const float4*>(P + s * LDP + j0);
        const float4 q = *reinterpret_cast<const float4*>(Q + s * LDQ + k0);
        const float pv[4] = {p.x, p.y, p.z, p.w};
        const float qv[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b) acc[a][b] = fmaf(pv[a], qv[b], acc[a][b]);
    }
}

// Hidden layers of one network on a tile: X[MT][LD] (chunk 0 resident) -> H1 = f(Z1), H2 = f(Z2), f = act.
// For O > KC the caller supplies a functor that (re)loads X chunk kc and W1 chunk kc.
template <int MT, class Act, typename LoadChunk>
__device__ __forceinline__ void mlp_hidden(const float* __restrict__ sX, float* __restrict__ sH1,
                                           float* __restrict__ sH2, NetSmem& W, int nchunks, const Act& act,
                                           LoadChunk load_chunk) {
    constexpr int MI = MT / 16;
    const int tm = threadIdx.x >> 4, tn = threadIdx.x & 15;
    float z[MI][4];
    float acc[MI][4];
    gemm_nt<MT, LD, LD>(sX, W.w1, KC, z);
    for (int kc = 1; kc < nchunks; ++kc) {
        __syncthreads();
        load_chunk(kc);
        __syncthreads();
        gemm_nt<MT, LD, LD>(sX, W.w1, KC, acc);
#pragma unroll
        for (int i = 0; i < MI; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) z[i][j] += acc[i][j];
    }
#pragma unroll
    for (int i = 0; i < MI; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = tn + 16 * j;
            sH1[(tm + 16 * i) * LD + n] = act(z[i][j] + W.b1[n], n, act.w1);
        }
    __syncthreads();
    gemm_nt<MT, LD, LD>(sH1, W.w2, HID, acc);
#pragma unroll
    for (int i = 0; i < MI; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = tn + 16 * j;
            sH2[(tm + 16 * i) * LD + n] = act(acc[i][j] + W.b2[n], n, act.w2);
        }
    __syncthreads();
}

// Output layer: sO[m][o] = b3[o] + sum_k H2[m][k] W3[o][k], o < out (<= OUTP).
template <int MT>
__device__ __forceinline__ void mlp_out(const float* __restrict__ sH2, float* __restrict__ sO,
                                        const NetSmem& W, int out) {
    // thread -> row m = tid % MT, output group og = tid / MT (NTHREADS/MT groups)
    constexpr int NG = NTHREADS / MT;
    const int m = threadIdx.x % MT, og = threadIdx.x / MT;
    for (int o = og; o < out; o += NG) {
        float c = 0.f;
#pragma unroll 4
        for (int k = 0; k < HID; k += 4) {
            const float4 h = *reinterpret_cast<const float4*>(sH2 + m * LD + k);
            const float4 w = *reinterpret_cast<const float4*>(W.w3 + o * LD + k);
            c = fmaf(h.x, w.x, c); c = fmaf(h.y, w.y, c);
            c = fmaf(h.z, w.z, c); c = fmaf(h.w, w.w, c);
        }
        sO[m * LDO + o] = c + W.b3[o];
    }
    __syncthreads();
}

}  // namespace osb
