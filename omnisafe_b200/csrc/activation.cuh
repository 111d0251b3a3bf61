// The hidden-layer activation of the MLP kernels (model_cfgs.actor / critic.activation, omnisafe/utils/model.py:L62-70):
// one definition of the forward, the derivative from the stored output and the pad mask, shared by every kernel.
//
//   tanh      f = tanh z (per precision: tanhf, MUFU tanh.approx, x3::tanh_acc)   f' = 1 - h^2
//   identity  f = z                                                               f' = 1
//   relu      f = max(z, 0)                                                       f' = [h > 0]
//   sigmoid   f = 1 / (1 + e^-z)  (2 ulp)                                         f' = h (1 - h)
//   softplus  f = z > 20 ? z : log1p(e^z)   (nn.Softplus defaults)                f' = -expm1(-h)  (= sigmoid(z))
//
// A narrower network is the 64-wide one with zero pads (models/actor_critic.py, ParamMap): a pad unit has z = +0.  tanh,
// identity and relu map it to +0; sigmoid and softplus do not, so for them a unit at or past its layer's real width
// outputs +0.  Every derivative above is then 0 at a pad (and the gradient reaching a pad is +-0 anyway), so gradients,
// Adam moments and Fisher-vector products stay +0 there.  The Fisher tangent pass needs f' only: the f'' terms of the
// double backward multiply dKL/dmu, which is 0 at p = q.
//
// Kernels take the activation as a template parameter ACT: one of the five codes, or ACT_MIXED in the kernels that run
// the actor and the critics in one launch with different activations, where the code of the CTA's network is read from
// the NetSpec at run time.  With a fixed ACT the unused branches fold away: the tanh instantiation is the tanh code.
#pragma once
#include <type_traits>

#include "common.cuh"

namespace osb {

// The codes of include/omnisafe_b200.h (OSB_ACT_*).
enum : int { ACT_TANH = 0, ACT_IDENTITY = 1, ACT_RELU = 2, ACT_SIGMOID = 3, ACT_SOFTPLUS = 4, ACT_MIXED = 5 };

// Activation and real hidden widths of the actor (index 0) and of both critics (index 1), as osb_set_net_spec set them.
struct NetSpec {
    int act[2];
    int width[2][2];
};

// The spec the next launches use (tanh, 64 wide unless osb_set_net_spec changed it).
const NetSpec& net_spec();

// The ACT a launch over the networks in net_mask (bit 0 actor, bits 1-2 critics) instantiates.
inline int launch_act(const NetSpec& s, int net_mask) {
    const bool actor = net_mask & 1, critic = net_mask & 6;
    if (actor && critic && s.act[0] != s.act[1]) return ACT_MIXED;
    return actor ? s.act[0] : s.act[1];
}

// f(std::integral_constant<int, ACT>{}) for the run-time code `act`; MIX = false: the launch runs one network, and
// ACT_MIXED is not instantiated.
template <bool MIX, class F>
inline int with_act(int act, F&& f) {
    switch (act) {
        case ACT_IDENTITY: return f(std::integral_constant<int, ACT_IDENTITY>{});
        case ACT_RELU: return f(std::integral_constant<int, ACT_RELU>{});
        case ACT_SIGMOID: return f(std::integral_constant<int, ACT_SIGMOID>{});
        case ACT_SOFTPLUS: return f(std::integral_constant<int, ACT_SOFTPLUS>{});
        case ACT_MIXED:
            if constexpr (MIX) return f(std::integral_constant<int, ACT_MIXED>{});
        default: return f(std::integral_constant<int, ACT_TANH>{});
    }
}

struct TanhExact {
    __device__ __forceinline__ float operator()(float x) const { return tanhf(x); }
};

// The hidden activation of network `net` (0 actor, 1 / 2 critics) in a kernel instantiated for ACT; Tanh is the
// precision's tanh.  f(z, col, width) is the layer output of unit `col` of a layer `width` units wide.
template <int ACT, class Tanh = TanhExact>
struct Hidden {
    int code, w1, w2;
    // constant indices: a run-time index into the kernel-parameter struct would copy it to local memory
    __device__ __forceinline__ Hidden(const NetSpec& s, int net)
        : code(ACT == ACT_MIXED ? (net ? s.act[1] : s.act[0]) : ACT), w1(net ? s.width[1][0] : s.width[0][0]),
          w2(net ? s.width[1][1] : s.width[0][1]) {}

    __device__ __forceinline__ int kind() const { return ACT == ACT_MIXED ? code : ACT; }

    __device__ __forceinline__ float operator()(float z, int col, int width) const {
        const int a = kind();
        if (a == ACT_TANH) return Tanh{}(z);
        if (a == ACT_IDENTITY) return z;
        if (a == ACT_RELU) return z > 0.f ? z : 0.f;
        if (col >= width) return 0.f;
        // __fdividef: 2 ulp like x3::tanh_acc, and no out-of-line slow path (the IEEE division's would put a call
        // frame on the persistent kernels' stack); below z = -87 it returns 0 for sigmoid's < 2^-126
        if (a == ACT_SIGMOID) return __fdividef(1.f, 1.f + expf(-z));
        return z > 20.f ? z : log1pf(expf(z));
    }

    // f'(z) from h = f(z)
    __device__ __forceinline__ float d(float h) const {
        const int a = kind();
        if (a == ACT_TANH) return 1.f - h * h;
        if (a == ACT_IDENTITY) return 1.f;
        if (a == ACT_RELU) return h > 0.f ? 1.f : 0.f;
        if (a == ACT_SIGMOID) return h * (1.f - h);
        return -expm1f(-h);
    }
};

}  // namespace osb
