// optim.cuh — the per-element update rules of Neon's optimizers as the reference constructs them
// (src/deepqnetwork.py:50-61): RMSProp (default), Adam, Adadelta.  One device function, shared by every kernel
// that applies an update (k_optimizer, k_opt_conv, k_opt_fc1, the fused fc1 wgrad epilogue), written with
// explicit _rn intrinsics in Neon's operation order so that, given equal gradients, the result is bit-identical
// to the numpy oracle (oracle/dqn_oracle.py::rmsprop_update / adam_update / adadelta_update).
//
// Optimizer state lives in `planes` fp32 arrays shaped like the parameters (Neon's `states` list per layer):
//   RMSProp  [s]            Adam  [m, v]            Adadelta  [E[g^2], E[dx^2], dx]
#pragma once
#include "common.cuh"

namespace b200 {

struct OptArgs {
  int kind;              // B200DQN_OPT_*
  int nstates;           // 1 / 2 / 3
  float bsz;             // grad = dW / be.bsz  (world x per-rank minibatch)
  float lr, decay, one_m_decay, eps;          // RMSProp: lr, decay_rate, eps 1e-6;  Adadelta: decay, eps 1e-6
  float b1, one_m_b1, b2, one_m_b2, adam_eps; // Adam: beta_1 0.9, beta_2 0.999, eps 1e-8
  const float* adam_l;   // device scalar written by the head kernel every step:
                         //   l = lr * sqrt(1 - beta_2^t) / (1 - beta_1^t),  t = optimize() calls so far + 1
  int64_t plane;         // elements between consecutive state planes
};

#ifdef __CUDACC__
__device__ __forceinline__ float opt_step_scalar(const OptArgs& o) {
  return o.kind == B200DQN_OPT_ADAM ? __ldcg(o.adam_l) : 0.f;
}

// one parameter's rule from its gradient gg = g / bsz: w = weight, s0..s2 = its state planes (unused ones untouched)
__device__ __forceinline__ void opt_rule1(const OptArgs& o, float l, float gg, float& w, float& s0, float& s1,
                                          float& s2) {
  if (o.kind == B200DQN_OPT_RMSPROP) {
    // state = decay*state + square(grad)*(1-decay);  param = param - (grad*lrate) / (sqrt(state+eps) + eps)
    const float ns = __fadd_rn(__fmul_rn(o.decay, s0), __fmul_rn(__fmul_rn(gg, gg), o.one_m_decay));
    const float den = __fadd_rn(__fsqrt_rn(__fadd_rn(ns, o.eps)), o.eps);
    w = __fsub_rn(w, __fdiv_rn(__fmul_rn(gg, o.lr), den));
    s0 = ns;
  } else if (o.kind == B200DQN_OPT_ADAM) {
    // m = m*beta_1 + (1-beta_1)*grad;  v = v*beta_2 + (1-beta_2)*grad*grad;  param -= (l*m) / (sqrt(v) + eps)
    const float m = __fadd_rn(__fmul_rn(s0, o.b1), __fmul_rn(o.one_m_b1, gg));
    const float v = __fadd_rn(__fmul_rn(s1, o.b2), __fmul_rn(__fmul_rn(o.one_m_b2, gg), gg));
    w = __fsub_rn(w, __fdiv_rn(__fmul_rn(l, m), __fadd_rn(__fsqrt_rn(v), o.adam_eps)));
    s0 = m;
    s1 = v;
  } else {
    // s0 = s0*decay + (1-decay)*g*g;  s2 = sqrt((s1+eps)/(s0+eps))*g;  s1 = s1*decay + (1-decay)*s2*s2;  param -= s2
    const float n0 = __fadd_rn(__fmul_rn(s0, o.decay), __fmul_rn(__fmul_rn(o.one_m_decay, gg), gg));
    const float dx = __fmul_rn(__fsqrt_rn(__fdiv_rn(__fadd_rn(s1, o.eps), __fadd_rn(n0, o.eps))), gg);
    const float n1 = __fadd_rn(__fmul_rn(s1, o.decay), __fmul_rn(__fmul_rn(o.one_m_decay, dx), dx));
    w = __fsub_rn(w, dx);
    s0 = n0;
    s1 = n1;
    s2 = dx;
  }
}

// one parameter: g = raw summed gradient, w = weight, s0..s2 = its state planes (unused ones untouched)
__device__ __forceinline__ void opt_update1(const OptArgs& o, float l, float g, float& w, float& s0, float& s1,
                                            float& s2) {
  opt_rule1(o, l, __fdiv_rn(g, o.bsz), w, s0, s1, s2);
}

// the same under global gradient-norm clipping (b200dqn_net_config::max_grad_norm): gg' = fl(fl(g / bsz) c), c the
// step's clip coefficient c32
__device__ __forceinline__ void opt_update1_clip(const OptArgs& o, float l, float g, float c, float& w, float& s0,
                                                 float& s1, float& s2) {
  opt_rule1(o, l, __fmul_rn(__fdiv_rn(g, o.bsz), c), w, s0, s1, s2);
}

// N consecutive parameters at element offset i: load the live state planes, update, store.  kClip: the clipped rule
// (opt_update1_clip) with coefficient c.
template <int N, bool kClip = false>
__device__ __forceinline__ void opt_update_vec(const OptArgs& o, float l, const float* g, float* w_out, float* w_ptr,
                                               float* s_ptr, float c = 1.f) {
  static_assert(N == 4 || N == 8, "vector width");
  float sv[3][N];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    if (k < o.nstates) {
#pragma unroll
      for (int v = 0; v < N / 4; ++v) {
        const float4 t = *reinterpret_cast<const float4*>(s_ptr + k * o.plane + 4 * v);
        sv[k][4 * v] = t.x; sv[k][4 * v + 1] = t.y; sv[k][4 * v + 2] = t.z; sv[k][4 * v + 3] = t.w;
      }
    } else {
#pragma unroll
      for (int j = 0; j < N; ++j) sv[k][j] = 0.f;
    }
  }
#pragma unroll
  for (int v = 0; v < N / 4; ++v) {
    const float4 t = *reinterpret_cast<const float4*>(w_ptr + 4 * v);
    w_out[4 * v] = t.x; w_out[4 * v + 1] = t.y; w_out[4 * v + 2] = t.z; w_out[4 * v + 3] = t.w;
  }
#pragma unroll
  for (int j = 0; j < N; ++j) {
    if constexpr (kClip) opt_update1_clip(o, l, g[j], c, w_out[j], sv[0][j], sv[1][j], sv[2][j]);
    else opt_update1(o, l, g[j], w_out[j], sv[0][j], sv[1][j], sv[2][j]);
  }
#pragma unroll
  for (int v = 0; v < N / 4; ++v)
    *reinterpret_cast<float4*>(w_ptr + 4 * v) = make_float4(w_out[4 * v], w_out[4 * v + 1], w_out[4 * v + 2], w_out[4 * v + 3]);
#pragma unroll
  for (int k = 0; k < 3; ++k)
    if (k < o.nstates) {
#pragma unroll
      for (int v = 0; v < N / 4; ++v)
        *reinterpret_cast<float4*>(s_ptr + k * o.plane + 4 * v) =
            make_float4(sv[k][4 * v], sv[k][4 * v + 1], sv[k][4 * v + 2], sv[k][4 * v + 3]);
    }
}

// soft target update of one weight (b200dqn_net_config::soft_target_tau): fl(fl(c tw) + fl(t w)), no contraction
__device__ __forceinline__ float soft_blend1(float tw, float w, float c, float t) {
  return __fadd_rn(__fmul_rn(c, tw), __fmul_rn(t, w));
}
#endif

}  // namespace b200
