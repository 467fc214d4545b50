// net.cu — Nature-DQN train / predict on the device behind DeepQNetwork's call surface
// (src/deepqnetwork.py:15-192 of the reference; per-entry citations in include/b200dqn.h).
#include <stdlib.h>

#include <cmath>
#include <new>
#include <type_traits>
#include <vector>

#include <cuda_fp16.h>

#include "net.cuh"
#include "net_umma.cuh"

namespace b200 {

// ------------------------------------------------------------------------------------------
// K2e + K3 + K4a/K5a ("head"): finish fc1 (sum split-K partials, Rectlin), run fc2 (Affine
// nout=A, no activation) for both networks of ONE sample per CTA, then — same CTA, no inter-CTA
// hand-off — the TD target / delta / cost / clip of src/deepqnetwork.py:124-159 and the fc2 backward:
//   dZ4[b][k] = (sum_a delta[b][a] W5[k][a]) * (H4[b][k] > 0),  dW5[k][a] = sum_b H4[b][k] delta[b][a].
// The reference forms the target on the host in Python floats (double) and stores it into a
// float32 array; we do the same arithmetic in fp64 and round once.  The per-sample cost
// 0.5*sum_a delta^2 (BEFORE the clip) goes to row_cost; the batch mean is formed off the critical
// chain by k_cost_finish.  grid = rows, block = 512 (one thread per hidden unit).
// kSlots = 3 (Double DQN, van Hasselt et al. 2016; nets = 3): slot 2 is the online network on the poststates.  Its Q row
// goes to q_online_post, and the target takes the target network's Q at the first index of that row's maximum (as
// np.argmax / torch.argmax) instead of the maximum of the target row.  kSlots = 2 serves every other forward.
// ------------------------------------------------------------------------------------------
struct HeadTrainArgs {
  int enable;
  const uint8_t* actions;
  const int64_t* rewards;
  const uint8_t* terminals;
  const int32_t* midx;
  double discount;
  double min_reward, max_reward;
  float clip;
  float* delta;       // [rows][A]
  const uint32_t* step;   // completed train steps (k_cost_finish increments it)
  float* row_cost;    // [rows]
  float* dz4;         // [rows][512]
  float* dw5_rows;    // [rows][512][A] per-row partials of dW5 (summed in row order by the optimizer)
  __half* dz4_hi;     // fp16 hi / scaled-lo planes of dZ4 for the tensor-core dgrad (nullptr in fp32 mode)
  int64_t dz4_lo_off;
  float* adam_l;      // Adam only: this step's scalar l = lr*sqrt(1-beta_2^t)/(1-beta_1^t) for the optimizer kernels
  float adam_lr;
  int num_actions;    // actions[] >= num_actions would index q / W5 out of bounds: flagged in err, clamped
  uint32_t* err;
  HeadPush push;      // data-parallel gather schedule: this CTA's dZ4 row goes straight to every rank (world = 0: off)
  // prioritized replay (nullptr: off, today's step): the sample's importance weight scales its cost and its clipped
  // delta; the TD error before the clip goes to td_err for the priority update
  const float* isw;
  float* td_err;
  // n-step returns (Hessel et al. 2018): N > 1 forms y = sum_{k<m} gamma^k clip(r[i+k]) (+ gamma^N Q^ when no terminal
  // in rewards/terminals[i .. i+N-1], m the first terminal) in fp64 without contraction; N <= 1 is today's one-step y
  int nstep;
};

// The TD scalars of sample b, shared by both heads.  They depend only on the sampler (several kernels upstream,
// complete by now), so the heads fetch them before the dependency wait, off the tail of the kernel.  Thread 0 gets the
// taken action a (clamped, out-of-range actions flagged in td.err), the reward r and the terminal flag; with kNstep it
// also gets the n-step return R, g = gamma^m and the flag "a terminal cut the window".  Thread 32 of CTA 0 writes
// Adam's step scalar.
template <bool kNstep>
__device__ __forceinline__ void head_td_scalars(const HeadTrainArgs& td, int b, int t, int& td_a, int64_t& td_r,
                                                int& td_term, double& td_ret, double& td_g) {
  if (td.enable && t == 0) {
    const int64_t mi = td.midx[b];
    td_a = td.actions[mi];
    td_r = td.rewards[mi];
    td_term = td.terminals[mi];
    if (td_a >= td.num_actions) {   // the reference would raise IndexError (deepqnetwork.py:141); here: sticky flag
      atomicExch(td.err, 1u);
      td_a = td.num_actions - 1;
    }
  }
  // n-step: lane k of warp 0 loads reward and terminal k (32 at a time), and every lane reduces them in k order through
  // shuffles: g = 1; for k: R = R + g c_k; stop at a terminal; g = g gamma.  Thread 0 keeps R, g and the flag.
  if (kNstep && td.enable && t < 32) {
    const int64_t mi = td.midx[b];
    double R = 0.0, g = 1.0;
    bool term = false;
    for (int base = 0; base < td.nstep && !term; base += 32) {
      const int k = base + t;
      double c = 0.0;
      int tk = 0;
      if (k < td.nstep) {
        c = fmin(fmax(double(td.rewards[mi + k]), td.min_reward), td.max_reward);
        tk = td.terminals[mi + k];
      }
      const int m = min(32, td.nstep - base);
      for (int j = 0; j < m; ++j) {
        const double cj = __shfl_sync(0xffffffffu, c, j);
        const int tj = __shfl_sync(0xffffffffu, tk, j);
        R = __dadd_rn(R, __dmul_rn(g, cj));
        if (tj) {
          term = true;
          break;
        }
        g = __dmul_rn(g, td.discount);
      }
    }
    if (t == 0) {
      td_ret = R;
      td_g = g;
      td_term = term ? 1 : 0;
    }
  }
  if (td.enable && td.adam_l && b == 0 && t == 32) {
    // Adam.optimize: self.t += 1;  l = lr * sqrt(1 - beta_2**t) / (1 - beta_1**t)  (Python doubles, fp32 tensor ops)
    const double tt = double(*td.step) + 1.0;
    const float a = float(1.0 - pow(0.999, tt)), c = float(1.0 - pow(0.9, tt));
    *td.adam_l = __fdiv_rn(__fmul_rn(td.adam_lr, __fsqrt_rn(a)), c);
  }
}

template <int kSlots, bool kNstep>
__global__ void __launch_bounds__(kHidden)
k_head(const float* __restrict__ part, int splits, int rows, int nets, float* h4_online, float* h4_target,
       const float* __restrict__ w5_online, const float* __restrict__ w5_target, float* q_online,
       float* q_target, float* q_online_post, int A, const HeadTrainArgs td, const KTrace kt) {
  static_assert(kSlots == 2 || kSlots == 3, "online + target, or Double DQN's three slots");
  // kNstep (td.nstep > 1): the n-step target; the one-step instantiation is today's kernel unchanged
  __shared__ float red[kSlots][kHidden / 32][kMaxActions];
  __shared__ float s_q[kSlots][kMaxActions];
  __shared__ float s_d;
  __shared__ int s_a;
  __shared__ __align__(16) __half s_row[2][kHidden];   // hi / lo of this sample's dZ4 row (peer push)
  const int b = blockIdx.x, t = threadIdx.x;
  kt_begin(kt);
  int td_a = 0, td_term = 0;
  int64_t td_r = 0;
  double td_ret = 0.0, td_g = 1.0;
  head_td_scalars<kNstep>(td, b, t, td_a, td_r, td_term, td_ret, td_g);
  pdl_wait();
  pdl_launch_dependents();
  float h[kSlots] = {};
#pragma unroll
  for (int z = 0; z < kSlots; ++z) {
    if (z < nets) {
      float acc = 0.f;
      for (int s = 0; s < splits; ++s) acc += part[((z * splits + s) * rows + b) * kHidden + t];
      h[z] = fmaxf(acc, 0.f);
      if (z < 2) (z ? h4_target : h4_online)[b * kHidden + t] = h[z];   // slot 2's H4 has no reader
    }
  }
#pragma unroll
  for (int z = 0; z < kSlots; ++z) {
    if (z < nets) {
      const float* w5 = z == 1 ? w5_target : w5_online;
      for (int a = 0; a < A; ++a) {
        float v = h[z] * w5[t * A + a];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((t & 31) == 0) red[z][t >> 5][a] = v;
      }
    }
  }
  __syncthreads();
  if (t < nets * A) {
    const int z = t / A, a = t % A;
    float v = 0.f;
#pragma unroll
    for (int wI = 0; wI < kHidden / 32; ++wI) v += red[z][wI][a];
    (z == 0 ? q_online : (kSlots == 3 && z == 2) ? q_online_post : q_target)[b * A + a] = v;
    s_q[z][a] = v;
  }
  if (!td.enable) {
    kt_end(kt);
    return;
  }
  __syncthreads();
  if (t == 0) {
    const int a = td_a;
    // np.clip (:136) with float bounds (main.py:43-44): maximum with the lower bound, then minimum with the upper
    // one, so crossed bounds give the upper bound.  For bounds that are exact doubles this is numpy's int64 clamp.
    const double rr = fmin(fmax(double(td_r), td.min_reward), td.max_reward);
    float maxq;
    if constexpr (kSlots == 3) {   // Double DQN: a* = argmax_a Q_online(s', a), valued by the target network
      int best = 0;
      for (int j = 1; j < A; ++j)
        if (s_q[2][j] > s_q[2][best]) best = j;
      maxq = s_q[1][best];
    } else {
      maxq = s_q[1][0];
      for (int j = 1; j < A; ++j) maxq = fmaxf(maxq, s_q[1][j]);                          // be.max(postq) (:124)
    }
    double y;
    if constexpr (kNstep) y = td_term ? td_ret : __dadd_rn(td_ret, __dmul_rn(td_g, double(maxq)));
    else y = td_term ? rr : rr + td.discount * double(maxq);                                // :140-143
    const float target = static_cast<float>(y);
    float d = s_q[0][a] - target;                                                         // SumSquared grad (:149)
    if (td.isw) {                                                                         // prioritized replay
      const float wb = td.isw[b];
      td.td_err[b] = d;
      td.row_cost[b] = wb * (0.5f * d * d);
      if (td.clip > 0.f) d = fminf(fmaxf(d, -td.clip), td.clip);
      d = d * wb;
    } else {
      td.row_cost[b] = 0.5f * d * d;                                                      // :154, before the clip
      if (td.clip > 0.f) d = fminf(fmaxf(d, -td.clip), td.clip);                          // :158-159
    }
    for (int j = 0; j < A; ++j) td.delta[b * A + j] = (j == a) ? d : 0.f;
    s_d = d;
    s_a = a;
  }
  __syncthreads();
  {
    const float d = s_d;
    const int a = s_a;
    const float hv = h[0];
    const float o = hv > 0.f ? d * w5_online[t * A + a] : 0.f;      // delta is non-zero only at the taken action
    td.dz4[b * kHidden + t] = o;
    if (td.dz4_hi) {
      const __half hh = __float2half_rn(o);
      const __half ll = __float2half_rn((o - __half2float(hh)) * 2048.0f);
      td.dz4_hi[b * kHidden + t] = hh;
      td.dz4_hi[td.dz4_lo_off + b * kHidden + t] = ll;
      s_row[0][t] = hh;
      s_row[1][t] = ll;
    }
    float* dw = td.dw5_rows + (int64_t(b) * kHidden + t) * A;        // per-row partial, summed by the optimizer
    for (int j = 0; j < A; ++j) dw[j] = (j == a) ? hv * d : 0.f;
  }
  if (td.push.world > 0) {
    // this sample's dZ4 row (1 KB per plane) to every rank's gather area, 16 bytes per store, then one counted
    // arrival per peer: the peers' fc1_wgrad over the global minibatch needs nothing else from this rank
    __syncthreads();
    const HeadPush& hp = td.push;
    if (t < 2 * (kHidden / 8)) {
      const int pl = t / (kHidden / 8), c = t % (kHidden / 8);
      const uint4 v = reinterpret_cast<const uint4*>(s_row[pl])[c];
      const int64_t par = int64_t((*reinterpret_cast<const volatile uint32_t*>(hp.epoch) + 1u) & 1u) * hp.parity16;
      const int64_t at = par + pl * hp.lo16 + (int64_t(hp.rank) * hp.rows + b) * (kHidden / 8) + c;
#pragma unroll
      for (int p = 0; p < kXMaxWorld; ++p)
        if (p < hp.world) hp.gat[p][at] = v;
    }
    __syncthreads();
    if (t < hp.world) {
      asm volatile("fence.acq_rel.sys;" ::: "memory");   // the CTA's stores (observed through the barrier) first
      asm volatile("red.release.sys.global.add.u32 [%0], 1;" ::"l"(hp.cnt[t] + hp.rank) : "memory");
    }
  }
  kt_end(kt);
}

// ------------------------------------------------------------------------------------------
// Dueling head (Wang et al. 2016; b200dqn.h has the rules): k_head's job on a dueling net.  One CTA of 1024 threads per
// sample, thread t = fc1 unit t: warps 0..15 hold the advantage units, warps 16..31 the value units.  Per slot,
// A_a = fc2 column a over the advantage units and V = column A over the value units, each as k_head forms Q (fp32
// products, xor butterfly, the 16 warp sums in warp order); m = (sum_j A_j in j order) / A; Q_a = V + (A_a - m).  With
// td.enable the TD step of k_head follows on these Q, then the backward: g = delta / A, dA_j = (j == a ? delta - g :
// -g), dV = delta; dZ4 = (sum_j dA_j W5[k][j], j order) on advantage unit k and delta W5[k][A] on value unit k, both
// under the H4 mask; the dW5 row partial is H4[k] dA_j (column j < A) and H4[512 + k] delta (column A).  Every
// operation is rounded on its own (explicit _rn intrinsics).
// ------------------------------------------------------------------------------------------
template <int kSlots, bool kNstep>
__global__ void __launch_bounds__(kDuelHidden)
k_head_duel(const float* __restrict__ part, int splits, int rows, int nets, int ld, float* h4_online, float* h4_target,
            const float* __restrict__ w5_online, const float* __restrict__ w5_target, float* q_online,
            float* q_target, float* q_online_post, float* va, int A, const HeadTrainArgs td, const KTrace kt) {
  static_assert(kSlots == 2 || kSlots == 3, "online + target, or Double DQN's three slots");
  constexpr int kWarps = kHidden / 32;   // warps per stream
  __shared__ float red[kSlots][2][kWarps][kMaxActions];   // [stream 0: advantages, 1: value][warp][column]
  __shared__ float s_va[kSlots][kMaxActions + 1];
  __shared__ float s_m[kSlots];
  __shared__ float s_q[kSlots][kMaxActions];
  __shared__ float s_d;
  __shared__ int s_a;
  const int b = blockIdx.x, t = threadIdx.x, C = A + 1;
  const bool value = t >= kHidden;
  const int k = value ? t - kHidden : t, w = k >> 5;
  kt_begin(kt);
  int td_a = 0, td_term = 0;
  int64_t td_r = 0;
  double td_ret = 0.0, td_g = 1.0;
  head_td_scalars<kNstep>(td, b, t, td_a, td_r, td_term, td_ret, td_g);
  pdl_wait();
  pdl_launch_dependents();
  float h[kSlots] = {};
#pragma unroll
  for (int z = 0; z < kSlots; ++z) {
    if (z < nets) {
      float acc = 0.f;
      for (int s = 0; s < splits; ++s) acc = __fadd_rn(acc, part[((z * splits + s) * rows + b) * kDuelHidden + t]);
      h[z] = fmaxf(acc, 0.f);
      if (z < 2) (z ? h4_target : h4_online)[b * kDuelHidden + t] = h[z];
    }
  }
#pragma unroll
  for (int z = 0; z < kSlots; ++z) {
    if (z < nets) {
      const float* w5 = (z == 1 ? w5_target : w5_online) + k * C;
      for (int a = value ? A : 0; a < (value ? C : A); ++a) {   // warp-uniform: a whole warp is one stream
        float v = __fmul_rn(h[z], w5[a]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
        if ((t & 31) == 0) red[z][value][w][value ? 0 : a] = v;
      }
    }
  }
  __syncthreads();
  if (t < nets * C) {
    const int z = t / C, a = t % C, sv = a == A;
    float v = 0.f;
#pragma unroll
    for (int wI = 0; wI < kWarps; ++wI) v = __fadd_rn(v, red[z][sv][wI][sv ? 0 : a]);
    s_va[z][a] = v;
    va[(int64_t(z) * ld + b) * C + a] = v;
  }
  __syncthreads();
  if (t < nets) {
    float s = 0.f;
    for (int j = 0; j < A; ++j) s = __fadd_rn(s, s_va[t][j]);
    s_m[t] = __fdiv_rn(s, float(A));
  }
  __syncthreads();
  if (t < nets * A) {
    const int z = t / A, a = t % A;
    const float q = __fadd_rn(s_va[z][A], __fsub_rn(s_va[z][a], s_m[z]));
    (z == 0 ? q_online : (kSlots == 3 && z == 2) ? q_online_post : q_target)[b * A + a] = q;
    s_q[z][a] = q;
  }
  if (!td.enable) {
    kt_end(kt);
    return;
  }
  __syncthreads();
  if (t == 0) {   // k_head's TD step, line for line, on the dueling Q (a shared helper changed k_head<3, false>'s SASS)
    const int a = td_a;
    const double rr = fmin(fmax(double(td_r), td.min_reward), td.max_reward);
    float maxq;
    if constexpr (kSlots == 3) {
      int best = 0;
      for (int j = 1; j < A; ++j)
        if (s_q[2][j] > s_q[2][best]) best = j;
      maxq = s_q[1][best];
    } else {
      maxq = s_q[1][0];
      for (int j = 1; j < A; ++j) maxq = fmaxf(maxq, s_q[1][j]);
    }
    double y;
    if constexpr (kNstep) y = td_term ? td_ret : __dadd_rn(td_ret, __dmul_rn(td_g, double(maxq)));
    else y = td_term ? rr : rr + td.discount * double(maxq);
    const float target = static_cast<float>(y);
    float d = s_q[0][a] - target;
    if (td.isw) {
      const float wb = td.isw[b];
      td.td_err[b] = d;
      td.row_cost[b] = wb * (0.5f * d * d);
      if (td.clip > 0.f) d = fminf(fmaxf(d, -td.clip), td.clip);
      d = d * wb;
    } else {
      td.row_cost[b] = 0.5f * d * d;
      if (td.clip > 0.f) d = fminf(fmaxf(d, -td.clip), td.clip);
    }
    for (int j = 0; j < A; ++j) td.delta[b * A + j] = (j == a) ? d : 0.f;
    s_d = d;
    s_a = a;
  }
  __syncthreads();
  const float d = s_d, g = __fdiv_rn(d, float(A)), hv = h[0];
  const int a = s_a;
  const float* w5 = w5_online + k * C;
  float* dw = td.dw5_rows + (int64_t(b) * kHidden + k) * C;   // per-row partial, summed by the optimizer
  float o;
  if (value) {
    o = __fmul_rn(d, w5[A]);
    dw[A] = __fmul_rn(hv, d);
  } else {
    o = 0.f;
    for (int j = 0; j < A; ++j) {
      const float dA = j == a ? __fsub_rn(d, g) : -g;
      o = __fadd_rn(o, __fmul_rn(dA, w5[j]));
      dw[j] = __fmul_rn(hv, dA);
    }
  }
  o = hv > 0.f ? o : 0.f;
  td.dz4[b * kDuelHidden + t] = o;
  if (td.dz4_hi) {   // the tensor-core dgrad / wgrad operand: hi and scaled lo fp16 planes, as k_head writes them
    const __half hh = __float2half_rn(o);
    td.dz4_hi[b * kDuelHidden + t] = hh;
    td.dz4_hi[td.dz4_lo_off + b * kDuelHidden + t] = __float2half_rn((o - __half2float(hh)) * 2048.0f);
  }
  kt_end(kt);
}

// ------------------------------------------------------------------------------------------
// Munchausen head (M-DQN, Vieillard, Pietquin and Geist 2020; b200dqn.h has the rules): k_head's job with the Munchausen
// target.  kSlots = 3: slot 2 is the target network on the prestates, whose fc1 partials the one-slot pass of
// train_step wrote; its fc2 takes the target W5 and its Q row goes to q_target_pre.  kSlots = 2 (target_steps = 0):
// slot 0's Q row is the prestate row of the policy.  Lane j < A of warp 0 forms e_j of both rows; every lane of the warp
// then forms the j-order sums and the logs (shuffles in j order: the operations of one serial loop, done redundantly),
// lane j the term of action j, and the j-order sum of the terms; thread 0 forms y and runs k_head's TD step and backward
// from target = float(y) on, line for line (a shared helper changed pinned SASS in the earlier heads).
// ------------------------------------------------------------------------------------------
struct MdqnArgs {
  double alpha, tau, clip;   // alpha, tau and l0 of b200dqn.h
  float* q_target_pre;       // [rows][A] Q row of slot 2 (kSlots = 3)
  float* targets;            // [rows] float(y)
};

template <int kSlots, bool kNstep>
__global__ void __launch_bounds__(kHidden)
k_head_mdqn(const float* __restrict__ part, int splits, int rows, float* h4_online, float* h4_target,
            const float* __restrict__ w5_online, const float* __restrict__ w5_target, float* q_online,
            float* q_target, int A, const MdqnArgs ma, const HeadTrainArgs td, const KTrace kt) {
  static_assert(kSlots == 2 || kSlots == 3, "online + target, and the target network on the prestates");
  __shared__ float red[kSlots][kHidden / 32][kMaxActions];
  __shared__ float s_q[kSlots][kMaxActions];
  __shared__ float s_d;
  __shared__ int s_a;
  const int b = blockIdx.x, t = threadIdx.x;
  kt_begin(kt);
  int td_a = 0, td_term = 0;
  int64_t td_r = 0;
  double td_ret = 0.0, td_g = 1.0;
  head_td_scalars<kNstep>(td, b, t, td_a, td_r, td_term, td_ret, td_g);
  pdl_wait();
  pdl_launch_dependents();
  float h[kSlots] = {};
#pragma unroll
  for (int z = 0; z < kSlots; ++z) {
    float acc = 0.f;
    for (int s = 0; s < splits; ++s) acc += part[((z * splits + s) * rows + b) * kHidden + t];
    h[z] = fmaxf(acc, 0.f);
    if (z < 2) (z ? h4_target : h4_online)[b * kHidden + t] = h[z];   // slot 2's H4 has no reader
  }
#pragma unroll
  for (int z = 0; z < kSlots; ++z) {
    const float* w5 = z == 0 ? w5_online : w5_target;
    for (int a = 0; a < A; ++a) {
      float v = h[z] * w5[t * A + a];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if ((t & 31) == 0) red[z][t >> 5][a] = v;
    }
  }
  __syncthreads();
  if (t < kSlots * A) {
    const int z = t / A, a = t % A;
    float v = 0.f;
#pragma unroll
    for (int wI = 0; wI < kHidden / 32; ++wI) v += red[z][wI][a];
    (z == 0 ? q_online : z == 2 ? ma.q_target_pre : q_target)[b * A + a] = v;
    s_q[z][a] = v;
  }
  __syncthreads();
  if (t < 32) {
    const float* qpre = s_q[kSlots == 3 ? 2 : 0];
    const bool live = t < A;
    const float xo = live ? s_q[1][t] : -INFINITY, xp = live ? qpre[t] : -INFINITY;   // poststate / prestate rows
    float mo = xo, mp = xp;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mo = fmaxf(mo, __shfl_xor_sync(0xffffffffu, mo, o));
      mp = fmaxf(mp, __shfl_xor_sync(0xffffffffu, mp, o));
    }
    const double tau = ma.tau;
    const double eo = live ? exp(__ddiv_rn(__dsub_rn(double(xo), double(mo)), tau)) : 0.0;
    const double ep = live ? exp(__ddiv_rn(__dsub_rn(double(xp), double(mp)), tau)) : 0.0;
    double so = 0.0, sp = 0.0;
    for (int j = 0; j < A; ++j) {
      so = __dadd_rn(so, __shfl_sync(0xffffffffu, eo, j));
      sp = __dadd_rn(sp, __shfl_sync(0xffffffffu, ep, j));
    }
    const double lseo = __dadd_rn(double(mo), __dmul_rn(tau, log(so)));
    const double lsep = __dadd_rn(double(mp), __dmul_rn(tau, log(sp)));
    // lane j: pi_post,j (x_post,j - tau ln pi_post,j)
    const double term = live ? __dmul_rn(__ddiv_rn(eo, so), __dsub_rn(double(xo), __dsub_rn(double(xo), lseo))) : 0.0;
    double next = 0.0;
    for (int j = 0; j < A; ++j) next = __dadd_rn(next, __shfl_sync(0xffffffffu, term, j));
    if (t == 0) {
      const int a = td_a;
      const double rr = fmin(fmax(double(td_r), td.min_reward), td.max_reward);
      const double bonus = __dmul_rn(ma.alpha, fmin(fmax(__dsub_rn(double(qpre[a]), lsep), ma.clip), 0.0));
      double y;
      if constexpr (kNstep) {
        const double rb = __dadd_rn(td_ret, bonus);
        y = td_term ? rb : __dadd_rn(rb, __dmul_rn(td_g, next));
      } else {
        const double rb = __dadd_rn(rr, bonus);
        y = td_term ? rb : rb + td.discount * next;   // as k_head's one-step target
      }
      const float target = static_cast<float>(y);
      ma.targets[b] = target;
      float d = s_q[0][a] - target;
      if (td.isw) {
        const float wb = td.isw[b];
        td.td_err[b] = d;
        td.row_cost[b] = wb * (0.5f * d * d);
        if (td.clip > 0.f) d = fminf(fmaxf(d, -td.clip), td.clip);
        d = d * wb;
      } else {
        td.row_cost[b] = 0.5f * d * d;
        if (td.clip > 0.f) d = fminf(fmaxf(d, -td.clip), td.clip);
      }
      for (int j = 0; j < A; ++j) td.delta[b * A + j] = (j == a) ? d : 0.f;
      s_d = d;
      s_a = a;
    }
  }
  __syncthreads();
  {
    const float d = s_d;
    const int a = s_a;
    const float hv = h[0];
    const float o = hv > 0.f ? d * w5_online[t * A + a] : 0.f;
    td.dz4[b * kHidden + t] = o;
    if (td.dz4_hi) {
      const __half hh = __float2half_rn(o);
      const __half ll = __float2half_rn((o - __half2float(hh)) * 2048.0f);
      td.dz4_hi[b * kHidden + t] = hh;
      td.dz4_hi[td.dz4_lo_off + b * kHidden + t] = ll;
    }
    float* dw = td.dw5_rows + (int64_t(b) * kHidden + t) * A;
    for (int j = 0; j < A; ++j) dw[j] = (j == a) ? hv * d : 0.f;
  }
  kt_end(kt);
}

// cost = mean over the batch of the per-sample costs (GeneralizedCost.get_cost, src/deepqnetwork.py:154), summed in
// row order by one thread (deterministic); advances the cost ring and the step counter.  Runs off the critical
// chain (the stream of the fc2 optimizer): nothing on the device waits for the scalar.
__global__ void __launch_bounds__(256)
k_cost_finish(const float* __restrict__ row_cost, int rows, float* cost_ring, uint32_t* step,
              volatile uint32_t* host_res, const uint32_t* __restrict__ sampler_words, volatile uint32_t* host_words,
              const KTrace kt) {
  __shared__ float s_c[1024];
  kt_begin(kt);
  float tot = 0.f;
  for (int base = 0; base < rows; base += 1024) {
    const int n = min(1024, rows - base);
    for (int i = threadIdx.x; i < n; i += blockDim.x) s_c[i] = row_cost[base + i];
    __syncthreads();
    if (threadIdx.x == 0)
      for (int i = 0; i < n; ++i) tot += s_c[i];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const uint32_t sidx = *step;
    const float cost = tot / float(rows);
    cost_ring[sidx % kCostRing] = cost;
    cost_ring[kCostRing] = cost;   // "latest" slot
    *step = sidx + 1;
    if (host_res) {                // the host polls [0]: data first, system fence, then the sequence number
      host_res[4 + sidx % kHostCosts] = __float_as_uint(cost);
      host_res[1] = __float_as_uint(cost_ring[kCostRing + 1]);   // action-range flag word
      if (sampler_words) {         // this step's index draw: words consumed, for the host's lock-step `random`
        host_words[1] = sampler_words[0];
        host_words[2] = sampler_words[1];
        host_words[3] = sampler_words[3];   // sticky error of the prioritized sampler
      }
      __threadfence_system();
      if (sampler_words) host_words[0] = sampler_words[2];
      host_res[0] = sidx + 1;
    }
  }
  kt_end(kt);
}

// Small-layer optimizer without tile images (fc2: 512 x A parameters, CUDA-core layer): 8 lanes per float4 sum the
// split partials (lane l takes partials l, l+8, ... in order; fixed xor tree across lanes — the summation order of
// k_optimizer, bit-identical) and lane 0 applies the configured update.
__global__ void __launch_bounds__(256)
k_opt_small(const float* __restrict__ part, int splits, int64_t size, float* __restrict__ w, float* __restrict__ sst,
            const OptArgs opt, const KTrace kt) {
  kt_begin(kt);
  pdl_wait();
  pdl_launch_dependents();
  const int tid = threadIdx.x, lane8 = tid & 7;
  const int64_t i = (int64_t(blockIdx.x) * 32 + (tid >> 3)) * 4;
  const bool live = i < size;
  float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
  if (live) {
    const float* p = part + i;
#pragma unroll 4
    for (int sp = lane8; sp < splits; sp += 8) {
      const float4 v = *reinterpret_cast<const float4*>(p + int64_t(sp) * size);
      g.x += v.x; g.y += v.y; g.z += v.z; g.w += v.w;
    }
  }
#pragma unroll
  for (int o = 1; o < 8; o <<= 1) {
    g.x += __shfl_xor_sync(0xffffffffu, g.x, o);
    g.y += __shfl_xor_sync(0xffffffffu, g.y, o);
    g.z += __shfl_xor_sync(0xffffffffu, g.z, o);
    g.w += __shfl_xor_sync(0xffffffffu, g.w, o);
  }
  if (live && lane8 == 0) {
    float nw[4];
    opt_update_vec<4>(opt, opt_step_scalar(opt), reinterpret_cast<const float*>(&g), nw, w + i, sst + i);
  }
  kt_end(kt);
}

// ------------------------------------------------------------------------------------------
// Distributional head (C51, Bellemare, Dabney and Munos 2017; b200dqn.h has the rules).  Three kernels:
//   k_fc2_dist       fc1 finish + fc2 for every slot: l[z][b][c] = sum_k H4[z][b][k] W5[k][c], c = a * atoms + i
//   k_head_dist      one CTA per sample: softmax, Q, a*, projection, cross-entropy, logit gradient, dZ4 (+ fp16
//                    planes) and the compact dW5 row partial [512][atoms] of the taken action
//   k_opt_fc2_dist   fc2's gradient from those partials (rows with the action, row order) + the configured update
// ------------------------------------------------------------------------------------------
struct DistArgs {
  int atoms;
  double v_min, v_max, dz;
  float* probs;      // [3][ld][A][atoms]
  float* tdist;      // [ld][atoms]
  float* lgrad;      // [ld][atoms]
  int32_t* act_rows; // [ld]
};

constexpr int kDistTB = 16, kDistTN = 64;   // k_fc2_dist tile: samples x output columns, 256 threads

// grid (sample tiles, column tiles, slots).  Each CTA finishes fc1 for its 16 samples (split-K partials summed in
// k_head's order, then Rectlin: H4 is bit-identical to the scalar head's) into shared memory, and then reads its W5
// column slice once for all of them.  Thread (c, group) accumulates 4 samples of column c in k order, fp32, without
// contraction.  The CTAs of column tile 0 store H4 of slots 0 and 1.
__global__ void __launch_bounds__(256)
k_fc2_dist(const float* __restrict__ part, int splits, int rows, int ld, float* h4_online, float* h4_target,
           const float* __restrict__ w5_online, const float* __restrict__ w5_target, float* __restrict__ logits,
           int ncols, const KTrace kt) {
  __shared__ float s_h[kDistTB][kHidden];
  const int z = blockIdx.z, b0 = blockIdx.x * kDistTB, t = threadIdx.x;
  const int c = blockIdx.y * kDistTN + t % kDistTN, g0 = (t / kDistTN) * 4;
  const int nrow = min(kDistTB, rows - b0);
  const float* w5 = (z == 1 ? w5_target : w5_online) + c;
  kt_begin(kt);
  pdl_wait();
  pdl_launch_dependents();
  for (int e = t; e < kDistTB * kHidden; e += 256) {
    const int r = e / kHidden, k = e % kHidden;
    float h = 0.f;
    if (r < nrow) {
      float acc = 0.f;
      for (int s = 0; s < splits; ++s) acc += part[((z * splits + s) * rows + b0 + r) * kHidden + k];
      h = fmaxf(acc, 0.f);
      if (z < 2 && blockIdx.y == 0) (z ? h4_target : h4_online)[(b0 + r) * kHidden + k] = h;
    }
    s_h[r][k] = h;
  }
  __syncthreads();
  if (c < ncols) {
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 8
    for (int k = 0; k < kHidden; ++k) {
      const float w = w5[int64_t(k) * ncols];
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[j] = __fadd_rn(acc[j], __fmul_rn(s_h[g0 + j][k], w));
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (g0 + j < nrow) logits[(int64_t(z) * ld + b0 + g0 + j) * ncols + c] = acc[j];
  }
  kt_end(kt);
}

// One CTA (512 threads) per sample b.  Thread r < nets * A owns row (slot z, action a): max, e_i = expf(l_i - max),
// s = sum_i e_i, p_i = e_i / s, Q = sum_i zf_i p_i, all sequential in i.  With td.enable the rest of the step follows
// (b200dqn.h): a* = first maximum of slot 1's Q (slot 2's with kSlots = 3), the fp64 projection of p[1][a*] (one
// thread per atom, j order, no contraction), the loss, gl, dZ4 and the dW5 row partial dw[b][k][i] = H4[k] gl_i.
// The TD scalars and Adam's step scalar come from head_td_scalars, before the dependency wait.
template <int kSlots, bool kNstep>
__global__ void __launch_bounds__(kHidden)
k_head_dist(const float* __restrict__ logits, int ld, int nets, const float* __restrict__ h4_online,
            const float* __restrict__ w5_online, float* q_online, float* q_target, float* q_online_post, int A,
            const DistArgs da, const HeadTrainArgs td, const KTrace kt) {
  static_assert(kSlots == 1 || kSlots == 2 || kSlots == 3, "predict, online + target, or Double DQN's three slots");
  __shared__ float s_p[kSlots][kMaxActions * kMaxAtoms];
  __shared__ float s_q[kSlots][kMaxActions];
  __shared__ float s_mx[kMaxActions], s_ls[kMaxActions];   // slot 0: row maximum and log of the sum
  __shared__ double s_b[kMaxAtoms], s_qd[kMaxAtoms];
  __shared__ float s_zf[kMaxAtoms], s_m[kMaxAtoms], s_g[kMaxAtoms], s_h4[kHidden];
  __shared__ double s_ret, s_gam;
  __shared__ int s_a, s_astar;
  const int b = blockIdx.x, t = threadIdx.x, atoms = da.atoms, ncols = A * atoms;
  kt_begin(kt);
  int td_a = 0, td_term = 0;
  int64_t td_r = 0;
  double td_ret = 0.0, td_g = 1.0;
  head_td_scalars<kNstep>(td, b, t, td_a, td_r, td_term, td_ret, td_g);
  if (t < atoms) s_zf[t] = float(__dadd_rn(da.v_min, __dmul_rn(double(t), da.dz)));
  pdl_wait();
  pdl_launch_dependents();
  if (td.enable) s_h4[t] = h4_online[b * kHidden + t];
  __syncthreads();
  if (t < nets * A) {
    const int z = t / A, a = t % A;
    const float* l = logits + (int64_t(z) * ld + b) * ncols + a * atoms;
    float* p = s_p[z] + a * atoms;
    float mx = l[0];
    for (int i = 1; i < atoms; ++i) mx = fmaxf(mx, l[i]);
    float s = 0.f;
    for (int i = 0; i < atoms; ++i) {
      p[i] = expf(__fsub_rn(l[i], mx));
      s = __fadd_rn(s, p[i]);
    }
    float q = 0.f;
    float* gp = da.probs + ((int64_t(z) * ld + b) * A + a) * atoms;
    for (int i = 0; i < atoms; ++i) {
      p[i] = __fdiv_rn(p[i], s);
      gp[i] = p[i];
      q = __fadd_rn(q, __fmul_rn(s_zf[i], p[i]));
    }
    s_q[z][a] = q;
    (z == 0 ? q_online : z == 2 ? q_online_post : q_target)[b * A + a] = q;
    if (z == 0) {
      s_mx[a] = mx;
      s_ls[a] = logf(s);
    }
  }
  if constexpr (kSlots > 1) {
    if (!td.enable) {
      kt_end(kt);
      return;
    }
    __syncthreads();
    if (t == 0) {
      const float* qs = s_q[kSlots == 3 ? 2 : 1];
      int best = 0;
      for (int j = 1; j < A; ++j)
        if (qs[j] > qs[best]) best = j;
      double R, g;
      if constexpr (kNstep) {
        R = td_ret;
        g = td_term ? 0.0 : td_g;
      } else {
        R = fmin(fmax(double(td_r), td.min_reward), td.max_reward);   // np.clip as the scalar head
        g = td_term ? 0.0 : td.discount;
      }
      s_ret = R;
      s_gam = g;
      s_a = td_a;
      s_astar = best;
      da.act_rows[b] = td_a;
    }
    __syncthreads();
    const int a = s_a;
    if (t < atoms) {   // T_j = clamp(R + g z_j), b_j = (T_j - v_min) / dz; q_j = target network's p[a*][j]
      const double zj = __dadd_rn(da.v_min, __dmul_rn(double(t), da.dz));
      const double T = fmin(fmax(__dadd_rn(s_ret, __dmul_rn(s_gam, zj)), da.v_min), da.v_max);
      s_b[t] = __ddiv_rn(__dsub_rn(T, da.v_min), da.dz);
      s_qd[t] = double(s_p[1][s_astar * atoms + t]);
    }
    __syncthreads();
    if (t < atoms) {   // m_i = sum_j q_j max(0, 1 - |b_j - i|): the floor/ceil split in gather form
      double acc = 0.0;
      for (int j = 0; j < atoms; ++j) {
        const double hat = fmax(0.0, __dsub_rn(1.0, fabs(__dsub_rn(s_b[j], double(t)))));
        acc = __dadd_rn(acc, __dmul_rn(s_qd[j], hat));
      }
      const float m = float(acc);
      float gl = __fsub_rn(s_p[0][a * atoms + t], m);
      if (td.isw) gl = __fmul_rn(gl, td.isw[b]);
      s_m[t] = m;
      s_g[t] = gl;
      da.tdist[b * atoms + t] = m;
      da.lgrad[b * atoms + t] = gl;
    }
    __syncthreads();
    if (t == 0) {   // cross-entropy at the taken action: -sum_i m_i (l_i - max - log s), i order
      const float* l = logits + int64_t(b) * ncols + a * atoms;
      float acc = 0.f;
      for (int i = 0; i < atoms; ++i) acc = __fadd_rn(acc, __fmul_rn(s_m[i], __fsub_rn(__fsub_rn(l[i], s_mx[a]), s_ls[a])));
      const float loss = -acc;
      if (td.isw) {
        td.td_err[b] = loss;
        td.row_cost[b] = __fmul_rn(td.isw[b], loss);
      } else {
        td.row_cost[b] = loss;
      }
    }
    {
      const float hv = s_h4[t];
      const float* w = w5_online + int64_t(t) * ncols + a * atoms;
      float o = 0.f;
      if (hv > 0.f)
        for (int i = 0; i < atoms; ++i) o = __fadd_rn(o, __fmul_rn(w[i], s_g[i]));
      td.dz4[b * kHidden + t] = o;
      if (td.dz4_hi) {
        const __half hh = __float2half_rn(o);
        const __half ll = __float2half_rn((o - __half2float(hh)) * 2048.0f);
        td.dz4_hi[b * kHidden + t] = hh;
        td.dz4_hi[td.dz4_lo_off + b * kHidden + t] = ll;
      }
    }
    float* dw = td.dw5_rows + int64_t(b) * kHidden * atoms;
    for (int e = t; e < kHidden * atoms; e += kHidden) dw[e] = __fmul_rn(s_h4[e / atoms], s_g[e % atoms]);
  }
  kt_end(kt);
}

// fc2's gradient and update on a distributional net.  grid (cdiv(512 * atoms, 256), A): CTA (x, a) lists, in row
// order, the rows whose taken action is a (warp 0, by ballot), then thread e sums dw[row][e] over that list (0 for an
// action no row took) for parameter (k, a * atoms + i), e = k * atoms + i.  mode bit1: write the sum to g (d_g,
// internal layout); bit2: apply the configured update.
__global__ void __launch_bounds__(256)
k_opt_fc2_dist(const float* __restrict__ part, const int32_t* __restrict__ act_rows, int rows, int A, int atoms,
               float* __restrict__ g_out, float* __restrict__ w, float* __restrict__ sst, int mode, const OptArgs opt,
               const KTrace kt) {
  __shared__ int s_list[4096];
  __shared__ int s_n;
  const int a = blockIdx.y, t = threadIdx.x, e = blockIdx.x * 256 + t;
  kt_begin(kt);
  pdl_wait();
  pdl_launch_dependents();
  if (t < 32) {
    int cnt = 0;
    for (int base = 0; base < rows; base += 32) {
      const int r = base + t;
      const bool hit = r < rows && act_rows[r] == a;
      const unsigned m = __ballot_sync(0xffffffffu, hit);
      if (hit) s_list[cnt + __popc(m & ((1u << t) - 1u))] = r;
      cnt += __popc(m);
    }
    if (t == 0) s_n = cnt;
  }
  __syncthreads();
  if (e < kHidden * atoms) {
    const int64_t stride = int64_t(kHidden) * atoms;
    float g = 0.f;
    for (int j = 0; j < s_n; ++j) g = __fadd_rn(g, part[s_list[j] * stride + e]);
    const int64_t wi = int64_t(e / atoms) * A * atoms + a * atoms + e % atoms;
    if (mode & 2) g_out[wi] = g;
    if (mode & 4) {
      float s[3] = {0.f, 0.f, 0.f};
      for (int k = 0; k < opt.nstates; ++k) s[k] = sst[k * opt.plane + wi];
      float wv = w[wi];
      opt_update1(opt, opt_step_scalar(opt), g, wv, s[0], s[1], s[2]);
      w[wi] = wv;
      for (int k = 0; k < opt.nstates; ++k) sst[k * opt.plane + wi] = s[k];
    }
  }
  kt_end(kt);
}

// ------------------------------------------------------------------------------------------
// Quantile-regression head (QR-DQN, Dabney, Rowland, Bellemare and Munos 2018; b200dqn.h has the rules).  fc2's outputs
// theta[z][b][a * N + i] come from k_fc2_dist unchanged, and fc2's gradient goes through k_opt_fc2_dist unchanged with N
// as the block width; k_head_qr does the rest: Q, a*, the target quantiles, the quantile Huber loss and its gradient,
// dZ4 (+ fp16 planes) and the compact dW5 row partial [512][N] of the taken action.  No expf / logf: every stage is
// +, -, *, / and comparisons, each rounded on its own.
// ------------------------------------------------------------------------------------------
struct QrArgs {
  int nq;            // N
  float kappa;       // the Huber threshold (clip_error); 0: the pure quantile loss
  float* tq;         // [ld][N] target quantiles T_j
  float* qgrad;      // [ld][N] gradient on the taken action's quantiles
  int32_t* act_rows; // [ld]
};

// One CTA (512 threads) per sample b.  Thread r < nets * A owns row (slot z, action a): Q = (sum_i theta_i, i order) / N.
// With td.enable: thread 0 picks a* (first maximum of slot 1's Q, slot 2's with kSlots = 3) and the fp64 return; thread
// j < N forms T_j = float(R + g theta[1][a*][j]); thread i < N runs the j loop of the loss and the gradient for quantile
// i of the taken action; thread 0 sums the row loss; every thread its dZ4 element and a stride of the dW5 row partial.
// The TD scalars and Adam's step scalar come from head_td_scalars, before the dependency wait.
template <int kSlots, bool kNstep>
__global__ void __launch_bounds__(kHidden)
k_head_qr(const float* __restrict__ theta, int ld, int nets, const float* __restrict__ h4_online,
          const float* __restrict__ w5_online, float* q_online, float* q_target, float* q_online_post, int A,
          const QrArgs qa, const HeadTrainArgs td, const KTrace kt) {
  static_assert(kSlots == 1 || kSlots == 2 || kSlots == 3, "predict, online + target, or Double DQN's three slots");
  __shared__ float s_q[kSlots][kMaxActions];
  __shared__ float s_wlo[kMaxQuantiles], s_whi[kMaxQuantiles], s_t[kMaxQuantiles], s_l[kMaxQuantiles];
  __shared__ float s_g[kMaxQuantiles], s_h4[kHidden];
  __shared__ double s_ret, s_gam;
  __shared__ int s_a, s_astar;
  const int b = blockIdx.x, t = threadIdx.x, nq = qa.nq, ncols = A * nq;
  kt_begin(kt);
  int td_a = 0, td_term = 0;
  int64_t td_r = 0;
  double td_ret = 0.0, td_g = 1.0;
  head_td_scalars<kNstep>(td, b, t, td_a, td_r, td_term, td_ret, td_g);
  if (t < nq) {   // quantile midpoints tau_i = (2i + 1) / 2N in fp64: weight tau_i for u >= 0, 1 - tau_i for u < 0
    s_wlo[t] = float(__ddiv_rn(double(2 * t + 1), double(2 * nq)));
    s_whi[t] = float(__ddiv_rn(double(2 * nq - 2 * t - 1), double(2 * nq)));
  }
  pdl_wait();
  pdl_launch_dependents();
  if (td.enable) s_h4[t] = h4_online[b * kHidden + t];
  if (t < nets * A) {
    const int z = t / A, a = t % A;
    const float* th = theta + (int64_t(z) * ld + b) * ncols + a * nq;
    float s = 0.f;
    for (int i = 0; i < nq; ++i) s = __fadd_rn(s, th[i]);
    const float q = __fdiv_rn(s, float(nq));
    s_q[z][a] = q;
    (z == 0 ? q_online : z == 2 ? q_online_post : q_target)[b * A + a] = q;
  }
  if constexpr (kSlots > 1) {
    if (!td.enable) {
      kt_end(kt);
      return;
    }
    __syncthreads();
    if (t == 0) {
      const float* qs = s_q[kSlots == 3 ? 2 : 1];
      int best = 0;
      for (int j = 1; j < A; ++j)
        if (qs[j] > qs[best]) best = j;
      double R, g;
      if constexpr (kNstep) {
        R = td_ret;
        g = td_term ? 0.0 : td_g;
      } else {
        R = fmin(fmax(double(td_r), td.min_reward), td.max_reward);   // np.clip as the scalar head
        g = td_term ? 0.0 : td.discount;
      }
      s_ret = R;
      s_gam = g;
      s_a = td_a;
      s_astar = best;
      qa.act_rows[b] = td_a;
    }
    __syncthreads();
    const int a = s_a;
    if (t < nq) {   // T_j = float(R + g q'_j), q'_j = the target network's theta[a*][j]
      const float qj = theta[(int64_t(ld) + b) * ncols + s_astar * nq + t];
      const float T = float(__dadd_rn(s_ret, __dmul_rn(s_gam, double(qj))));
      s_t[t] = T;
      qa.tq[b * nq + t] = T;
    }
    __syncthreads();
    if (t < nq) {   // quantile i of the taken action against every target quantile j, j order
      const float th = theta[int64_t(b) * ncols + a * nq + t];
      const float wlo = s_wlo[t], whi = s_whi[t], kap = qa.kappa;
      float rho = 0.f, c = 0.f;
      for (int j = 0; j < nq; ++j) {
        const float u = __fsub_rn(s_t[j], th);
        const float w = u < 0.f ? whi : wlo;
        const float au = fabsf(u);
        if (kap > 0.f) {
          const float L = au <= kap ? __fmul_rn(0.5f, __fmul_rn(u, u)) : __fmul_rn(kap, __fsub_rn(au, __fmul_rn(0.5f, kap)));
          rho = __fadd_rn(rho, __fdiv_rn(__fmul_rn(w, L), kap));
          c = __fadd_rn(c, __fdiv_rn(__fmul_rn(w, fminf(fmaxf(u, -kap), kap)), kap));
        } else {
          rho = __fadd_rn(rho, __fmul_rn(w, au));
          c = __fadd_rn(c, u > 0.f ? w : u < 0.f ? -w : 0.f);
        }
      }
      float g = -__fdiv_rn(c, float(nq));
      if (td.isw) g = __fmul_rn(g, td.isw[b]);
      s_l[t] = __fdiv_rn(rho, float(nq));
      s_g[t] = g;
      qa.qgrad[b * nq + t] = g;
    }
    __syncthreads();
    if (t == 0) {   // the row loss: sum_i Loss_i, i order
      float l = 0.f;
      for (int i = 0; i < nq; ++i) l = __fadd_rn(l, s_l[i]);
      if (td.isw) {
        td.td_err[b] = l;
        td.row_cost[b] = __fmul_rn(td.isw[b], l);
      } else {
        td.row_cost[b] = l;
      }
    }
    {
      const float hv = s_h4[t];
      const float* w = w5_online + int64_t(t) * ncols + a * nq;
      float o = 0.f;
      if (hv > 0.f)
        for (int i = 0; i < nq; ++i) o = __fadd_rn(o, __fmul_rn(w[i], s_g[i]));
      td.dz4[b * kHidden + t] = o;
      if (td.dz4_hi) {
        const __half hh = __float2half_rn(o);
        const __half ll = __float2half_rn((o - __half2float(hh)) * 2048.0f);
        td.dz4_hi[b * kHidden + t] = hh;
        td.dz4_hi[td.dz4_lo_off + b * kHidden + t] = ll;
      }
    }
    float* dw = td.dw5_rows + int64_t(b) * kHidden * nq;
    for (int e = t; e < kHidden * nq; e += kHidden) dw[e] = __fmul_rn(s_h4[e / nq], s_g[e % nq]);
  }
  kt_end(kt);
}

// ------------------------------------------------------------------------------------------
// Implicit quantile network head (IQN, Dabney, Ostrovski, Silver and Munos 2018; b200dqn.h has the rules).  fc1 and fc2
// run on the expanded rows r = b * per + j with the scalar net's fc1 kernels and k_fc2_dist (A columns); fc2's gradient
// goes through k_opt_fc2_dist with block width 1.  The new kernels:
//   k_iqn_tau      one CTA: tau of every (slot, row) from the stated hash at the draw counter, then the counter + 1
//   k_iqn_phi      the cosine features c and the embedding phi = max(0, c We), 16 rows per CTA
//   k_iqn_mod      X = psi * phi, psi = conv3's output H3 of the row's sample
//   k_head_iqn     one CTA per sample: Q, a*, the target quantiles, the quantile Huber loss and dtheta, dZ4 and fc2's
//                  per-row partials
//   k_iqn_mod_bwd  dpsi (conv3's dZ) and dphi from fc1's dgrad dX
//   k_iqn_we       dWe and the embedding's update
// Every fp32 operation is rounded on its own (explicit _rn intrinsics).
// ------------------------------------------------------------------------------------------
constexpr int kIqnCos = 64;      // cosine features per row
constexpr int kIqnMaxPer = 64;   // N, K <= 64
constexpr int kIqnTB = 16;       // k_iqn_phi: rows per CTA

__device__ __forceinline__ unsigned long long iqn_mix(unsigned long long x) {   // splitmix64's finaliser
  x ^= x >> 30;
  x *= 0xBF58476D1CE4E5B9ull;
  x ^= x >> 27;
  x *= 0x94D049BB133111EBull;
  x ^= x >> 31;
  return x;
}

// tau[z][b * per + j] for z < nets, b < rows, j < per, drawn at the counter's value; thread 0 then advances the counter
// (every thread has read it by the barrier), so the next forward, or the next replay of a captured graph, draws fresh.
__global__ void __launch_bounds__(1024)
k_iqn_tau(unsigned long long* ctr, unsigned long long seed, int nets, int rows, int per, int ld, float* tau,
          const KTrace kt) {
  kt_begin(kt);
  pdl_wait();
  pdl_launch_dependents();
  const unsigned long long c = *ctr;
  const unsigned long long base = iqn_mix(seed + 0x9E3779B97F4A7C15ull * (c + 1ull));
  const int per_slot = rows * per;
  for (int e = threadIdx.x; e < nets * per_slot; e += blockDim.x) {
    const int z = e / per_slot, r = e % per_slot, b = r / per, j = r % per;
    const unsigned long long x = iqn_mix(base ^ ((unsigned long long)z << 32 | (unsigned long long)b << 8 | unsigned(j)));
    const unsigned m = unsigned(x >> 32) >> 9;   // the top 23 bits of the 32-bit hash
    tau[int64_t(z) * ld + r] = __fmul_rn(float(2u * m + 1u), 5.9604644775390625e-08f);   // (2m + 1) 2^-24, exact
  }
  __syncthreads();
  if (threadIdx.x == 0) *ctr = c + 1ull;
  kt_end(kt);
}

// Random-shift augmentation (b200dqn.h states the rule): crop[z][b] = (dy, dx) in [-p, p]^2 for slot z (0 prestates,
// 1 poststates) and sample b, drawn at the counter's value; thread 0 then advances the counter, so every train step,
// and every replay of a captured step graph, draws fresh offsets.  The hash is k_iqn_tau's, with its own seed and counter.
__global__ void __launch_bounds__(1024)
k_shift_draw(unsigned long long* ctr, unsigned long long seed, int pad, int rows, int32_t* crop, const KTrace kt) {
  kt_begin(kt);
  pdl_wait();
  pdl_launch_dependents();
  const unsigned long long c = *ctr;
  const unsigned long long base = iqn_mix(seed + 0x9E3779B97F4A7C15ull * (c + 1ull));
  const unsigned long long span = 2ull * unsigned(pad) + 1ull;
  for (int e = threadIdx.x; e < 2 * rows; e += blockDim.x) {
    const int z = e / rows, b = e % rows;
    const unsigned long long x = iqn_mix(base ^ ((unsigned long long)z << 32 | unsigned(b)));
    crop[2 * e] = int32_t(((x >> 32) * span) >> 32) - pad;
    crop[2 * e + 1] = int32_t(((x & 0xffffffffull) * span) >> 32) - pad;
  }
  __syncthreads();
  if (threadIdx.x == 0) *ctr = c + 1ull;
  kt_end(kt);
}

// ------------------------------------------------------------------------------------------
// Random ensemble mixture head (REM, Agarwal, Schuurmans and Norouzi 2020; b200dqn.h has the rules).  fc2's outputs
// theta[z][b][a * K + k] come from k_fc2_dist unchanged, fc2's gradient goes through k_opt_fc2_dist unchanged with K as
// the block width, and predict's Q is k_head_qr<1, false>'s mean over the K heads.  The new kernels:
//   k_rem_alpha   one CTA: the step's mixture alpha from the stated hash at the draw counter, then the counter + 1
//   k_head_rem    one CTA per sample: Q under alpha, the scalar head's TD step, dtheta, dZ4 (+ fp16 planes) and the
//                 compact dW5 row partial [512][K] of the taken action
// No expf / logf: every stage is +, -, *, / and comparisons, each rounded on its own.
// ------------------------------------------------------------------------------------------
// alpha_k = float(u_k / S) with u_k from k_iqn_tau's hash at (z, b, j) = (0, 0, k) and S = sum_k u_k in fp64, k order.
// One CTA, so the counter advance after the barrier cannot race a read: every thread has read it by then, and the step's
// head reads alpha, never the counter.
__global__ void __launch_bounds__(256)
k_rem_alpha(unsigned long long* ctr, unsigned long long seed, int K, float* alpha, const KTrace kt) {
  __shared__ double s_u[kMaxRemHeads];
  __shared__ double s_sum;
  kt_begin(kt);
  pdl_wait();
  pdl_launch_dependents();
  const int t = threadIdx.x;
  const unsigned long long c = *ctr;
  if (t < K) {
    const unsigned long long base = iqn_mix(seed + 0x9E3779B97F4A7C15ull * (c + 1ull));
    const unsigned m = unsigned(iqn_mix(base ^ (unsigned long long)unsigned(t)) >> 32) >> 9;   // top 23 bits
    s_u[t] = double(__fmul_rn(float(2u * m + 1u), 5.9604644775390625e-08f));   // (2m + 1) 2^-24, exact
  }
  __syncthreads();
  if (t == 0) {
    double S = 0.0;
    for (int k = 0; k < K; ++k) S = __dadd_rn(S, s_u[k]);
    s_sum = S;
    *ctr = c + 1ull;
  }
  __syncthreads();
  if (t < K) alpha[t] = float(__ddiv_rn(s_u[t], s_sum));
  kt_end(kt);
}

// One CTA (512 threads) per sample b of a train step.  Thread r < nets * A owns row (slot z, action a):
// Q = sum_k alpha_k theta_k in k order.  Thread 0 runs k_head's TD step on these Q; thread k < K forms dtheta_k =
// alpha_k d; every thread its dZ4 element and a stride of the dW5 row partial.  The TD scalars and Adam's step scalar
// come from head_td_scalars, before the dependency wait.
template <int kSlots, bool kNstep>
__global__ void __launch_bounds__(kHidden)
k_head_rem(const float* __restrict__ theta, int ld, int nets, const float* __restrict__ h4_online,
           const float* __restrict__ w5_online, float* q_online, float* q_target, float* q_online_post, int A, int K,
           const float* __restrict__ alpha, float* rgrad, int32_t* act_rows, const HeadTrainArgs td, const KTrace kt) {
  static_assert(kSlots == 2 || kSlots == 3, "online + target, or Double DQN's three slots");
  __shared__ float s_q[kSlots][kMaxActions];
  __shared__ float s_al[kMaxRemHeads], s_g[kMaxRemHeads], s_h4[kHidden];
  __shared__ float s_d;
  __shared__ int s_a;
  const int b = blockIdx.x, t = threadIdx.x, ncols = A * K;
  kt_begin(kt);
  int td_a = 0, td_term = 0;
  int64_t td_r = 0;
  double td_ret = 0.0, td_g = 1.0;
  head_td_scalars<kNstep>(td, b, t, td_a, td_r, td_term, td_ret, td_g);
  pdl_wait();
  pdl_launch_dependents();
  s_h4[t] = h4_online[b * kHidden + t];
  if (t < K) s_al[t] = alpha[t];
  __syncthreads();
  if (t < nets * A) {
    const int z = t / A, a = t % A;
    const float* th = theta + (int64_t(z) * ld + b) * ncols + a * K;
    float q = 0.f;
    for (int k = 0; k < K; ++k) q = __fadd_rn(q, __fmul_rn(s_al[k], th[k]));
    s_q[z][a] = q;
    (z == 0 ? q_online : z == 2 ? q_online_post : q_target)[b * A + a] = q;
  }
  __syncthreads();
  if (t == 0) {   // k_head's TD step on the mixed Q, with its contractions made explicit
    const int a = td_a;
    const double rr = fmin(fmax(double(td_r), td.min_reward), td.max_reward);
    float maxq;
    if constexpr (kSlots == 3) {
      int best = 0;
      for (int j = 1; j < A; ++j)
        if (s_q[2][j] > s_q[2][best]) best = j;
      maxq = s_q[1][best];
    } else {
      maxq = s_q[1][0];
      for (int j = 1; j < A; ++j) maxq = fmaxf(maxq, s_q[1][j]);
    }
    double y;
    if constexpr (kNstep) y = td_term ? td_ret : __dadd_rn(td_ret, __dmul_rn(td_g, double(maxq)));
    else y = td_term ? rr : __fma_rn(td.discount, double(maxq), rr);
    const float target = static_cast<float>(y);
    float d = __fsub_rn(s_q[0][a], target);
    if (td.isw) {
      const float wb = td.isw[b];
      td.td_err[b] = d;
      td.row_cost[b] = __fmul_rn(wb, __fmul_rn(__fmul_rn(0.5f, d), d));
      if (td.clip > 0.f) d = fminf(fmaxf(d, -td.clip), td.clip);
      d = __fmul_rn(d, wb);
    } else {
      td.row_cost[b] = __fmul_rn(__fmul_rn(0.5f, d), d);
      if (td.clip > 0.f) d = fminf(fmaxf(d, -td.clip), td.clip);
    }
    s_d = d;
    s_a = a;
    act_rows[b] = a;
  }
  __syncthreads();
  const int a = s_a;
  if (t < K) {
    const float g = __fmul_rn(s_al[t], s_d);
    s_g[t] = g;
    rgrad[b * K + t] = g;
  }
  __syncthreads();
  {
    const float hv = s_h4[t];
    const float* w = w5_online + int64_t(t) * ncols + a * K;
    float o = 0.f;
    if (hv > 0.f)
      for (int k = 0; k < K; ++k) o = __fadd_rn(o, __fmul_rn(w[k], s_g[k]));
    td.dz4[b * kHidden + t] = o;
    if (td.dz4_hi) {
      const __half hh = __float2half_rn(o);
      const __half ll = __float2half_rn((o - __half2float(hh)) * 2048.0f);
      td.dz4_hi[b * kHidden + t] = hh;
      td.dz4_hi[td.dz4_lo_off + b * kHidden + t] = ll;
    }
  }
  float* dw = td.dw5_rows + int64_t(b) * kHidden * K;
  for (int e = t; e < kHidden * K; e += kHidden) dw[e] = __fmul_rn(s_h4[e / K], s_g[e % K]);
  kt_end(kt);
}

// ------------------------------------------------------------------------------------------
// Bootstrapped DQN heads (Osband, Blundell, Pritzel and Van Roy 2016; b200dqn.h has the rules).  The REM head's K-headed
// fc2 (k_fc2_dist, and k_opt_fc2_dist with K as the block width, both unchanged) with one TD step per head in place of
// the mixture.  The new kernels:
//   k_head_boot      one CTA per sample: the masks of the sample's ring slot, each head's target, delta and masked
//                    gradient, the mean-over-heads Q rows, dZ4 (+ fp16 planes) and the compact dW5 row partial [512][K]
//   k_boot_predict   one CTA per row: Q at the device-resident active head, or the mean over the heads
//   k_boot_set_head  one thread: writes the active head in stream order
// No expf / logf: every stage is +, -, *, / and comparisons, each rounded on its own.
// ------------------------------------------------------------------------------------------
struct BootArgs {
  unsigned long long seed;
  double p;             // the mask probability
  uint8_t* mask;        // [ld][K] m_k
  float* y;             // [ld][K] float(y_k)
  float* delta;         // [ld][K] delta_k
  float* grad;          // [ld][K] dtheta on the taken action's heads
  int32_t* act_rows;    // [ld]
};

// One CTA (512 threads) per sample b of a train step.  Thread k < K hashes head k's mask from the ring slot midx[b]
// (before the dependency wait: it depends on the sampler alone, as the TD scalars do) and runs head k's TD step;
// thread r < nets * A writes the Q row (slot z, action a) as the mean over the heads; thread 0 sums the row cost and
// the TD error; every thread forms its dZ4 element and a stride of the dW5 row partial.
template <int kSlots, bool kNstep>
__global__ void __launch_bounds__(kHidden)
k_head_boot(const float* __restrict__ theta, int ld, int nets, const float* __restrict__ h4_online,
            const float* __restrict__ w5_online, float* q_online, float* q_target, float* q_online_post, int A, int K,
            const BootArgs ba, const HeadTrainArgs td, const KTrace kt) {
  static_assert(kSlots == 2 || kSlots == 3, "online + target, or Double DQN's three slots");
  __shared__ float s_h4[kHidden], s_g[kMaxRemHeads], s_c[kMaxRemHeads], s_e[kMaxRemHeads];
  __shared__ double s_ret, s_gam;
  __shared__ int s_a, s_term;
  const int b = blockIdx.x, t = threadIdx.x, ncols = A * K;
  kt_begin(kt);
  int td_a = 0, td_term = 0;
  int64_t td_r = 0;
  double td_ret = 0.0, td_g = 1.0;
  head_td_scalars<kNstep>(td, b, t, td_a, td_r, td_term, td_ret, td_g);
  bool m = false;
  if (t < K) {   // u = (2 (h >> 9) + 1) 2^-24 from the REM draw's hash at counter value midx[b]; exact in fp64
    const unsigned long long slot = (unsigned long long)td.midx[b];
    const unsigned long long base = iqn_mix(ba.seed + 0x9E3779B97F4A7C15ull * (slot + 1ull));
    const unsigned h = unsigned(iqn_mix(base ^ (unsigned long long)unsigned(t)) >> 32);
    m = __dmul_rn(double(2u * (h >> 9) + 1u), 5.9604644775390625e-08) < ba.p;
  }
  pdl_wait();
  pdl_launch_dependents();
  s_h4[t] = h4_online[b * kHidden + t];
  if (t < nets * A) {
    const int z = t / A, a = t % A;
    const float* th = theta + (int64_t(z) * ld + b) * ncols + a * K;
    float s = 0.f;
    for (int k = 0; k < K; ++k) s = __fadd_rn(s, th[k]);
    (z == 0 ? q_online : z == 2 ? q_online_post : q_target)[b * A + a] = __fdiv_rn(s, float(K));
  }
  if (t == 0) {
    if constexpr (kNstep) {
      s_ret = td_ret;
      s_gam = td_g;
    } else {
      s_ret = fmin(fmax(double(td_r), td.min_reward), td.max_reward);   // np.clip as the scalar head
      s_gam = td.discount;
    }
    s_term = td_term;
    s_a = td_a;
    ba.act_rows[b] = td_a;
  }
  __syncthreads();
  const int a = s_a;
  if (t < K) {   // head k = t: a*_k over slot 1's (slot 2's) column k, y_k, delta_k, the masked clipped gradient
    const float* th1 = theta + (int64_t(ld) + b) * ncols + t;
    const float* thc = kSlots == 3 ? theta + (int64_t(2) * ld + b) * ncols + t : th1;
    int best = 0;
    for (int j = 1; j < A; ++j)
      if (thc[j * K] > thc[best * K]) best = j;
    const double maxq = double(th1[best * K]);
    double y;
    if constexpr (kNstep) y = s_term ? s_ret : __dadd_rn(s_ret, __dmul_rn(s_gam, maxq));
    else y = s_term ? s_ret : __fma_rn(s_gam, maxq, s_ret);
    const float target = static_cast<float>(y);
    const float dl = __fsub_rn(theta[int64_t(b) * ncols + a * K + t], target);
    float d = dl;
    if (td.clip > 0.f) d = fminf(fmaxf(d, -td.clip), td.clip);
    if (td.isw) d = __fmul_rn(d, td.isw[b]);
    const float g = m ? d : 0.f;
    s_c[t] = m ? __fmul_rn(__fmul_rn(0.5f, dl), dl) : 0.f;
    s_e[t] = fabsf(dl);
    s_g[t] = g;
    ba.mask[b * K + t] = m ? 1 : 0;
    ba.y[b * K + t] = target;
    ba.delta[b * K + t] = dl;
    ba.grad[b * K + t] = g;
  }
  __syncthreads();
  if (t == 0) {   // the row cost over the unmasked heads and the TD error over every head, k order, then / K
    float c = 0.f, e = 0.f;
    for (int k = 0; k < K; ++k) {
      c = __fadd_rn(c, s_c[k]);
      e = __fadd_rn(e, s_e[k]);
    }
    c = __fdiv_rn(c, float(K));
    if (td.isw) {
      td.td_err[b] = __fdiv_rn(e, float(K));
      c = __fmul_rn(td.isw[b], c);
    }
    td.row_cost[b] = c;
  }
  {   // the shared network's gradient is the mean over the heads; the heads get their full dtheta
    const float hv = s_h4[t];
    const float* w = w5_online + int64_t(t) * ncols + a * K;
    float o = 0.f;
    if (hv > 0.f) {
      for (int k = 0; k < K; ++k) o = __fadd_rn(o, __fmul_rn(w[k], s_g[k]));
      o = __fdiv_rn(o, float(K));
    }
    td.dz4[b * kHidden + t] = o;
    if (td.dz4_hi) {
      const __half hh = __float2half_rn(o);
      const __half ll = __float2half_rn((o - __half2float(hh)) * 2048.0f);
      td.dz4_hi[b * kHidden + t] = hh;
      td.dz4_hi[td.dz4_lo_off + b * kHidden + t] = ll;
    }
  }
  float* dw = td.dw5_rows + int64_t(b) * kHidden * K;
  for (int e = t; e < kHidden * K; e += kHidden) dw[e] = __fmul_rn(s_h4[e / K], s_g[e % K]);
  kt_end(kt);
}

// One CTA of 32 threads per predict row b; thread a < A writes Q[b][a] at the active head read at run time, so a
// captured predict graph follows b200dqn_net_set_active_head without recapture.  h = -1: k_head_qr<1, false>'s mean.
__global__ void __launch_bounds__(32)
k_boot_predict(const float* __restrict__ theta, int A, int K, const int32_t* __restrict__ head, float* q,
               const KTrace kt) {
  kt_begin(kt);
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.x, a = threadIdx.x;
  if (a < A) {
    const int h = *head;
    const float* th = theta + (int64_t(b) * A + a) * K;
    float v;
    if (h >= 0) {
      v = th[h];
    } else {
      float s = 0.f;
      for (int k = 0; k < K; ++k) s = __fadd_rn(s, th[k]);
      v = __fdiv_rn(s, float(K));
    }
    q[b * A + a] = v;
  }
  kt_end(kt);
}

__global__ void k_boot_set_head(int32_t* head, int h) { *head = h; }

// grid (cdiv(rows, 16), nets).  c[r][i] = float(cos((pi i) tau_r)) in fp64, stored for the embedding's gradient; then
// thread t takes columns t, t + 256, ... and accumulates the CTA's 16 rows of column col in i order.
__global__ void __launch_bounds__(256)
k_iqn_phi(const float* __restrict__ tau, int rows, int ld, const float* __restrict__ we_online,
          const float* __restrict__ we_target, float* __restrict__ cosf, float* __restrict__ phi, const KTrace kt) {
  __shared__ float s_c[kIqnTB][kIqnCos];
  const int z = blockIdx.y, r0 = blockIdx.x * kIqnTB, t = threadIdx.x;
  const int nrow = min(kIqnTB, rows - r0);
  const float* we = z ? we_target : we_online;
  kt_begin(kt);
  pdl_wait();
  pdl_launch_dependents();
  for (int e = t; e < kIqnTB * kIqnCos; e += 256) {
    const int r = e / kIqnCos, i = e % kIqnCos;
    float c = 0.f;
    if (r < nrow) {
      c = float(cos(__dmul_rn(__dmul_rn(3.141592653589793, double(i)), double(tau[int64_t(z) * ld + r0 + r]))));
      cosf[(int64_t(z) * ld + r0 + r) * kIqnCos + i] = c;
    }
    s_c[r][i] = c;
  }
  __syncthreads();
  for (int col = t; col < kFlat; col += 256) {
    float acc[kIqnTB];
#pragma unroll
    for (int j = 0; j < kIqnTB; ++j) acc[j] = 0.f;
    for (int i = 0; i < kIqnCos; ++i) {
      const float w = we[i * kFlat + col];
#pragma unroll
      for (int j = 0; j < kIqnTB; ++j) acc[j] = __fadd_rn(acc[j], __fmul_rn(s_c[j][i], w));
    }
#pragma unroll
    for (int j = 0; j < kIqnTB; ++j)
      if (j < nrow) phi[(int64_t(z) * ld + r0 + j) * kFlat + col] = fmaxf(acc[j], 0.f);
  }
  kt_end(kt);
}

// X[z][r][col] = H3[z][r / per][col] * phi[z][r][col] over nets slots of `rows` expanded rows (grid-stride), and on the
// tensor-core engine (x16 != nullptr) its hi / lo fp16 planes
__global__ void __launch_bounds__(256)
k_iqn_mod(const float* __restrict__ h3_online, const float* __restrict__ h3_target, const float* __restrict__ phi,
          float* __restrict__ x, __half* __restrict__ x16, int nets, int rows, int per, int ld, const KTrace kt) {
  kt_begin(kt);
  pdl_wait();
  pdl_launch_dependents();
  const int64_t slot = int64_t(rows) * kFlat, total = nets * slot;
  for (int64_t e = int64_t(blockIdx.x) * 256 + threadIdx.x; e < total; e += int64_t(gridDim.x) * 256) {
    const int z = int(e / slot);
    const int64_t re = e - z * slot;
    const int r = int(re / kFlat), col = int(re % kFlat);
    const float psi = (z ? h3_target : h3_online)[int64_t(r / per) * kFlat + col];
    const int64_t o = int64_t(z) * ld * kFlat + re;
    const float v = __fmul_rn(psi, phi[o]);
    x[o] = v;
    if (x16) {   // tensor-core engine: fc1's operand planes, hi and lo scaled by 2048, slot z at z * 2 * ld * 3136
      const __half hh = __float2half_rn(v);
      __half* hp = x16 + 2 * int64_t(z) * ld * kFlat + re;
      hp[0] = hh;
      hp[int64_t(ld) * kFlat] = __float2half_rn((v - __half2float(hh)) * 2048.0f);
    }
  }
  kt_end(kt);
}

struct IqnArgs {
  int per;            // rows per sample: N (train) or K (predict)
  int ld;             // slot stride of tau and theta (iqn_rows)
  float kappa;        // the Huber threshold (clip_error); 0: the pure quantile loss
  const float* tau;   // [2][ld]
  float* tq;          // [nb][N] target quantiles T_j
  float* qgrad;       // [nb N] dtheta of each online row
  int32_t* act_rows;  // [nb N] taken action of each online row (selects fc2's gradient column)
};

// The FQF head's additions to k_head_iqn (b200dqn.h's FQF rules 4 and 7)
struct FqfArgs {
  const float* frac;    // [nb][N + 1] tau
  const float* prob;    // [nb][N] q
  const float* bnd;     // [nb (N - 1)][A] theta_bnd
  float* g;             // [nb][N - 1]
  float* dl;            // [nb][N]
  float adam_flr;       // Adam: fraction_lr, and where this step's l of the fraction layer goes (nullptr otherwise)
  float* adam_lf;
};

// One CTA (512 threads) per sample b; its rows are r = b * per + j.  Thread t < nets * A owns (slot z, action a):
// Q = (sum_j theta[z][r][a], j order) / per (FQF: sum_j dtau_j theta[z][r][a]).  With td.enable (kSlots = 2): thread 0
// picks a* and the fp64 return, thread j < N forms T_j, thread i < N runs k_head_qr's j loop for online row b N + i with
// the weights tau_i and 1 - tau_i, thread 0 sums the row loss (FQF: and forms g, dq and dl), and thread k writes dZ4 and
// fc2's row partial of unit k for every online row of the sample.  The body is shared by k_head_iqn and k_head_fqf.
template <int kSlots, bool kNstep, bool kFqf>
__device__ __forceinline__ void
head_iqn_body(const float* __restrict__ theta, int nets, const float* __restrict__ h4_online,
              const float* __restrict__ w5_online, float* q_online, float* q_target, int A, const IqnArgs& ia,
              const FqfArgs& fa, const HeadTrainArgs& td, const KTrace& kt) {
  static_assert(kSlots == 1 || kSlots == 2, "predict, or online + target");
  __shared__ float s_q[kSlots][kMaxActions];
  __shared__ float s_t[kIqnMaxPer], s_l[kIqnMaxPer], s_g[kIqnMaxPer];
  __shared__ double s_ret, s_gam;
  __shared__ int s_a, s_astar;
  const int b = blockIdx.x, t = threadIdx.x, np = ia.per;
  const int64_t ld = ia.ld, r0 = int64_t(b) * np;
  kt_begin(kt);
  int td_a = 0, td_term = 0;
  int64_t td_r = 0;
  double td_ret = 0.0, td_g = 1.0;
  head_td_scalars<kNstep>(td, b, t, td_a, td_r, td_term, td_ret, td_g);
  if constexpr (kFqf) {
    if (td.enable && fa.adam_lf && b == 0 && t == 32) {   // head_td_scalars' Adam scalar at lr = fraction_lr
      const double tt = double(*td.step) + 1.0;
      const float a = float(1.0 - pow(0.999, tt)), c = float(1.0 - pow(0.9, tt));
      *fa.adam_lf = __fdiv_rn(__fmul_rn(fa.adam_flr, __fsqrt_rn(a)), c);
    }
  }
  pdl_wait();
  pdl_launch_dependents();
  if (t < nets * A) {
    const int z = t / A, a = t % A;
    const float* th = theta + (z * ld + r0) * A + a;
    float q;
    if constexpr (kFqf) {
      const float* fr = fa.frac + int64_t(b) * (np + 1);
      q = 0.f;
      for (int j = 0; j < np; ++j) q = __fadd_rn(q, __fmul_rn(__fsub_rn(fr[j + 1], fr[j]), th[int64_t(j) * A]));
    } else {
      float s = 0.f;
      for (int j = 0; j < np; ++j) s = __fadd_rn(s, th[int64_t(j) * A]);
      q = __fdiv_rn(s, float(np));
    }
    s_q[z][a] = q;
    (z == 0 ? q_online : q_target)[b * A + a] = q;
  }
  if constexpr (kSlots > 1) {
    if (!td.enable) {
      kt_end(kt);
      return;
    }
    __syncthreads();
    if (t == 0) {
      int best = 0;
      for (int j = 1; j < A; ++j)
        if (s_q[1][j] > s_q[1][best]) best = j;
      double R, g;
      if constexpr (kNstep) {
        R = td_ret;
        g = td_term ? 0.0 : td_g;
      } else {
        R = fmin(fmax(double(td_r), td.min_reward), td.max_reward);   // np.clip as the scalar head
        g = td_term ? 0.0 : td.discount;
      }
      s_ret = R;
      s_gam = g;
      s_a = td_a;
      s_astar = best;
    }
    __syncthreads();
    const int a = s_a;
    if (t < np) {   // T_j = float(R + g q'_j), q'_j = the target network's theta of row b N + j at a*
      const float qj = theta[(ld + r0 + t) * A + s_astar];
      const float T = float(__dadd_rn(s_ret, __dmul_rn(s_gam, double(qj))));
      s_t[t] = T;
      ia.tq[r0 + t] = T;
    }
    __syncthreads();
    if (t < np) {   // online row b N + i (i = t) against every target sample j, j order
      const float th = theta[(r0 + t) * A + a];
      const float wlo = ia.tau[r0 + t], whi = __fsub_rn(1.f, wlo), kap = ia.kappa;
      float rho = 0.f, c = 0.f;
      for (int j = 0; j < np; ++j) {
        const float u = __fsub_rn(s_t[j], th);
        const float w = u < 0.f ? whi : wlo;
        const float au = fabsf(u);
        if (kap > 0.f) {
          const float L = au <= kap ? __fmul_rn(0.5f, __fmul_rn(u, u)) : __fmul_rn(kap, __fsub_rn(au, __fmul_rn(0.5f, kap)));
          rho = __fadd_rn(rho, __fdiv_rn(__fmul_rn(w, L), kap));
          c = __fadd_rn(c, __fdiv_rn(__fmul_rn(w, fminf(fmaxf(u, -kap), kap)), kap));
        } else {
          rho = __fadd_rn(rho, __fmul_rn(w, au));
          c = __fadd_rn(c, u > 0.f ? w : u < 0.f ? -w : 0.f);
        }
      }
      float g = -__fdiv_rn(c, float(np));
      if (td.isw) g = __fmul_rn(g, td.isw[b]);
      s_l[t] = __fdiv_rn(rho, float(np));
      s_g[t] = g;
      ia.qgrad[r0 + t] = g;
      ia.act_rows[r0 + t] = a;
    }
    __syncthreads();
    if (t == 0) {   // the row loss: sum_i Loss_i, i order
      float l = 0.f;
      for (int i = 0; i < np; ++i) l = __fadd_rn(l, s_l[i]);
      if (td.isw) {
        td.td_err[b] = l;
        td.row_cost[b] = __fmul_rn(td.isw[b], l);
      } else {
        td.row_cost[b] = l;
      }
      if constexpr (kFqf) {   // the fraction gradient g, dq and the logit gradient dl (s_t and s_l are free again)
        const int nb1 = np - 1;
        const float* th0 = theta + r0 * A + a;
        const float* bt = fa.bnd + int64_t(b) * nb1 * A + a;
        for (int i = 1; i < np; ++i) {
          float gi = __fsub_rn(__fsub_rn(__fmul_rn(2.f, bt[int64_t(i - 1) * A]), th0[int64_t(i) * A]),
                               th0[int64_t(i - 1) * A]);
          if (td.isw) gi = __fmul_rn(gi, td.isw[b]);
          s_t[i] = gi;
          fa.g[int64_t(b) * nb1 + i - 1] = gi;
        }
        float acc = 0.f;
        s_l[np - 1] = 0.f;
        for (int k = np - 2; k >= 0; --k) {
          acc = __fadd_rn(acc, s_t[k + 1]);
          s_l[k] = acc;
        }
        const float* qk = fa.prob + int64_t(b) * np;
        float s = 0.f;
        for (int k = 0; k < np; ++k) s = __fadd_rn(s, __fmul_rn(qk[k], s_l[k]));
        for (int k = 0; k < np; ++k) fa.dl[int64_t(b) * np + k] = __fmul_rn(qk[k], __fsub_rn(s_l[k], s));
      }
    }
    const float w5a = w5_online[t * A + a];
    for (int i = 0; i < np; ++i) {
      const int64_t r = r0 + i;
      const float hv = h4_online[r * kHidden + t], g = s_g[i];
      const float o = hv > 0.f ? __fmul_rn(w5a, g) : 0.f;
      td.dz4[r * kHidden + t] = o;
      if (td.dz4_hi) {   // the tensor-core fc1 dgrad / wgrad operand
        const __half hh = __float2half_rn(o);
        td.dz4_hi[r * kHidden + t] = hh;
        td.dz4_hi[td.dz4_lo_off + r * kHidden + t] = __float2half_rn((o - __half2float(hh)) * 2048.0f);
      }
      td.dw5_rows[r * kHidden + t] = __fmul_rn(hv, g);
    }
  }
  kt_end(kt);
}

template <int kSlots, bool kNstep>
__global__ void __launch_bounds__(kHidden)
k_head_iqn(const float* __restrict__ theta, int nets, const float* __restrict__ h4_online,
           const float* __restrict__ w5_online, float* q_online, float* q_target, int A, const IqnArgs ia,
           const HeadTrainArgs td, const KTrace kt) {
  head_iqn_body<kSlots, kNstep, false>(theta, nets, h4_online, w5_online, q_online, q_target, A, ia, FqfArgs{}, td, kt);
}

template <int kSlots, bool kNstep>
__global__ void __launch_bounds__(kHidden)
k_head_fqf(const float* __restrict__ theta, int nets, const float* __restrict__ h4_online,
           const float* __restrict__ w5_online, float* q_online, float* q_target, int A, const IqnArgs ia,
           const FqfArgs fa, const HeadTrainArgs td, const KTrace kt) {
  head_iqn_body<kSlots, kNstep, true>(theta, nets, h4_online, w5_online, q_online, q_target, A, ia, fa, td, kt);
}

// One thread per (sample b, column col) of `rows` samples: dpsi[b][col] = (sum_j dX[r][col] phi[r][col], j order) under
// psi's mask (and its fp16 planes on the tensor-core engine), and dphi[r][col] = phi > 0 ? dX[r][col] psi : 0,
// r = b * per + j.
__global__ void __launch_bounds__(256)
k_iqn_mod_bwd(const float* __restrict__ dx, const float* __restrict__ phi, const float* __restrict__ h3,
              float* __restrict__ dpsi, __half* __restrict__ dpsi16, int64_t dpsi_lo, float* __restrict__ dphi, int rows,
              int per, const KTrace kt) {
  kt_begin(kt);
  pdl_wait();
  pdl_launch_dependents();
  const int e = blockIdx.x * 256 + threadIdx.x;
  if (e < rows * kFlat) {
    const int b = e / kFlat, col = e % kFlat;
    const float psi = h3[e];
    float acc = 0.f;
    for (int j = 0; j < per; ++j) {
      const int64_t o = (int64_t(b) * per + j) * kFlat + col;
      const float d = dx[o], p = phi[o];
      acc = __fadd_rn(acc, __fmul_rn(d, p));
      dphi[o] = p > 0.f ? __fmul_rn(d, psi) : 0.f;
    }
    const float o = psi > 0.f ? acc : 0.f;
    dpsi[e] = o;
    if (dpsi16) {   // tensor-core engine: the planes conv3's dgrad and wgrad read
      const __half hh = __float2half_rn(o);
      dpsi16[e] = hh;
      dpsi16[dpsi_lo + e] = __float2half_rn((o - __half2float(hh)) * 2048.0f);
    }
  }
  kt_end(kt);
}

// dWe[i][col] = sum_r c[r][i] dphi[r][col] over `rows` online rows in row order, then (update) the configured optimizer.
// grid cdiv(3136, 32): thread (ig, cl) of a CTA owns column blockIdx.x * 32 + cl and features ig * 8 .. ig * 8 + 7; the
// rows pass through shared memory 32 at a time.
constexpr int kWeCols = 32, kWeRows = 32;
__global__ void __launch_bounds__(256)
k_iqn_we(const float* __restrict__ cosf, const float* __restrict__ dphi, int rows, float* __restrict__ g_out,
         float* __restrict__ w, float* __restrict__ sst, int update, const OptArgs opt, const KTrace kt) {
  __shared__ float s_c[kWeRows][kIqnCos];
  __shared__ float s_d[kWeRows][kWeCols];
  const int t = threadIdx.x, cl = t % kWeCols, ig = t / kWeCols, c0 = blockIdx.x * kWeCols;
  kt_begin(kt);
  pdl_wait();
  pdl_launch_dependents();
  float acc[8];
#pragma unroll
  for (int u = 0; u < 8; ++u) acc[u] = 0.f;
  for (int rb = 0; rb < rows; rb += kWeRows) {
    const int nr = min(kWeRows, rows - rb);
    __syncthreads();
    for (int e = t; e < kWeRows * kIqnCos; e += 256) {
      const int r = e / kIqnCos, i = e % kIqnCos;
      s_c[r][i] = r < nr ? cosf[int64_t(rb + r) * kIqnCos + i] : 0.f;
    }
    for (int e = t; e < kWeRows * kWeCols; e += 256) {
      const int r = e / kWeCols, cc = c0 + e % kWeCols;
      s_d[r][e % kWeCols] = r < nr && cc < kFlat ? dphi[int64_t(rb + r) * kFlat + cc] : 0.f;
    }
    __syncthreads();
    for (int r = 0; r < nr; ++r) {
      const float d = s_d[r][cl];
#pragma unroll
      for (int u = 0; u < 8; ++u) acc[u] = __fadd_rn(acc[u], __fmul_rn(s_c[r][ig * 8 + u], d));
    }
  }
  const int col = c0 + cl;
  if (col < kFlat) {
    const float l = opt_step_scalar(opt);
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int64_t wi = int64_t(ig * 8 + u) * kFlat + col;
      g_out[wi] = acc[u];
      if (update) {
        float s[3] = {0.f, 0.f, 0.f};
        for (int k = 0; k < opt.nstates; ++k) s[k] = sst[k * opt.plane + wi];
        float wv = w[wi];
        opt_update1(opt, l, acc[u], wv, s[0], s[1], s[2]);
        w[wi] = wv;
        for (int k = 0; k < opt.nstates; ++k) sst[k * opt.plane + wi] = s[k];
      }
    }
  }
  kt_end(kt);
}

// ------------------------------------------------------------------------------------------
// Fully parameterized quantile function head (FQF, Yang et al. 2019; b200dqn.h has the rules).  It is the IQN head with
// tau = the fraction proposal's tauhat: k_iqn_phi, k_iqn_mod, fc1, k_fc2_dist, k_iqn_mod_bwd and k_iqn_we run unchanged,
// and the boundary pass runs phi, mod, fc1 and k_fc2_dist once more on the online network at tau_1..tau_{N-1}.  The new
// kernels:
//   k_fqf_fraction  one CTA per sample: the logits, the fp64 proposal q, tau and tauhat
//   k_head_fqf      k_head_iqn's body with the FQF Q rule and, in a train step, the fraction and logit gradients
//   k_fqf_wf        dW_f and the fraction layer's update at fraction_lr
// ------------------------------------------------------------------------------------------
constexpr int kFqfMaxN = 64;

// One CTA (256 threads) per sample b.  Warp w computes the logits k = w, w + 8, ... (rule 1's lane order), thread 0 the
// fp64 prefix sums, then thread i writes tau_i, q_i and tauhat_i: into both slots of tau (nets = 2) at rows b N + i, and
// tau_1..tau_{N-1} into btau (a train step; nullptr on predict).
__global__ void __launch_bounds__(256)
k_fqf_fraction(const float* __restrict__ psi, const float* __restrict__ wf, int N, int nets, int ld,
               float* __restrict__ logit, float* __restrict__ prob, float* __restrict__ frac, float* __restrict__ tau,
               float* __restrict__ btau, const KTrace kt) {
  __shared__ float s_psi[kFlat];
  __shared__ float s_l[kFqfMaxN];
  __shared__ double s_e[kFqfMaxN], s_c[kFqfMaxN + 1];
  const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  kt_begin(kt);
  pdl_wait();
  pdl_launch_dependents();
  for (int col = t; col < kFlat; col += 256) s_psi[col] = psi[int64_t(b) * kFlat + col];
  __syncthreads();
  for (int k = warp; k < N; k += 8) {
    const float* w = wf + int64_t(k) * kFlat;
    float acc = 0.f;
    for (int col = lane; col < kFlat; col += 32) acc = __fadd_rn(acc, __fmul_rn(s_psi[col], w[col]));
    for (int h = 16; h > 0; h >>= 1) acc = __fadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, h));
    if (lane == 0) {
      s_l[k] = acc;
      logit[int64_t(b) * N + k] = acc;
    }
  }
  __syncthreads();
  if (t == 0) {
    double m = double(s_l[0]);
    for (int k = 1; k < N; ++k) m = fmax(m, double(s_l[k]));
    double c = 0.0;
    s_c[0] = 0.0;
    for (int k = 0; k < N; ++k) {
      const double e = exp(__dsub_rn(double(s_l[k]), m));
      s_e[k] = e;
      c = __dadd_rn(c, e);
      s_c[k + 1] = c;
    }
  }
  __syncthreads();
  const double S = s_c[N];
  for (int i = t; i <= N; i += 256) {
    const float ti = float(__ddiv_rn(s_c[i], S));
    frac[int64_t(b) * (N + 1) + i] = ti;
    if (btau && i >= 1 && i < N) btau[int64_t(b) * (N - 1) + i - 1] = ti;
    if (i < N) {
      prob[int64_t(b) * N + i] = float(__ddiv_rn(s_e[i], S));
      const float th = float(__ddiv_rn(__dadd_rn(s_c[i], s_c[i + 1]), __dmul_rn(2.0, S)));
      for (int z = 0; z < nets; ++z) tau[int64_t(z) * ld + int64_t(b) * N + i] = th;
    }
  }
  kt_end(kt);
}

// dW_f[k][col] = sum_b dl[b][k] psi[b][col] in b order, one thread per (k, col); then (update) the configured optimizer
// with opt.lr = fraction_lr.
__global__ void __launch_bounds__(256)
k_fqf_wf(const float* __restrict__ dl, const float* __restrict__ psi, int rows, int N, float* __restrict__ g_out,
         float* __restrict__ w, float* __restrict__ sst, int update, const OptArgs opt, const KTrace kt) {
  kt_begin(kt);
  pdl_wait();
  pdl_launch_dependents();
  const int e = blockIdx.x * 256 + threadIdx.x;
  if (e < N * kFlat) {
    const int k = e / kFlat, col = e % kFlat;
    float acc = 0.f;
    for (int b = 0; b < rows; ++b) acc = __fadd_rn(acc, __fmul_rn(dl[int64_t(b) * N + k], psi[int64_t(b) * kFlat + col]));
    g_out[e] = acc;
    if (update) {
      const float l = opt_step_scalar(opt);
      float s[3] = {0.f, 0.f, 0.f};
      for (int q = 0; q < opt.nstates; ++q) s[q] = sst[q * opt.plane + e];
      float wv = w[e];
      opt_update1(opt, l, acc, wv, s[0], s[1], s[2]);
      w[e] = wv;
      for (int q = 0; q < opt.nstates; ++q) sst[q * opt.plane + e] = s[q];
    }
  }
  kt_end(kt);
}

// ------------------------------------------------------------------------------------------
// K6: gradient reduction + the configured Neon optimizer (src/deepqnetwork.py:50-61,165; rules in optim.cuh).
// RMSProp:  g = dW / bsz;  s = decay*s + g*g*(1-decay);  W = W - (g*lr) / (sqrt(s + eps) + eps)
// The split-K partials of every layer are summed here in fixed order (deterministic), so the
// wgrad kernels never need atomics.  mode bit0: sum partials (else read g_buf); bit1: write the
// summed gradient to g_buf (all-reduce input / get_grads); bit2: apply the update.
// Explicit _rn intrinsics keep the compiler from contracting into FMAs, so given identical
// gradients the update is bit-identical to the numpy oracle.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_optimizer(const LayerTable lt, const float* __restrict__ part, float* __restrict__ g_buf, float* __restrict__ w,
            float* __restrict__ s, int64_t b4, int64_t e4, int mode, const OptArgs opt, const KTrace kt) {
  const int64_t i4 = b4 + blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
  kt_begin(kt);
  pdl_wait();
  pdl_launch_dependents();
  if (i4 >= e4) return;
  const int64_t i = i4 * 4;
  float4 g;
  if (mode & 1) {
    int l = 0;
#pragma unroll
    for (int j = 1; j < kLayers; ++j) l += (i >= lt.off[j]) ? 1 : 0;
    const int64_t lsize = lt.off[l + 1] - lt.off[l];
    const float* p = part + lt.part_off[l] + (i - lt.off[l]);
    // Fixed summation tree shared with k_opt_conv (net_umma.cu): eight strided running sums
    // a[l] = sum_{sp = l (mod 8)} part[sp], combined as ((a0+a1)+(a2+a3)) + ((a4+a5)+(a6+a7)).
    const int nsp = lt.splits[l];
    float4 a[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) a[u] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int sp0 = 0; sp0 < nsp; sp0 += 8) {
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        if (sp0 + u < nsp) {
          const float4 v = *reinterpret_cast<const float4*>(p + (sp0 + u) * lsize);
          a[u].x += v.x; a[u].y += v.y; a[u].z += v.z; a[u].w += v.w;
        }
      }
    }
#pragma unroll
    for (int o = 1; o < 8; o <<= 1)
#pragma unroll
      for (int u = 0; u < 8; u += 2 * o) {
        a[u].x += a[u + o].x; a[u].y += a[u + o].y; a[u].z += a[u + o].z; a[u].w += a[u + o].w;
      }
    g = a[0];
  } else {
    g = *reinterpret_cast<const float4*>(g_buf + i);
  }
  if (mode & 2) *reinterpret_cast<float4*>(g_buf + i) = g;
  if (mode & 4) {
    float nw[4];
    opt_update_vec<4>(opt, opt_step_scalar(opt), reinterpret_cast<const float*>(&g), nw, w + i, s + i);
  }
  kt_end(kt);
}

// Soft target update of a parameter range (b200dqn_net_config::soft_target_tau): tw <- fl(fl(c tw) + fl(t w)), four
// elements per thread.  The only update of fc2, the IQN / FQF embedding and the FQF fraction layer, and of every layer
// on the SIMT engine; the tensor-core engine fuses conv1..fc1 into their image packs (umma_soft_pack).
__global__ void __launch_bounds__(256)
k_soft_blend(const float* __restrict__ w, float* __restrict__ tw, int64_t n4, float c, float t, const KTrace kt) {
  const int64_t i4 = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
  kt_begin(kt);
  pdl_wait();
  pdl_launch_dependents();
  if (i4 < n4) {
    const float4 a = reinterpret_cast<const float4*>(tw)[i4];
    const float4 b = reinterpret_cast<const float4*>(w)[i4];
    reinterpret_cast<float4*>(tw)[i4] = make_float4(soft_blend1(a.x, b.x, c, t), soft_blend1(a.y, b.y, c, t),
                                                    soft_blend1(a.z, b.z, c, t), soft_blend1(a.w, b.w, c, t));
  }
  kt_end(kt);
}

// ------------------------------------------------------------------------------------------
// Global gradient-norm clipping (b200dqn_net_config::max_grad_norm; b200dqn.h has the rule).  Three kernels:
//   k_grad_sq     one layer's sum of squares of gg = fl(g / bsz) in fp64, one partial per CTA of kSqChunk elements
//   k_clip_scale  one CTA: each layer's partials in slot order into S_l, then N and c32
//   k_opt_clip    the clipped update of a parameter range from its summed gradient (every layer but the tensor-core
//                 engine's fc1, which k_opt_fc1_clip updates and repacks in one pass; its conv layers are repacked after)
// Every sum runs in a fixed order (per thread, then the warp's xor butterfly, then the warps in order): no atomics, so
// two runs give the same bits.
// ------------------------------------------------------------------------------------------
constexpr int kSqChunk = 4096;   // elements per k_grad_sq CTA: 256 threads x 4 float4

__device__ __forceinline__ double block_sum_f64(double acc, double* s_w) {
  for (int h = 16; h > 0; h >>= 1) acc = __dadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, h));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = acc;
  __syncthreads();
  double s = s_w[0];
  for (int w = 1; w < int(blockDim.x >> 5); ++w) s = __dadd_rn(s, s_w[w]);
  return s;
}

__global__ void __launch_bounds__(256)
k_grad_sq(const float* __restrict__ g, int64_t n4, float bsz, double* __restrict__ part, const KTrace kt) {
  __shared__ double s_w[8];
  kt_begin(kt);
  pdl_wait();
  pdl_launch_dependents();
  double acc = 0.0;
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int64_t i4 = int64_t(blockIdx.x) * (kSqChunk / 4) + u * 256 + threadIdx.x;
    if (i4 < n4) {
      const float4 v = reinterpret_cast<const float4*>(g)[i4];
      const double a = __fdiv_rn(v.x, bsz), b = __fdiv_rn(v.y, bsz), c = __fdiv_rn(v.z, bsz), d = __fdiv_rn(v.w, bsz);
      acc = __dadd_rn(acc, __dmul_rn(a, a));
      acc = __dadd_rn(acc, __dmul_rn(b, b));
      acc = __dadd_rn(acc, __dmul_rn(c, c));
      acc = __dadd_rn(acc, __dmul_rn(d, d));
    }
  }
  const double s = block_sum_f64(acc, s_w);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
  kt_end(kt);
}

// clip: [0, 6) S_l, [6] N, [7] c32 (as f32), then the partials; layer l's are slots 8 + base[l] .. 8 + base[l + 1] - 1
struct SqLayout { int64_t base[7]; };

__global__ void __launch_bounds__(256)
k_clip_scale(double* __restrict__ clip, const SqLayout lay, double max_norm, const KTrace kt) {
  __shared__ double s_w[8];
  kt_begin(kt);
  pdl_wait();
  pdl_launch_dependents();
  double S = 0.0;
  for (int l = 0; l < 6; ++l) {
    double acc = 0.0;
    for (int64_t j = lay.base[l] + threadIdx.x; j < lay.base[l + 1]; j += 256) acc = __dadd_rn(acc, clip[8 + j]);
    const double Sl = block_sum_f64(acc, s_w);
    if (threadIdx.x == 0) clip[l] = Sl;
    S = __dadd_rn(S, Sl);
  }
  if (threadIdx.x == 0) {
    const double N = __dsqrt_rn(S);
    const double c = __ddiv_rn(max_norm, __dadd_rn(N, 1e-6));
    clip[6] = N;
    reinterpret_cast<float*>(clip + 7)[0] = c < 1.0 ? __double2float_rn(c) : 1.f;   // NaN: 1
  }
  kt_end(kt);
}

__global__ void __launch_bounds__(256)
k_opt_clip(const float* __restrict__ g, float* __restrict__ w, float* __restrict__ s, int64_t n4, const OptArgs opt,
           const float* __restrict__ clip, const KTrace kt) {
  const int64_t i4 = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
  kt_begin(kt);
  pdl_wait();
  pdl_launch_dependents();
  if (i4 < n4) {
    const int64_t i = i4 * 4;
    const float4 gv = *reinterpret_cast<const float4*>(g + i);
    float nw[4];
    opt_update_vec<4, true>(opt, opt_step_scalar(opt), reinterpret_cast<const float*>(&gv), nw, w + i, s + i,
                            __ldcg(clip));
  }
  kt_end(kt);
}

__global__ void k_iota(int32_t* a, int32_t* b, int n, int mult) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    a[i] = i;
    b[i] = i * mult;
  }
}

__global__ void k_zero_rows(float* q, int from, int to, int A) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < (to - from) * A) q[from * A + i] = 0.f;
}

static inline unsigned cdiv(int64_t a, int64_t b) { return unsigned((a + b - 1) / b); }
static inline int round_up(int a, int b) { return (a + b - 1) / b * b; }

#define B2_TRY(expr)          \
  do {                        \
    int rc__ = (expr);        \
    if (rc__) return rc__;    \
  } while (0)

template <class P, int BM, int BN, int BK, int TM, int TN>
static int launch_gemm(const char* label, const P& p, int M, int N, int Z, cudaStream_t st) {
  dim3 grid(cdiv(M, BM), cdiv(N, BN), Z);
  ++g_launch_count;
  k_simt_gemm<P, BM, BN, BK, TM, TN><<<grid, (BM / TM) * (BN / TN), 0, st>>>(p);
  B2_LAUNCH_CHECK();
  B2_PROF(label, st);
  return B200DQN_OK;
}

// Where the first conv layer reads its frames: in place from the ring (fused) or from staged states.
// crop: the random-shift crop offsets of each source ([nb][2] (dy, dx) int32, slot 0's then slot 1's), nullptr when
// the states are not shifted (augmentation off, predict).
struct FrameSource {
  const uint8_t* src[2];
  const int32_t* idx[2];
  int shift[2];
  const int32_t* crop[2] = {};
};

// conv1's forward on the SIMT engine for `nets` slots: slot 2 (Double DQN) reads slot 1's frames and crop offsets
static int conv1_fwd_simt(b200dqn_net* n, const FrameSource& fs, const float* const w[3], int nets, int rows,
                          cudaStream_t st) {
  auto fill = [&](Conv1Fwd& p) {
    for (int z = 0; z < 3; ++z) {
      const int f = z ? 1 : 0;
      p.src[z] = fs.src[f]; p.idx[z] = fs.idx[f]; p.shift[z] = fs.shift[f];
      p.w[z] = w[z] + n->lt.off[0]; p.out[z] = n->d_h1[z];
    }
    p.nb = rows;
    p.k1 = n->lt.rows[0];
  };
  if (fs.crop[0]) {
    Conv1FwdCrop p;
    fill(p);
    p.crop[0] = fs.crop[0]; p.crop[1] = fs.crop[1]; p.crop[2] = fs.crop[1];
    return launch_gemm<Conv1FwdCrop, 64, 32, 16, 4, 2>("conv1_fwd", p, rows * kP1 * kP1, kC1, nets, st);
  }
  Conv1Fwd p;
  fill(p);
  return launch_gemm<Conv1Fwd, 64, 32, 16, 4, 2>("conv1_fwd", p, rows * kP1 * kP1, kC1, nets, st);
}

// conv2 and conv3's forward on the SIMT engine for `nets` slots
static int conv23_fwd_simt(b200dqn_net* n, const float* const w[3], int nets, int rows, cudaStream_t st) {
  const LayerTable& lt = n->lt;
  {
    using P = ConvFwd<kP1, kC1, 4, 2, kC2>;
    P p;
    for (int z = 0; z < 3; ++z) { p.in[z] = n->d_h1[z]; p.w[z] = w[z] + lt.off[1]; p.out[z] = n->d_h2[z]; }
    p.nb = rows;
    B2_TRY((launch_gemm<P, 32, 64, 16, 2, 4>("conv2_fwd", p, rows * kP2 * kP2, kC2, nets, st)));
  }
  using P = ConvFwd<kP2, kC2, 3, 1, kC3>;
  P p;
  for (int z = 0; z < 3; ++z) { p.in[z] = n->d_h2[z]; p.w[z] = w[z] + lt.off[2]; p.out[z] = n->d_h3[z]; }
  p.nb = rows;
  return launch_gemm<P, 32, 64, 16, 2, 4>("conv3_fwd", p, rows * kP3 * kP3, kC3, nets, st);
}

// fc1's forward on the SIMT engine at width W (kHidden, or kDuelHidden on a dueling net)
template <int W>
static int fc1_fwd_simt(b200dqn_net* n, const float* const w[3], int nets, int rows, cudaStream_t st) {
  Fc1Fwd<W> p;
  for (int z = 0; z < 3; ++z) { p.in[z] = n->d_h3[z]; p.w[z] = w[z] + n->lt.off[3]; }
  p.part = n->d_fc1part; p.nb = rows; p.splits = kFc1Splits; p.kchunk = kFc1Chunk;
  return launch_gemm<Fc1Fwd<W>, 32, 64, 16, 2, 4>("fc1_fwd", p, rows, W, nets * kFc1Splits, st);
}

// fc1's forward on the SIMT engine on IQN / FQF modulated rows: `nets` slots of `rows` rows, slot z's at in[z]
static int fc1_fwd_x_simt(b200dqn_net* n, const float* const in[3], const float* const w[3], int nets, int rows,
                          cudaStream_t st) {
  Fc1Fwd<kHidden> p;
  for (int z = 0; z < 3; ++z) { p.in[z] = in[z]; p.w[z] = w[z] + n->lt.off[3]; }
  p.part = n->d_fc1part; p.nb = rows; p.splits = kFc1Splits; p.kchunk = kFc1Chunk;
  return launch_gemm<Fc1Fwd<kHidden>, 32, 64, 16, 2, 4>("fc1_fwd", p, rows, kHidden, nets * kFc1Splits, st);
}

// fc1's forward on the IQN / FQF modulated rows X: `nets` slots (slot 1's X at ld rows past slot 0's) of `rows`
// expanded rows, `splits` the k-split count the tensor-core engine was given
static int fc1_fwd_x(b200dqn_net* n, int nets, int rows, int ld, int splits, cudaStream_t st) {
  if (n->cfg.math_mode == B200DQN_MATH_TCGEN05) return umma_fc1_fwd_iqn(n, nets, rows, splits, st);
  const float* x[3] = {n->d_x, n->d_x + int64_t(ld) * kFlat, n->d_x};
  const float* w[3] = {n->d_w, n->d_tw, n->d_w};
  return fc1_fwd_x_simt(n, x, w, nets, rows, st);
}

// The conv trunk for `nets` network slots of `rows` samples, and fc1 on H3 unless trunk_only (an IQN or FQF head runs
// fc1 on its modulated rows instead), on whichever engine math_mode selects.  One GPU: the tensor-core forward launches
// are links of the critical chain (umma_forward picks the ones that release early).
static int forward_trunk(b200dqn_net* n, const FrameSource& fs, int nets, int rows, cudaStream_t st, bool trunk_only) {
  if (n->cfg.math_mode == B200DQN_MATH_TCGEN05)
    return umma_forward(n, fs.src, fs.idx, fs.shift, fs.crop, nets, rows, st, n->world == 1, trunk_only);
  const float* w[3] = {n->d_w, n->d_tw, n->d_w};
  B2_TRY(conv1_fwd_simt(n, fs, w, nets, rows, st));
  B2_TRY(conv23_fwd_simt(n, w, nets, rows, st));
  if (trunk_only) return B200DQN_OK;
  return n->dueling ? fc1_fwd_simt<kDuelHidden>(n, w, nets, rows, st) : fc1_fwd_simt<kHidden>(n, w, nets, rows, st);
}

// fc2 of a per-action head (C51, QR, REM) or of the IQN / FQF rows: `nets` slots of `rows` rows from the fc1 partials
// at `splits` k-splits, slot z's H4 at h4[z] and weights at w[z], into out (slot stride ld rows) at `ncols` columns
static int fc2_dist(b200dqn_net* n, int nets, int rows, int ld, int splits, float* const h4[2],
                    const float* const w[2], float* out, int ncols, const char* prof, cudaStream_t st) {
  const int64_t o = n->lt.off[4];
  B2_CHECK_CUDA(launch_pdl(k_fc2_dist, dim3(cdiv(rows, kDistTB), cdiv(ncols, kDistTN), nets), dim3(256), 0, st,
                           (const float*)n->d_fc1part, splits, rows, ld, h4[0], h4[1], w[0] + o, w[1] + o, out, ncols,
                           ktrace_slot("fc2_dist")));
  B2_PROF(prof, st);
  return B200DQN_OK;
}

// Calls f(std::integral_constant<int, S>{}, std::bool_constant<N>{}) with the instantiation <S, N> of a head kernel
// for `slots` network slots and the n-step flag.  Every head is instantiated at S = 2; kOther lists the other slot
// counts it has: 3 (Double DQN, the Munchausen target pass) and 1 (predict, one-step only).  An unlisted count takes 2.
// The instantiations are made in the order 3, 2, 1, the order of the kernels in the library.
template <int... kOther, class F>
static auto with_head(int slots, bool nstep, F&& f) {
  auto at = [&](auto s) { return nstep ? f(s, std::true_type{}) : f(s, std::false_type{}); };
  if constexpr (((kOther == 3) || ...)) {
    if (slots == 3) return at(std::integral_constant<int, 3>{});
  }
  if constexpr (((kOther == 1) || ...)) {
    if (slots != 1) return at(std::integral_constant<int, 2>{});
    return f(std::integral_constant<int, 1>{}, std::false_type{});
  } else {
    return at(std::integral_constant<int, 2>{});
  }
}

// Side branches of a step on a stream: a draw that reads only its counter, or the Munchausen target pass, which reads
// only weights and frames, forks from st onto a side stream and joins st later, overlapping the chain.  Work on a branch
// gets ordinary dependencies (see NoPdlScope).  Branches are off without a stream, on the serial schedule and under the
// event profiler.
static bool branches_on(const b200dqn_net* n, cudaStream_t st) { return n->use_branches && st != nullptr && !g_prof_on; }

// body(s) on a branch forked from st when `on`: on n->side[side], between events ev[e] (the fork, on st) and ev[e + 1]
// (its end, on the branch, returned in *done).  Otherwise body(st) runs in line and *done is nullptr.
template <class F>
static int fork_branch(b200dqn_net* n, cudaStream_t st, bool on, int side, int e, cudaEvent_t* done, F&& body) {
  *done = nullptr;
  if (!on) return body(st);
  cudaStream_t s = n->side[side];
  B2_CHECK_CUDA(cudaEventRecord(n->ev[e], st));
  B2_CHECK_CUDA(cudaStreamWaitEvent(s, n->ev[e], 0));
  {
    NoPdlScope branch;
    B2_TRY(body(s));
  }
  B2_CHECK_CUDA(cudaEventRecord(n->ev[e + 1], s));
  *done = n->ev[e + 1];
  return B200DQN_OK;
}

// st waits for a branch's end `done` (nothing when the branch ran in line)
static int join_branch(cudaStream_t st, cudaEvent_t done) {
  if (done) B2_CHECK_CUDA(cudaStreamWaitEvent(st, done, 0));
  return B200DQN_OK;
}

// ... and launch(), the first launch on st that reads the branch's work, gets ordinary dependencies on both
template <class F>
static int join_branch(cudaStream_t st, cudaEvent_t done, F&& launch) {
  B2_TRY(join_branch(st, done));
  if (!done) return launch();
  NoPdlScope joined;
  return launch();
}

// The IQN forward for `nets` slots of `rows` samples: tau and phi, the conv trunk at `rows`, then X = psi
// phi, fc1, fc2 and the head at rows * per expanded rows.  phi depends only on tau and We, so on a stream the draw and
// the embedding run on their own branch from the head of the forward and join before the modulation.
static int forward_iqn(b200dqn_net* n, const FrameSource& fs, int nets, int rows, cudaStream_t st,
                       const HeadTrainArgs& td) {
  const LayerTable& lt = n->lt;
  const float* w[3] = {n->d_w, n->d_tw, n->d_w};
  const int per = td.enable ? n->iqn_n : n->iqn_k, R = rows * per, ld = n->iqn_rows;
  cudaEvent_t embedded;
  B2_TRY(fork_branch(n, st, branches_on(n, st), 0, 15, &embedded, [&](cudaStream_t sP) {
    B2_CHECK_CUDA(launch_pdl(k_iqn_tau, dim3(1), dim3(1024), 0, sP, n->d_tau_ctr, (unsigned long long)n->cfg.tau_seed,
                             nets, rows, per, ld, n->d_tau, ktrace_slot("iqn_tau")));
    B2_CHECK_CUDA(launch_pdl(k_iqn_phi, dim3(cdiv(R, kIqnTB), nets), dim3(256), 0, sP, (const float*)n->d_tau, R, ld,
                             (const float*)n->d_we, (const float*)n->d_twe, n->d_cos, n->d_phi, ktrace_slot("iqn_phi")));
    B2_PROF("iqn_tau+phi", sP);
    return B200DQN_OK;
  }));
  const bool tc = n->cfg.math_mode == B200DQN_MATH_TCGEN05;
  // the tensor-core fc1 picks its split count by row count; it is taken at the full minibatch, so a predict on fewer
  // live rows sums every row as the full one does
  const int splits = tc ? umma_fc1_splits(n->nb * per) : kFc1Splits;
  B2_TRY(forward_trunk(n, fs, nets, rows, st, true));
  const int64_t total = int64_t(nets) * R * kFlat;
  B2_TRY(join_branch(st, embedded, [&] {
    B2_CHECK_CUDA(launch_pdl(k_iqn_mod, dim3(unsigned(std::min<int64_t>(cdiv(total, 256), int64_t(n->sm_count) * 16))),
                             dim3(256), 0, st, (const float*)n->d_h3[0], (const float*)n->d_h3[1],
                             (const float*)n->d_phi, n->d_x, n->d_x16, nets, R, per, ld, ktrace_slot("iqn_mod")));
    return B200DQN_OK;
  }));
  B2_PROF("iqn_mod", st);
  B2_TRY(fc1_fwd_x(n, nets, R, ld, splits, st));
  B2_TRY(fc2_dist(n, nets, R, ld, splits, n->d_h4, w, n->d_iqn_theta, n->A, "fc2_dist", st));
  const IqnArgs ia{per, ld, float(n->cfg.clip_error), n->d_tau, n->d_iqn_tq, n->d_iqn_qgrad, n->d_act_rows};
  const bool nstep = td.enable && td.nstep > 1;
  B2_CHECK_CUDA(with_head<1>(nets, nstep, [&](auto s, auto ns) {
    return launch_pdl(k_head_iqn<decltype(s)::value, decltype(ns)::value>, dim3(rows), dim3(kHidden), 0, st,
                      (const float*)n->d_iqn_theta, nets, (const float*)n->d_h4[0], w[0] + lt.off[4], n->d_q[0],
                      n->d_q[1], n->A, ia, td, ktrace_slot("head_iqn"));
  }));
  B2_PROF(td.enable ? "head_iqn(td+fc2_bwd)" : "head_iqn", st);
  return B200DQN_OK;
}

// The FQF forward for `nets` slots of `rows` samples, every launch on st (b200dqn.h's FQF rules): the conv trunk, the
// fraction proposal from the online psi, then phi, X, fc1 and fc2 of both slots at tauhat, and in a train step the
// boundary pass (the online network at tau_1..tau_{N-1}) before the head, all in line: tauhat depends on the trunk, and
// the boundary pass reads the weights the step's updates overwrite, so nothing here can leave the chain.
static int forward_fqf(b200dqn_net* n, const FrameSource& fs, int nets, int rows, cudaStream_t st,
                       const HeadTrainArgs& td) {
  const LayerTable& lt = n->lt;
  const float* w[3] = {n->d_w, n->d_tw, n->d_w};
  const int N = n->fqf_n, R = rows * N, ld = n->iqn_rows, Rb = rows * (N - 1);
  const bool tc = n->cfg.math_mode == B200DQN_MATH_TCGEN05;
  // split counts are taken at the full minibatch, so a predict on fewer live rows sums every row as the full one does
  const int splits = tc ? umma_fc1_splits(n->nb * N) : kFc1Splits;
  B2_TRY(forward_trunk(n, fs, nets, rows, st, true));
  B2_CHECK_CUDA(launch_pdl(k_fqf_fraction, dim3(rows), dim3(256), 0, st, (const float*)n->d_h3[0], (const float*)n->d_wf,
                           N, nets, ld, n->d_fl, n->d_fq, n->d_ftau, n->d_tau, td.enable ? n->d_btau : nullptr,
                           ktrace_slot("fqf_fraction")));
  B2_PROF("fqf_fraction", st);
  B2_CHECK_CUDA(launch_pdl(k_iqn_phi, dim3(cdiv(R, kIqnTB), nets), dim3(256), 0, st, (const float*)n->d_tau, R, ld,
                           (const float*)n->d_we, (const float*)n->d_twe, n->d_cos, n->d_phi, ktrace_slot("iqn_phi")));
  B2_PROF("iqn_phi", st);
  const int64_t total = int64_t(nets) * R * kFlat;
  B2_CHECK_CUDA(launch_pdl(k_iqn_mod, dim3(unsigned(std::min<int64_t>(cdiv(total, 256), int64_t(n->sm_count) * 16))),
                           dim3(256), 0, st, (const float*)n->d_h3[0], (const float*)n->d_h3[1], (const float*)n->d_phi,
                           n->d_x, n->d_x16, nets, R, N, ld, ktrace_slot("iqn_mod")));
  B2_PROF("iqn_mod", st);
  B2_TRY(fc1_fwd_x(n, nets, R, ld, splits, st));
  B2_TRY(fc2_dist(n, nets, R, ld, splits, n->d_h4, w, n->d_iqn_theta, n->A, "fc2_dist", st));
  if (td.enable) {   // the boundary pass: the online network at tau_1..tau_{N-1}, on buffers of its own
    B2_CHECK_CUDA(launch_pdl(k_iqn_phi, dim3(cdiv(Rb, kIqnTB), 1), dim3(256), 0, st, (const float*)n->d_btau, Rb, Rb,
                             (const float*)n->d_we, (const float*)n->d_we, n->d_bcos, n->d_bphi, ktrace_slot("iqn_phi")));
    B2_PROF("fqf_bnd_phi", st);
    B2_CHECK_CUDA(launch_pdl(k_iqn_mod, dim3(unsigned(std::min<int64_t>(cdiv(int64_t(Rb) * kFlat, 256),
                                                                         int64_t(n->sm_count) * 16))),
                             dim3(256), 0, st, (const float*)n->d_h3[0], (const float*)n->d_h3[0],
                             (const float*)n->d_bphi, n->d_bx, n->d_bx16, 1, Rb, N - 1, Rb, ktrace_slot("iqn_mod")));
    B2_PROF("fqf_bnd_mod", st);
    const int bsplits = tc ? umma_fc1_splits(Rb) : kFc1Splits;
    const float* bx[3] = {n->d_bx, n->d_bx, n->d_bx};
    const float* bw[3] = {w[0], w[0], w[0]};
    B2_TRY(tc ? umma_fc1_fwd_fqf_boundary(n, Rb, bsplits, st) : fc1_fwd_x_simt(n, bx, bw, 1, Rb, st));
    float* bh4[2] = {n->d_bh4, n->d_bh4};
    B2_TRY(fc2_dist(n, 1, Rb, Rb, bsplits, bh4, bw, n->d_btheta, n->A, "fqf_bnd_fc2", st));
  }
  const IqnArgs ia{N, ld, float(n->cfg.clip_error), n->d_tau, n->d_iqn_tq, n->d_iqn_qgrad, n->d_act_rows};
  const bool adam = n->cfg.optimizer == B200DQN_OPT_ADAM;
  const FqfArgs fa{n->d_ftau, n->d_fq, n->d_btheta, n->d_fg, n->d_fdl, float(n->cfg.fraction_lr),
                   adam ? n->d_optscal + 2 : nullptr};
  const bool nstep = td.enable && td.nstep > 1;
  B2_CHECK_CUDA(with_head<1>(nets, nstep, [&](auto s, auto ns) {
    return launch_pdl(k_head_fqf<decltype(s)::value, decltype(ns)::value>, dim3(rows), dim3(kHidden), 0, st,
                      (const float*)n->d_iqn_theta, nets, (const float*)n->d_h4[0], w[0] + lt.off[4], n->d_q[0],
                      n->d_q[1], n->A, ia, fa, td, ktrace_slot("head_fqf"));
  }));
  B2_PROF(td.enable ? "head_fqf(td+fc2_bwd)" : "head_fqf", st);
  return B200DQN_OK;
}

// The IQN backward between fc1's dgrad and conv3's (on st): dpsi into dZ3 and dphi; then dWe and the embedding's update,
// on side stream sW when given (its own branch: nothing later in the step reads We), else in line.  An FQF net adds
// dW_f and the fraction layer's update on the same branch.  Under gradient-norm clipping the embedding's update waits
// for c32 (clip_apply); the fraction layer's does not.
static int iqn_backward(b200dqn_net* n, int rows, cudaStream_t st, cudaStream_t sW, bool update) {
  __half* dpsi16 = nullptr;
  int64_t dpsi_lo = 0;
  umma_dz3_planes(n, &dpsi16, &dpsi_lo);
  B2_CHECK_CUDA(launch_pdl(k_iqn_mod_bwd, dim3(cdiv(int64_t(rows) * kFlat, 256)), dim3(256), 0, st,
                           (const float*)n->d_dx, (const float*)n->d_phi, (const float*)n->d_h3[0], n->d_dz3, dpsi16,
                           dpsi_lo, n->d_dphi, rows, n->iqn_n, ktrace_slot("iqn_mod_bwd")));
  B2_PROF("iqn_mod_bwd", st);
  cudaStream_t s = st;
  if (sW) {
    B2_CHECK_CUDA(cudaEventRecord(n->ev[8], st));
    B2_CHECK_CUDA(cudaStreamWaitEvent(sW, n->ev[8], 0));
    s = sW;
  }
  NoPdlScope side;
  OptArgs o = make_opt_args(n, rows);
  o.plane = int64_t(kIqnCos) * kFlat;
  B2_CHECK_CUDA(launch_pdl(k_iqn_we, dim3(cdiv(kFlat, kWeCols)), dim3(256), 0, s, (const float*)n->d_cos,
                           (const float*)n->d_dphi, rows * n->iqn_n, n->d_weg, n->d_we, n->d_wes, update && !n->clip ? 1 : 0, o,
                           ktrace_slot("iqn_we")));
  B2_PROF("iqn_we", s);
  if (n->fqf_n) {
    OptArgs of = make_opt_args(n, rows);
    of.lr = float(n->cfg.fraction_lr);
    of.adam_l = n->d_optscal + 2;   // the FQF head's Adam scalar at fraction_lr
    of.plane = int64_t(n->fqf_n) * kFlat;
    B2_CHECK_CUDA(launch_pdl(k_fqf_wf, dim3(cdiv(int64_t(n->fqf_n) * kFlat, 256)), dim3(256), 0, s,
                             (const float*)n->d_fdl, (const float*)n->d_h3[0], rows, n->fqf_n, n->d_wfg, n->d_wf,
                             n->d_wfs, update ? 1 : 0, of, ktrace_slot("fqf_wf")));
    B2_PROF("fqf_wf", s);
  }
  return B200DQN_OK;
}

// Model.fprop for `nets` network slots on `rows` samples: z = 0 online (prestates), z = 1 target (poststates) and,
// for a Double DQN train step (nets = 3), z = 2 online on slot 1's frames (the poststates).
// join (Munchausen or REM train step on a stream): the end of the target pass's or the mixture draw's branch, joined
// before the head.
static int forward(b200dqn_net* n, const FrameSource& fs, int nets, int rows, cudaStream_t st,
                   const HeadTrainArgs& td, cudaEvent_t join = nullptr) {
  if (n->fqf_n) return forward_fqf(n, fs, nets, rows, st, td);
  if (n->iqn_n) return forward_iqn(n, fs, nets, rows, st, td);
  const LayerTable& lt = n->lt;
  const float* w[3] = {n->d_w, n->d_tw, n->d_w};
  B2_TRY(forward_trunk(n, fs, nets, rows, st, false));
  const int fc1_splits = n->cfg.math_mode == B200DQN_MATH_TCGEN05 ? umma_fc1_splits(rows) : kFc1Splits;
  const bool nstep = td.enable && td.nstep > 1;
  if (n->dueling) {
    B2_CHECK_CUDA(with_head<3>(nets, nstep, [&](auto s, auto ns) {
      return launch_pdl(k_head_duel<decltype(s)::value, decltype(ns)::value>, dim3(rows), dim3(kDuelHidden), 0, st,
                        (const float*)n->d_fc1part, fc1_splits, rows, nets, n->nb, n->d_h4[0], n->d_h4[1],
                        w[0] + lt.off[4], w[1] + lt.off[4], n->d_q[0], n->d_q[1], n->d_q[2], n->d_va, n->A, td,
                        ktrace_slot("head_duel"));
    }));
    B2_PROF(td.enable ? "head_duel(td+fc2_bwd)" : "head_duel", st);
    return B200DQN_OK;
  }
  if (n->atoms) {
    B2_TRY(fc2_dist(n, nets, rows, n->nb, fc1_splits, n->d_h4, w, n->d_logits, n->fc2_cols(), "fc2_dist", st));
    const DistArgs da{n->atoms, n->cfg.v_min, n->cfg.v_max, n->dz, n->d_probs, n->d_tdist, n->d_lgrad, n->d_act_rows};
    B2_CHECK_CUDA((with_head<3, 1>(nets, nstep, [&](auto s, auto ns) {
      return launch_pdl(k_head_dist<decltype(s)::value, decltype(ns)::value>, dim3(rows), dim3(kHidden), 0, st,
                        (const float*)n->d_logits, n->nb, nets, (const float*)n->d_h4[0], w[0] + lt.off[4], n->d_q[0],
                        n->d_q[1], n->d_q[2], n->A, da, td, ktrace_slot("head_dist"));
    })));
    B2_PROF(td.enable ? "head_dist(td+fc2_bwd)" : "head_dist", st);
    return B200DQN_OK;
  }
  if (n->quantiles) {
    B2_TRY(fc2_dist(n, nets, rows, n->nb, fc1_splits, n->d_h4, w, n->d_theta, n->fc2_cols(), "fc2_dist", st));
    const QrArgs qa{n->quantiles, float(n->cfg.clip_error), n->d_tquant, n->d_qgrad, n->d_act_rows};
    B2_CHECK_CUDA((with_head<3, 1>(nets, nstep, [&](auto s, auto ns) {
      return launch_pdl(k_head_qr<decltype(s)::value, decltype(ns)::value>, dim3(rows), dim3(kHidden), 0, st,
                        (const float*)n->d_theta, n->nb, nets, (const float*)n->d_h4[0], w[0] + lt.off[4], n->d_q[0],
                        n->d_q[1], n->d_q[2], n->A, qa, td, ktrace_slot("head_qr"));
    })));
    B2_PROF(td.enable ? "head_qr(td+fc2_bwd)" : "head_qr", st);
    return B200DQN_OK;
  }
  if (n->rem_k) {
    B2_TRY(fc2_dist(n, nets, rows, n->nb, fc1_splits, n->d_h4, w, n->d_theta, n->fc2_cols(), "fc2_dist", st));
    if (!td.enable && n->boot) {   // predict at the active head, read on the device
      B2_CHECK_CUDA(launch_pdl(k_boot_predict, dim3(rows), dim3(32), 0, st, (const float*)n->d_theta, n->A, n->rem_k,
                               (const int32_t*)n->d_boot_head, n->d_q[0], ktrace_slot("boot_predict")));
      B2_PROF("boot_predict", st);
      return B200DQN_OK;
    }
    if (n->boot) {
      const BootArgs ba{(unsigned long long)n->cfg.bootstrap_seed, n->cfg.bootstrap_p, n->d_boot_mask, n->d_boot_y,
                        n->d_boot_delta, n->d_rem_grad, n->d_act_rows};
      B2_CHECK_CUDA(with_head<3>(nets, nstep, [&](auto s, auto ns) {
        return launch_pdl(k_head_boot<decltype(s)::value, decltype(ns)::value>, dim3(rows), dim3(kHidden), 0, st,
                          (const float*)n->d_theta, n->nb, nets, (const float*)n->d_h4[0], w[0] + lt.off[4], n->d_q[0],
                          n->d_q[1], n->d_q[2], n->A, n->rem_k, ba, td, ktrace_slot("head_boot"));
      }));
      B2_PROF("head_boot(td+fc2_bwd)", st);
      return B200DQN_OK;
    }
    if (!td.enable) {   // predict: the mean over the K heads, the quantile-regression head's Q
      const QrArgs qa{n->rem_k, 0.f, nullptr, nullptr, nullptr};
      B2_CHECK_CUDA(launch_pdl(k_head_qr<1, false>, dim3(rows), dim3(kHidden), 0, st, (const float*)n->d_theta, n->nb,
                               nets, (const float*)n->d_h4[0], w[0] + lt.off[4], n->d_q[0], n->d_q[1], n->d_q[2], n->A,
                               qa, td, ktrace_slot("head_qr")));
      B2_PROF("head_qr", st);
      return B200DQN_OK;
    }
    B2_TRY(join_branch(st, join, [&] {   // the mixture draw's branch
      return with_head<3>(nets, nstep, [&](auto s, auto ns) {
        B2_CHECK_CUDA(launch_pdl(k_head_rem<decltype(s)::value, decltype(ns)::value>, dim3(rows), dim3(kHidden), 0, st,
                                 (const float*)n->d_theta, n->nb, nets, (const float*)n->d_h4[0], w[0] + lt.off[4],
                                 n->d_q[0], n->d_q[1], n->d_q[2], n->A, n->rem_k, (const float*)n->d_rem_alpha,
                                 n->d_rem_grad, n->d_act_rows, td, ktrace_slot("head_rem")));
        return B200DQN_OK;
      });
    }));
    B2_PROF("head_rem(td+fc2_bwd)", st);
    return B200DQN_OK;
  }
  if (n->munchausen && td.enable) {   // predict takes the scalar head below
    // slot 2, the target network on the prestates, exists with a separate target network only (train_step's pass)
    const bool pre = n->d_tw != n->d_w;
    const MdqnArgs ma{n->cfg.munchausen_alpha, n->cfg.munchausen_tau, n->cfg.munchausen_clip, n->d_q[2], n->d_tdtarget};
    B2_TRY(join_branch(st, join, [&] {   // the target pass's branch
      return with_head<3>(pre ? 3 : 2, nstep, [&](auto s, auto ns) {
        B2_CHECK_CUDA(launch_pdl(k_head_mdqn<decltype(s)::value, decltype(ns)::value>, dim3(rows), dim3(kHidden), 0,
                                 st, (const float*)n->d_fc1part, fc1_splits, rows, n->d_h4[0], n->d_h4[1],
                                 w[0] + lt.off[4], w[1] + lt.off[4], n->d_q[0], n->d_q[1], n->A, ma, td,
                                 ktrace_slot("head_mdqn")));
        return B200DQN_OK;
      });
    }));
    B2_PROF("head_mdqn(td+fc2_bwd)", st);
    return B200DQN_OK;
  }
  B2_CHECK_CUDA(with_head<3>(nets, nstep, [&](auto s, auto ns) {
    return launch_pdl(k_head<decltype(s)::value, decltype(ns)::value>, dim3(rows), dim3(kHidden), 0, st,
                      (const float*)n->d_fc1part, fc1_splits, rows, nets, n->d_h4[0], n->d_h4[1], w[0] + lt.off[4],
                      w[1] + lt.off[4], n->d_q[0], n->d_q[1], n->d_q[2], n->A, td, ktrace_slot("head"));
  }));
  B2_PROF(td.enable ? "head(fc2+td+fc2_bwd)" : "fc2_fwd", st);
  return B200DQN_OK;
}

// The Munchausen target pass: the target network on slot 0's frames (the prestates) as forward()'s backbone launches
// with one network slot (nets = 1) and remapped pointers, into the third slot's activations (SIMT) or fp16 planes
// (tensor cores) and slot 2's region of the three-slot fc1 partials, which k_head_mdqn<3, .> sums.
static int forward_target_pre(b200dqn_net* n, const FrameSource& fs, int rows, cudaStream_t st) {
  if (n->cfg.math_mode == B200DQN_MATH_TCGEN05)
    return umma_forward_target_pre(n, fs.src[0], fs.idx[0], fs.shift[0], fs.crop[0], rows, st);
  const LayerTable& lt = n->lt;
  const float* w = n->d_tw;
  int rc;
  {
    auto fill = [&](Conv1Fwd& p) {
      p.src[0] = fs.src[0]; p.idx[0] = fs.idx[0]; p.shift[0] = fs.shift[0];
      p.w[0] = w + lt.off[0]; p.out[0] = n->d_h1[2];
      p.nb = rows;
      p.k1 = lt.rows[0];
    };
    if (fs.crop[0]) {   // the prestates, shifted by slot 0's offsets
      Conv1FwdCrop p{};
      fill(p);
      p.crop[0] = fs.crop[0];
      rc = launch_gemm<Conv1FwdCrop, 64, 32, 16, 4, 2>("conv1_fwd", p, rows * kP1 * kP1, kC1, 1, st);
    } else {
      Conv1Fwd p{};
      fill(p);
      rc = launch_gemm<Conv1Fwd, 64, 32, 16, 4, 2>("conv1_fwd", p, rows * kP1 * kP1, kC1, 1, st);
    }
    if (rc) return rc;
  }
  {
    using P = ConvFwd<kP1, kC1, 4, 2, kC2>;
    P p{};
    p.in[0] = n->d_h1[2]; p.w[0] = w + lt.off[1]; p.out[0] = n->d_h2[2];
    p.nb = rows;
    if ((rc = launch_gemm<P, 32, 64, 16, 2, 4>("conv2_fwd", p, rows * kP2 * kP2, kC2, 1, st))) return rc;
  }
  {
    using P = ConvFwd<kP2, kC2, 3, 1, kC3>;
    P p{};
    p.in[0] = n->d_h2[2]; p.w[0] = w + lt.off[2]; p.out[0] = n->d_h3[2];
    p.nb = rows;
    if ((rc = launch_gemm<P, 32, 64, 16, 2, 4>("conv3_fwd", p, rows * kP3 * kP3, kC3, 1, st))) return rc;
  }
  Fc1Fwd<kHidden> p{};   // 512 wide: a Munchausen net is not a dueling one
  p.in[0] = n->d_h3[2]; p.w[0] = w + lt.off[3];
  p.part = n->d_fc1part + int64_t(2) * kFc1Splits * rows * kHidden;
  p.nb = rows; p.splits = kFc1Splits; p.kchunk = kFc1Chunk;
  return launch_gemm<Fc1Fwd<kHidden>, 32, 64, 16, 2, 4>("fc1_fwd", p, rows, kHidden, kFc1Splits, st);
}

static int wgrad_chunk(int kred, int base) {
  int c = (kred + 31) / 32;
  if (c < base) c = base;
  return round_up(c, 16);
}

template <int W>
static int fc1_wgrad_simt(b200dqn_net* n, int rows, cudaStream_t st) {
  Fc1Wgrad<W> p{n->d_h3[0], n->d_dz4, n->d_part + n->lt.part_off[3], rows};
  return launch_gemm<Fc1Wgrad<W>, 64, 64, 16, 4, 4>("fc1_wgrad", p, kFlat, W, 1, st);
}

template <int W>
static int fc1_dgrad_simt(b200dqn_net* n, int rows, cudaStream_t st) {
  Fc1Dgrad<W> p{n->d_dz4, n->d_w + n->lt.off[3], n->d_h3[0], n->d_dz3, rows};
  return launch_gemm<Fc1Dgrad<W>, 32, 32, 16, 2, 2>("fc1_dgrad", p, rows, kFlat, 1, st);
}

enum BwdOp { kFc1Wgrad, kFc1Dgrad, kConv3Wgrad, kConv3Dgrad, kConv2Wgrad, kConv2Dgrad, kConv1Wgrad };

// One GEMM-shaped backward op on stream `st`, on whichever engine math_mode selects.  release_early (tensor-core
// engine): the op is a link of the single-GPU critical chain and lets its successor pre-launch right after its own
// dependency wait.
static int bwd_op(b200dqn_net* n, const FrameSource& fs, int rows, BwdOp op, cudaStream_t st,
                  bool release_early = false) {
  const LayerTable& lt = n->lt;
  const float* w = n->d_w;
  if (n->cfg.math_mode == B200DQN_MATH_TCGEN05)
    return umma_backward_op(n, int(op), fs.src[0], fs.idx[0], fs.shift[0], rows, st, release_early);
  switch (op) {
    case kFc1Wgrad:
      if (n->iqn_n) {   // IQN: fc1 ran on X at rows N expanded rows
        Fc1Wgrad<kHidden> p{n->d_x, n->d_dz4, n->d_part + lt.part_off[3], rows * n->iqn_n};
        return launch_gemm<Fc1Wgrad<kHidden>, 64, 64, 16, 4, 4>("fc1_wgrad", p, kFlat, kHidden, 1, st);
      }
      return n->dueling ? fc1_wgrad_simt<kDuelHidden>(n, rows, st) : fc1_wgrad_simt<kHidden>(n, rows, st);
    case kFc1Dgrad:
      if (n->iqn_n) {   // dX, masked by X > 0 (harmless: see rule 11 of b200dqn.h)
        Fc1Dgrad<kHidden> p{n->d_dz4, w + lt.off[3], n->d_x, n->d_dx, rows * n->iqn_n};
        return launch_gemm<Fc1Dgrad<kHidden>, 32, 32, 16, 2, 2>("fc1_dgrad", p, rows * n->iqn_n, kFlat, 1, st);
      }
      return n->dueling ? fc1_dgrad_simt<kDuelHidden>(n, rows, st) : fc1_dgrad_simt<kHidden>(n, rows, st);
    case kConv3Wgrad: {
      using P = ConvWgrad<kP2, kC2, 3, 1, kC3>;
      P p{n->d_h2[0], n->d_dz3, n->d_part + lt.part_off[2], rows, wgrad_chunk(rows * kP3 * kP3, 112)};
      return launch_gemm<P, 64, 64, 16, 4, 4>("conv3_wgrad", p, P::KW, kC3, lt.splits[2], st);
    }
    case kConv3Dgrad: {
      using P = ConvDgrad<kP2, kC2, 3, 1, kC3>;
      P p{n->d_dz3, w + lt.off[2], n->d_h2[0], n->d_dz2, rows};
      return launch_gemm<P, 32, 64, 16, 2, 4>("conv3_dgrad", p, rows * P::HC * P::HC, kC2, 1, st);
    }
    case kConv2Wgrad: {
      using P = ConvWgrad<kP1, kC1, 4, 2, kC2>;
      P p{n->d_h1[0], n->d_dz2, n->d_part + lt.part_off[1], rows, wgrad_chunk(rows * kP2 * kP2, 96)};
      return launch_gemm<P, 64, 64, 16, 4, 4>("conv2_wgrad", p, P::KW, kC2, lt.splits[1], st);
    }
    case kConv2Dgrad: {
      using P = ConvDgrad<kP1, kC1, 4, 2, kC2>;
      P p{n->d_dz2, w + lt.off[1], n->d_h1[0], n->d_dz1, rows};
      return launch_gemm<P, 64, 32, 16, 4, 2>("conv2_dgrad", p, rows * P::HC * P::HC, kC1, 4, st);
    }
    default: {
      Conv1Wgrad p{fs.src[0], fs.idx[0], fs.shift[0], n->d_dz1, n->d_part + lt.part_off[0], rows,
                   wgrad_chunk(rows * kP1 * kP1, 512), lt.rows[0]};
      if (fs.crop[0]) {   // the prestates as slot 0's forward saw them
        Conv1WgradCrop pc{p, fs.crop[0]};
        return launch_gemm<Conv1WgradCrop, 64, 32, 16, 4, 2>("conv1_wgrad", pc, lt.rows[0], kC1, lt.splits[0], st);
      }
      return launch_gemm<Conv1Wgrad, 64, 32, 16, 4, 2>("conv1_wgrad", p, lt.rows[0], kC1, lt.splits[0], st);
    }
  }
}

// RMSProp (or gradient reduction) over layers [l0, l1] on stream st; mode bits as in k_optimizer.
// The optimizer constants of this net (src/deepqnetwork.py:50-59; Neon's defaults for what the reference leaves unset)
OptArgs make_opt_args(const b200dqn_net* n, int rows) {
  OptArgs o{};
  o.kind = n->cfg.optimizer;
  o.nstates = n->n_states;
  o.bsz = float(rows * n->world);
  o.lr = float(n->cfg.learning_rate);
  o.decay = float(n->cfg.decay_rate);
  o.one_m_decay = float(1.0 - n->cfg.decay_rate);
  o.eps = 1e-6f;
  o.b1 = float(0.9); o.one_m_b1 = float(1.0 - 0.9);
  o.b2 = float(0.999); o.one_m_b2 = float(1.0 - 0.999);
  o.adam_eps = 1e-8f;
  o.adam_l = n->d_optscal;
  o.plane = n->n_params;
  return o;
}

// optimizer update (or gradient reduction) over layers [l0, l1] on stream st; mode bits as in k_optimizer.
static int optimizer_range(b200dqn_net* n, int l0, int l1, int mode, int rows, cudaStream_t st, const char* label) {
  const LayerTable& lt = n->lt;
  const int64_t b4 = lt.off[l0] / 4, e4 = lt.off[l1 + 1] / 4;
  B2_CHECK_CUDA(launch_pdl(k_optimizer, dim3(cdiv(e4 - b4, 256)), dim3(256), 0, st, lt, (const float*)n->d_part, n->d_g,
                           n->d_w, n->d_s, b4, e4, mode, make_opt_args(n, rows), ktrace_slot(label)));
  B2_PROF(label, st);
  if (mode & 4) return umma_pack_layers(n, 0, l0, l1, st);   // refresh the fp16 tile images of the updated layers
  return B200DQN_OK;
}

// batch-mean cost -> cost ring, step counter + 1 (once per train step, after the head, on any stream behind it)
static int cost_finish_on(b200dqn_net* n, int rows, cudaStream_t s) {
  NoPdlScope plain;
  b200dqn_replay* r = n->step_replay;     // the ring this step samples from (nullptr: host-supplied minibatch)
  B2_CHECK_CUDA(launch_pdl(k_cost_finish, dim3(1), dim3(256), 0, s, (const float*)n->d_rowcost, rows, n->d_cost, n->d_step,
                           n->h_res, (const uint32_t*)(r ? r->d_words : nullptr),
                           (volatile uint32_t*)(r ? r->h_words : nullptr), ktrace_slot("cost")));
  B2_PROF("cost", s);
  if (r && r->per_on)   // priorities of the sampled slots, after the head (td_err) on the same off-chain branch
    return launch_per_update(r, r->d_idx + n->rank * n->nb, n->d_td_err, rows, s);
  return B200DQN_OK;
}

// fc2 of a distributional, quantile or IQN net from the head's compact row partials (an IQN net has one per expanded
// row; the optimizer's batch size stays `rows`); mode bits as k_opt_fc2_dist's
static int opt_fc2_dist(b200dqn_net* n, int rows, int mode, cudaStream_t s, const char* label) {
  const LayerTable& lt = n->lt;
  const int blk = n->fc2_block();
  B2_CHECK_CUDA(launch_pdl(k_opt_fc2_dist, dim3(cdiv(int64_t(kHidden) * blk, 256), n->A), dim3(256), 0, s,
                           (const float*)n->d_part + lt.part_off[4], (const int32_t*)n->d_act_rows,
                           n->expanded(rows, true), n->A, blk,
                           n->d_g + lt.off[4], n->d_w + lt.off[4], n->d_s + lt.off[4], mode, make_opt_args(n, rows),
                           ktrace_slot(label)));
  B2_PROF(label, s);
  return B200DQN_OK;
}

// The update over layers [l0, l1] of the single-learner schedules (mode 1 | 4): fc2 of a distributional or quantile
// net goes through opt_fc2_dist, every other layer through optimizer_range.
static int update_range(b200dqn_net* n, int l0, int l1, int rows, cudaStream_t st, const char* label) {
  if (!n->fc2_block() || l1 < 4) return optimizer_range(n, l0, l1, 1 | 4, rows, st, label);
  if (l0 < 4) {
    const int rc = optimizer_range(n, l0, 3, 1 | 4, rows, st, label);
    if (rc) return rc;
  }
  return opt_fc2_dist(n, rows, 4, st, "opt_fc2_dist");
}

// fc2 update from the head's per-row partials (single-GPU schedules): 8-lane reduction, no image
static int opt_fc2_small(b200dqn_net* n, int rows, cudaStream_t s) {
  if (n->fc2_block()) return opt_fc2_dist(n, rows, 4, s, "opt_fc2_dist");
  const LayerTable& lt = n->lt;
  const int64_t size = lt.off[5] - lt.off[4];
  B2_CHECK_CUDA(launch_pdl(k_opt_small, dim3(cdiv(size / 4, 32)), dim3(256), 0, s, (const float*)n->d_part + lt.part_off[4],
                           lt.splits[4], size, n->d_w + lt.off[4], n->d_s + lt.off[4], make_opt_args(n, rows),
                           ktrace_slot("opt_fc2")));
  B2_PROF("opt_fc2", s);
  return B200DQN_OK;
}

// Soft target update of `elems` parameters at w / tw (elems a multiple of 4).
static int soft_blend_range(b200dqn_net* n, const float* w, float* tw, int64_t elems, float c, float t, cudaStream_t st,
                            const char* label) {
  const int64_t n4 = elems / 4;
  B2_CHECK_CUDA(launch_pdl(k_soft_blend, dim3(cdiv(n4, 256)), dim3(256), 0, st, w, tw, n4, c, t, ktrace_slot(label)));
  B2_PROF(label, st);
  return B200DQN_OK;
}

// Soft target update of layers [l0, l1] on st: on the tensor-core engine conv1..fc1 one fused blend-and-pack launch
// each, the fp32-only layers (fc2; every layer on the SIMT engine) one blend over their contiguous range.
static int soft_update_layers(b200dqn_net* n, int l0, int l1, float c, float t, cudaStream_t st) {
  const LayerTable& lt = n->lt;
  if (n->cfg.math_mode == B200DQN_MATH_TCGEN05)
    for (; l0 <= l1 && l0 < 4; ++l0) B2_TRY(umma_soft_pack(n, l0, c, t, st));
  if (l0 > l1) return B200DQN_OK;
  static const char* const one[kLayers] = {"soft_c1", "soft_c2", "soft_c3", "soft_fc1", "soft_fc2"};
  return soft_blend_range(n, n->d_w + lt.off[l0], n->d_tw + lt.off[l0], lt.off[l1 + 1] - lt.off[l0], c, t, st,
                          l0 == l1 ? one[l0] : l0 == 3 ? "soft_fc" : "soft_layers");
}

// Soft target update of the IQN / FQF embedding and the FQF fraction layer on st (nothing on other nets).
static int soft_update_extra(b200dqn_net* n, float c, float t, cudaStream_t st) {
  if (n->iqn_n) B2_TRY(soft_blend_range(n, n->d_we, n->d_twe, int64_t(kIqnCos) * kFlat, c, t, st, "soft_we"));
  if (n->fqf_n) B2_TRY(soft_blend_range(n, n->d_wf, n->d_twf, int64_t(n->fqf_n) * kFlat, c, t, st, "soft_wf"));
  return B200DQN_OK;
}

// ---- global gradient-norm clipping (cfg.max_grad_norm > 0).  Layer 5 is the IQN / FQF embedding.
static int64_t clip_layer_size(const b200dqn_net* n, int l) {
  return l == kLayers ? int64_t(kIqnCos) * kFlat : n->lt.off[l + 1] - n->lt.off[l];
}

// the summed gradient of layer l the clipped step reads: the tensor-core engine's fc1 from its single wgrad partial (as
// umma_opt_fc1 reads it), the embedding from d_weg (k_iqn_we), every other layer from d_g after clip_layer_end's reduce
static const float* clip_grad_src(const b200dqn_net* n, int l) {
  if (l == kLayers) return n->d_weg;
  if (l == 3 && n->cfg.math_mode == B200DQN_MATH_TCGEN05 && n->lt.splits[3] == 1) return n->d_part + n->lt.part_off[3];
  return n->d_g + n->lt.off[l];
}

// the end of layer l's branch in a clipped step: its partials summed into d_g, then its sum of squares
static int clip_layer_end(b200dqn_net* n, int l, int rows, cudaStream_t st) {
  static const char* const red[kLayers] = {"reduce_conv1", "reduce_conv2", "reduce_conv3", "reduce_fc1", "reduce_fc2"};
  static const char* const sq[kLayers + 1] = {"grad_sq_c1", "grad_sq_c2", "grad_sq_c3", "grad_sq_fc1", "grad_sq_fc2",
                                              "grad_sq_we"};
  if (l == 4 && n->fc2_block()) B2_TRY(opt_fc2_dist(n, rows, 2, st, "reduce_fc2_dist"));
  else if (l < kLayers && clip_grad_src(n, l) == n->d_g + n->lt.off[l])
    B2_TRY(optimizer_range(n, l, l, 1 | 2, rows, st, red[l]));
  const int64_t n4 = clip_layer_size(n, l) / 4;
  B2_CHECK_CUDA(launch_pdl(k_grad_sq, dim3(cdiv(n4 * 4, kSqChunk)), dim3(256), 0, st, clip_grad_src(n, l), n4,
                           make_opt_args(n, rows).bsz, n->d_clip + 8 + n->sq_base[l], ktrace_slot(sq[l])));
  B2_PROF(sq[l], st);
  return B200DQN_OK;
}

// N and c32 from every layer's partials (one CTA), once every clip_layer_end of the step has run
static int clip_scale(b200dqn_net* n, cudaStream_t st) {
  SqLayout lay{};
  for (int l = 0; l < 7; ++l) lay.base[l] = n->sq_base[l];
  B2_CHECK_CUDA(launch_pdl(k_clip_scale, dim3(1), dim3(256), 0, st, n->d_clip, lay, n->cfg.max_grad_norm,
                           ktrace_slot("clip_scale")));
  B2_PROF("clip_scale", st);
  return B200DQN_OK;
}

// the clipped update of layer l from clip_grad_src(n, l), with the tensor-core engine's image refresh: fc1 in one pass
// (k_opt_fc1_clip), the conv layers by their packers after k_opt_clip
static int clip_apply(b200dqn_net* n, int l, int rows, cudaStream_t st) {
  static const char* const lbl[kLayers + 1] = {"opt_conv1_clip", "opt_conv2_clip", "opt_conv3_clip", "opt_fc1_clip",
                                               "opt_fc2_clip", "opt_we_clip"};
  if (n->cfg.math_mode == B200DQN_MATH_TCGEN05 && l == 3)
    return umma_opt_fc1(n, rows, st, n->lt.splits[3] > 1, n->d_clip_c());
  OptArgs o = make_opt_args(n, rows);
  float* w = n->d_we, *s = n->d_wes;
  if (l == kLayers) o.plane = clip_layer_size(n, l);
  else w = n->d_w + n->lt.off[l], s = n->d_s + n->lt.off[l];
  const int64_t n4 = clip_layer_size(n, l) / 4;
  B2_CHECK_CUDA(launch_pdl(k_opt_clip, dim3(cdiv(n4, 256)), dim3(256), 0, st, clip_grad_src(n, l), w, s, n4, o,
                           (const float*)n->d_clip_c(), ktrace_slot(lbl[l])));
  B2_PROF(lbl[l], st);
  // the tensor-core engine's conv layers: their tile images from the new weights (forward; conv2 and conv3 also dgrad)
  return l < 3 ? umma_pack_layers(n, 0, l, l, st) : B200DQN_OK;
}

// the serial form: every layer's end, c32, then every clipped update, in order on st
static int clip_step_serial(b200dqn_net* n, int rows, cudaStream_t st) {
  const int last = n->iqn_n ? kLayers : kLayers - 1;
  for (int l = 0; l <= last; ++l) B2_TRY(clip_layer_end(n, l, rows, st));
  B2_TRY(clip_scale(n, st));
  for (int l = 0; l <= last; ++l) B2_TRY(clip_apply(n, l, rows, st));
  return B200DQN_OK;
}

// Model.bprop + optimizer.optimize for the online network (src/deepqnetwork.py:162-165).
//
// The dgrad chain fc1 -> conv3 -> conv2 is the critical path; every wgrad only needs the dZ of its
// own layer, and every per-layer RMSProp update only needs that layer's wgrad plus the guarantee
// that the dgrad reading the old weights has finished.  On a single GPU those independent pieces
// run on three side streams (graph branches under capture):
//   main : head . fc1_dgrad . conv3_dgrad . conv2_dgrad . conv1_wgrad . opt(conv1)
//   sA   :          fc1_wgrad ......... [after fc1_dgrad]   opt(fc1, fc2)
//   sB   :                    conv3_wgrad .. [after conv3_dgrad] opt(conv3)
//   sC   :                               conv2_wgrad .. [after conv2_dgrad] opt(conv2)
// In a communicator the update follows one all-reduce of the whole gradient, so the simple
// serial order is kept.
// Data-parallel schedule (communicator, tensor-core engine): the fc gradient (95 % of the bytes) is summed and
// all-reduced as soon as fc1_wgrad is done, hidden behind the dgrad chain; the three small conv gradients
// share one all-reduce at the tail: small NCCL all-reduces cost ~15-20 us each inside the graph, so fewer is
// better once the big one is hidden.  (Multi-GPU schedules have not been re-measured on H100.)  Both collectives run in this order on one dedicated stream (a NCCL
// communicator must not be used from two streams at once); updates read the reduced gradient from d_g.
// Peer-memory exchange (comm_p2p.cuh): no shared communicator, so every layer's gradient is reduced
// the moment its wgrad has finished, on that layer's own branch, and only conv1's 32 KB exchange is left
// on the critical chain:  wgrad -> partial sums -> exchange (in place, all ranks) -> RMSProp from d_g.
static void destroy_step_graphs(b200dqn_net* n) {
  n->graph_step.drop();
  n->graph_train.drop();
}

static int backward_and_update_xchg(b200dqn_net* n, const FrameSource& fs, int rows, cudaStream_t st) {
  cudaStream_t sA = n->side[0], sB = n->side[1], sC = n->side[2];
  cudaEvent_t* ev = n->ev;
  B2_CHECK_CUDA(cudaEventRecord(ev[0], st));                 // head done: dZ4, dW5 partials
  B2_CHECK_CUDA(cudaStreamWaitEvent(sA, ev[0], 0));
  {
    NoPdlScope side;
    B2_TRY(bwd_op(n, fs, rows, kFc1Wgrad, sA));
    B2_TRY(cost_finish_on(n, rows, sA));
    B2_TRY(optimizer_range(n, 3, 4, 1 | 2, rows, sA, "reduce_fc"));
    B2_TRY(comm_xchg_range(n, 3, 4, 3, sA, "xchg_fc"));
  }
  B2_TRY(bwd_op(n, fs, rows, kFc1Dgrad, st));
  B2_CHECK_CUDA(cudaEventRecord(ev[1], st));                 // W4 no longer needed
  {
    NoPdlScope side;
    B2_CHECK_CUDA(cudaStreamWaitEvent(sA, ev[1], 0));
    B2_TRY(umma_opt_fc1(n, rows, sA, true));
    B2_TRY(optimizer_range(n, 4, 4, 4, rows, sA, "opt_fc2"));
    B2_CHECK_CUDA(cudaStreamWaitEvent(sB, ev[1], 0));
    B2_TRY(bwd_op(n, fs, rows, kConv3Wgrad, sB));
    B2_TRY(optimizer_range(n, 2, 2, 1 | 2, rows, sB, "reduce_conv3"));
    B2_TRY(comm_xchg_range(n, 2, 2, 2, sB, "xchg_conv3"));
  }
  B2_TRY(bwd_op(n, fs, rows, kConv3Dgrad, st));
  B2_CHECK_CUDA(cudaEventRecord(ev[2], st));                 // W3 no longer needed
  {
    NoPdlScope side;
    B2_CHECK_CUDA(cudaStreamWaitEvent(sB, ev[2], 0));
    B2_TRY(umma_opt_conv(n, 2, rows, sB, "opt_conv3", true));
    B2_CHECK_CUDA(cudaStreamWaitEvent(sC, ev[2], 0));
    B2_TRY(bwd_op(n, fs, rows, kConv2Wgrad, sC));
    B2_TRY(optimizer_range(n, 1, 1, 1 | 2, rows, sC, "reduce_conv2"));
    B2_TRY(comm_xchg_range(n, 1, 1, 1, sC, "xchg_conv2"));
  }
  B2_TRY(bwd_op(n, fs, rows, kConv2Dgrad, st));
  B2_CHECK_CUDA(cudaEventRecord(ev[3], st));                 // W2 no longer needed
  {
    NoPdlScope side;
    B2_CHECK_CUDA(cudaStreamWaitEvent(sC, ev[3], 0));
    B2_TRY(umma_opt_conv(n, 1, rows, sC, "opt_conv2", true));
  }
  B2_TRY(bwd_op(n, fs, rows, kConv1Wgrad, st));
  {
    NoPdlScope tail;
    B2_TRY(optimizer_range(n, 0, 0, 1 | 2, rows, st, "reduce_conv1"));
    B2_TRY(comm_xchg_range(n, 0, 0, 0, st, "xchg_conv1"));
    B2_TRY(umma_opt_conv(n, 0, rows, st, "opt_conv1", true));
  }
  B2_CHECK_CUDA(cudaEventRecord(ev[4], sA));
  B2_CHECK_CUDA(cudaEventRecord(ev[5], sB));
  B2_CHECK_CUDA(cudaEventRecord(ev[6], sC));
  B2_CHECK_CUDA(cudaStreamWaitEvent(st, ev[4], 0));
  B2_CHECK_CUDA(cudaStreamWaitEvent(st, ev[5], 0));
  B2_CHECK_CUDA(cudaStreamWaitEvent(st, ev[6], 0));
  return B200DQN_OK;
}

// Default data-parallel schedule (comm_p2p.cuh): the step keeps the single-GPU shape.  fc1's gradient is never
// exchanged — every rank gathers all learners' H3 / dZ4 rows (pushed by their producers' successors) and runs
// fc1_wgrad over the global minibatch; the four small layers go through the one-shot LL all-reduce the moment
// their wgrad is done.  Bytes received per step and rank: (W-1) x (0.47 MB planes + 0.64 MB LL lines).
static int backward_and_update_gather(b200dqn_net* n, const FrameSource& fs, int rows, cudaStream_t st) {
  cudaStream_t sA = n->side[0], sB = n->side[1], sC = n->side[2], sN = n->side[3];
  cudaEvent_t* ev = n->ev;
  // experimental: one launch per conv layer for reduce + LL exchange + RMSProp (umma_opt_conv_xll), off by default
  // one launch per conv layer for reduce + LL exchange + update (umma_opt_conv_xll): default since it was validated on
  // hardware at W = 2 (tests/test_gpu_multi.py; ~4.5 us per step); B200DQN_FUSED_XLL=0 restores the three launches
  // At W = 2 the fused kernel shortens the step; at W = 8 its polling CTAs spin while the peers catch up and delay the
  // chain's own kernels, so beyond two ranks the default is the three-launch form with its small polling grid.
  // (Chosen on an earlier GPU generation; multi-GPU schedules have not been re-measured on H100.)
  static const int fused_env = getenv("B200DQN_FUSED_XLL") ? atoi(getenv("B200DQN_FUSED_XLL")) : -1;
  const bool fused_xll = fused_env >= 0 ? fused_env != 0 : n->world <= 2;
  B2_CHECK_CUDA(cudaEventRecord(ev[0], st));                 // head done: dZ4 planes, dW5 partials
  B2_CHECK_CUDA(cudaStreamWaitEvent(sA, ev[0], 0));
  {
    NoPdlScope side;
    const bool head_pushed = comm_head_push(n, st, nullptr);  // (opt-in) the head kernel already sent this rank's dZ4 rows
    const bool dz_ll = !head_pushed && comm_dz4_ll_enabled();
    B2_CHECK_CUDA(cudaStreamWaitEvent(sA, ev[14], 0));       // own H3 push (forward, umma_push_h3) has been issued
    if (dz_ll) {
      // all ranks' dZ4 rows in the LL protocol (no flag word, no system fence); the same kernel polls the H3 flags
      B2_TRY(umma_gather_dz4_ll(n, sA));
    } else {
      if (!head_pushed) B2_TRY(umma_push_dz4(n, sA));        // peers' fc1_wgrad wait for these 64 KB
      B2_TRY(comm_wait_pushes(n, sA, head_pushed ? rows : 0));
    }
    B2_TRY(umma_fc1_wgrad_gathered(n, sA));
    // fc2 (8 KB) on the stream the H3 push has left idle: nothing later in the step reads W5
    B2_CHECK_CUDA(cudaStreamWaitEvent(sN, ev[0], 0));
    B2_TRY(cost_finish_on(n, rows, sN));
    B2_TRY(optimizer_range(n, 4, 4, 1 | 2, rows, sN, "reduce_fc2"));
    B2_TRY(comm_xll_layer(n, 4, sN, "xll_fc2"));
    B2_TRY(optimizer_range(n, 4, 4, 4, rows, sN, "opt_fc2"));
    B2_CHECK_CUDA(cudaEventRecord(ev[7], sN));
  }
  B2_TRY(bwd_op(n, fs, rows, kFc1Dgrad, st));
  B2_CHECK_CUDA(cudaEventRecord(ev[1], st));                 // W4 no longer needed
  {
    NoPdlScope side;
    B2_CHECK_CUDA(cudaStreamWaitEvent(sA, ev[1], 0));
    B2_TRY(umma_opt_fc1(n, rows, sA));                       // dW4 is already the global sum
    B2_CHECK_CUDA(cudaStreamWaitEvent(sB, ev[1], 0));
    B2_TRY(bwd_op(n, fs, rows, kConv3Wgrad, sB));
    if (!fused_xll) {
      B2_TRY(optimizer_range(n, 2, 2, 1 | 2, rows, sB, "reduce_conv3"));
      B2_TRY(comm_xll_layer(n, 2, sB, "xll_conv3"));
    }
  }
  B2_TRY(bwd_op(n, fs, rows, kConv3Dgrad, st));
  B2_CHECK_CUDA(cudaEventRecord(ev[2], st));                 // W3 no longer needed
  {
    NoPdlScope side;
    B2_CHECK_CUDA(cudaStreamWaitEvent(sB, ev[2], 0));
    if (fused_xll) B2_TRY(umma_opt_conv_xll(n, 2, rows, sB, "optx_conv3"));
    else B2_TRY(umma_opt_conv(n, 2, rows, sB, "opt_conv3", true));
    B2_CHECK_CUDA(cudaStreamWaitEvent(sC, ev[2], 0));
    B2_TRY(bwd_op(n, fs, rows, kConv2Wgrad, sC));
    if (!fused_xll) {
      B2_TRY(optimizer_range(n, 1, 1, 1 | 2, rows, sC, "reduce_conv2"));
      B2_TRY(comm_xll_layer(n, 1, sC, "xll_conv2"));
    }
  }
  B2_TRY(bwd_op(n, fs, rows, kConv2Dgrad, st));
  B2_CHECK_CUDA(cudaEventRecord(ev[3], st));                 // W2 no longer needed
  {
    NoPdlScope side;
    B2_CHECK_CUDA(cudaStreamWaitEvent(sC, ev[3], 0));
    if (fused_xll) B2_TRY(umma_opt_conv_xll(n, 1, rows, sC, "optx_conv2"));
    else B2_TRY(umma_opt_conv(n, 1, rows, sC, "opt_conv2", true));
  }
  B2_TRY(bwd_op(n, fs, rows, kConv1Wgrad, st));
  {
    NoPdlScope tail;
    if (fused_xll) {
      B2_TRY(umma_opt_conv_xll(n, 0, rows, st, "optx_conv1"));
    } else {
      B2_TRY(optimizer_range(n, 0, 0, 1 | 2, rows, st, "reduce_conv1"));
      B2_TRY(comm_xll_layer(n, 0, st, "xll_conv1"));
      B2_TRY(umma_opt_conv(n, 0, rows, st, "opt_conv1", true));
    }
  }
  B2_CHECK_CUDA(cudaEventRecord(ev[4], sA));
  B2_CHECK_CUDA(cudaEventRecord(ev[5], sB));
  B2_CHECK_CUDA(cudaEventRecord(ev[6], sC));
  B2_CHECK_CUDA(cudaStreamWaitEvent(st, ev[4], 0));
  B2_CHECK_CUDA(cudaStreamWaitEvent(st, ev[5], 0));
  B2_CHECK_CUDA(cudaStreamWaitEvent(st, ev[6], 0));
  B2_CHECK_CUDA(cudaStreamWaitEvent(st, ev[7], 0));
  return B200DQN_OK;
}

static int backward_and_update_multi(b200dqn_net* n, const FrameSource& fs, int rows, cudaStream_t st) {
  if (comm_gather_active(n, st)) return backward_and_update_gather(n, fs, rows, st);
  if (n->xchg_ok && n->xchg_sched == 1) return backward_and_update_xchg(n, fs, rows, st);
  cudaStream_t sA = n->side[0], sB = n->side[1], sC = n->side[2], sN = n->side[3];
  cudaEvent_t* ev = n->ev;
  B2_CHECK_CUDA(cudaEventRecord(ev[0], st));                 // head done: dZ4, dW5 partials
  B2_CHECK_CUDA(cudaStreamWaitEvent(sA, ev[0], 0));
  {
    NoPdlScope side;
    B2_TRY(bwd_op(n, fs, rows, kFc1Wgrad, sA));
    B2_TRY(cost_finish_on(n, rows, sA));
    B2_TRY(optimizer_range(n, 3, 4, 1 | 2, rows, sA, "reduce_fc"));        // partials -> d_g[fc1, fc2]
    B2_CHECK_CUDA(cudaEventRecord(ev[7], sA));
    B2_CHECK_CUDA(cudaStreamWaitEvent(sN, ev[7], 0));
    B2_TRY(comm_allreduce_range(n, 3, 4, sN));
    B2_CHECK_CUDA(cudaEventRecord(ev[8], sN));
  }
  B2_TRY(bwd_op(n, fs, rows, kFc1Dgrad, st));
  B2_CHECK_CUDA(cudaEventRecord(ev[1], st));                 // W4 no longer needed
  {
    NoPdlScope side;
    B2_CHECK_CUDA(cudaStreamWaitEvent(sA, ev[8], 0));
    B2_CHECK_CUDA(cudaStreamWaitEvent(sA, ev[1], 0));
    B2_TRY(umma_opt_fc1(n, rows, sA, true));
    B2_TRY(optimizer_range(n, 4, 4, 4, rows, sA, "opt_fc2"));
    B2_CHECK_CUDA(cudaStreamWaitEvent(sB, ev[1], 0));
    B2_TRY(bwd_op(n, fs, rows, kConv3Wgrad, sB));
  }
  B2_TRY(bwd_op(n, fs, rows, kConv3Dgrad, st));
  B2_CHECK_CUDA(cudaEventRecord(ev[2], st));
  {
    NoPdlScope side;
    B2_TRY(optimizer_range(n, 2, 2, 1 | 2, rows, sB, "reduce_conv3"));     // partials -> d_g, early, off the chain
    B2_CHECK_CUDA(cudaStreamWaitEvent(sC, ev[2], 0));
    B2_TRY(bwd_op(n, fs, rows, kConv2Wgrad, sC));
    B2_TRY(optimizer_range(n, 1, 1, 1 | 2, rows, sC, "reduce_conv2"));
  }
  B2_TRY(bwd_op(n, fs, rows, kConv2Dgrad, st));
  B2_TRY(bwd_op(n, fs, rows, kConv1Wgrad, st));
  {
    NoPdlScope tail;   // kernels around the collective use ordinary dependencies
    B2_TRY(optimizer_range(n, 0, 0, 1 | 2, rows, st, "reduce_conv1"));
    B2_CHECK_CUDA(cudaEventRecord(ev[5], sB));
    B2_CHECK_CUDA(cudaEventRecord(ev[6], sC));
    B2_CHECK_CUDA(cudaEventRecord(ev[9], st));
    B2_CHECK_CUDA(cudaStreamWaitEvent(sN, ev[5], 0));
    B2_CHECK_CUDA(cudaStreamWaitEvent(sN, ev[6], 0));
    B2_CHECK_CUDA(cudaStreamWaitEvent(sN, ev[9], 0));
    B2_TRY(comm_allreduce_range(n, 0, 2, sN));                              // one small collective for conv1..3
    B2_CHECK_CUDA(cudaEventRecord(ev[10], sN));
    B2_CHECK_CUDA(cudaStreamWaitEvent(st, ev[10], 0));
    B2_CHECK_CUDA(cudaStreamWaitEvent(sB, ev[10], 0));
    B2_CHECK_CUDA(cudaStreamWaitEvent(sC, ev[10], 0));
    B2_TRY(umma_opt_conv(n, 2, rows, sB, "opt_conv3", true));               // the three tiny updates run side by side
    B2_TRY(umma_opt_conv(n, 1, rows, sC, "opt_conv2", true));
    B2_TRY(umma_opt_conv(n, 0, rows, st, "opt_conv1", true));
    B2_CHECK_CUDA(cudaEventRecord(ev[11], sB));
    B2_CHECK_CUDA(cudaEventRecord(ev[12], sC));
    B2_CHECK_CUDA(cudaStreamWaitEvent(st, ev[11], 0));
    B2_CHECK_CUDA(cudaStreamWaitEvent(st, ev[12], 0));
  }
  B2_CHECK_CUDA(cudaEventRecord(ev[4], sA));
  B2_CHECK_CUDA(cudaStreamWaitEvent(st, ev[4], 0));
  return B200DQN_OK;
}

// The branch streams of the single-GPU step: fc1 (sA), conv3 (sB), conv2 (sC) and the fourth branch (sN)
struct StepBranches {
  cudaStream_t sA, sB, sC, sN;
};

// the single-GPU step's end: every branch joins the main stream
static int join_branches(b200dqn_net* n, cudaStream_t st, const StepBranches& br) {
  const cudaStream_t s[4] = {br.sA, br.sB, br.sC, br.sN};
  for (int i = 0; i < 4; ++i) B2_CHECK_CUDA(cudaEventRecord(n->ev[4 + i], s[i]));
  for (int i = 0; i < 4; ++i) B2_CHECK_CUDA(cudaStreamWaitEvent(st, n->ev[4 + i], 0));
  return B200DQN_OK;
}

// conv layer l's update on the single-GPU branch schedule, on whichever engine math_mode selects, then its soft target
// blend
static int update_conv(b200dqn_net* n, int l, int rows, cudaStream_t s) {
  static const char* const lbl[3] = {"opt_conv1", "opt_conv2", "opt_conv3"};
  if (n->cfg.math_mode == B200DQN_MATH_TCGEN05) B2_TRY(umma_opt_conv(n, l, rows, s, lbl[l]));
  else B2_TRY(optimizer_range(n, l, l, 1 | 4, rows, s, lbl[l]));
  if (n->soft) B2_TRY(soft_update_layers(n, l, l, n->soft_c, n->soft_t, s));
  return B200DQN_OK;
}

// The rest of the branches schedule under gradient-norm clipping, from fc1's dgrad on (ev[1] recorded, sA waiting on
// it): each branch ends with its layer's reduce and sum of squares instead of its update; main joins every branch,
// forms c32 and fans the clipped updates (with their image refreshes and soft target blends) back out over the same
// branches; the caller's end-of-step join follows.
//   main : ... conv2_dgrad . conv1_wgrad . end(conv1) . [join] clip_scale . opt(conv1)
//   sA   : fc1_wgrad ... [after fc1_dgrad] end(fc1)            [fan-out] opt(fc1)
//   sB   : conv3_wgrad .. [after conv3_dgrad] end(conv3)       [fan-out] opt(conv3)
//   sC   : conv2_wgrad .. [after conv2_dgrad] end(conv2)       [fan-out] opt(conv2)
//   sN   : cost . end(fc2) . end(embedding)                    [fan-out] opt(fc2) . opt(embedding)
static int clip_branches(b200dqn_net* n, const FrameSource& fs, int rows, cudaStream_t st, const StepBranches& br) {
  const auto [sA, sB, sC, sN] = br;
  cudaEvent_t* ev = n->ev;
  const bool tc = n->cfg.math_mode == B200DQN_MATH_TCGEN05;
  const bool fc2_on_sn = tc || n->fc2_block();   // else the SIMT engine's scalar fc2 rides with fc1 on sA
  {
    NoPdlScope side;
    B2_TRY(clip_layer_end(n, 3, rows, sA));
    if (!fc2_on_sn) B2_TRY(clip_layer_end(n, 4, rows, sA));
  }
  B2_CHECK_CUDA(cudaStreamWaitEvent(sB, ev[1], 0));
  { NoPdlScope side; B2_TRY(bwd_op(n, fs, rows, kConv3Wgrad, sB)); }
  B2_TRY(bwd_op(n, fs, rows, kConv3Dgrad, st, true));
  B2_CHECK_CUDA(cudaEventRecord(ev[2], st));                 // dZ2 ready, W3 no longer needed
  B2_CHECK_CUDA(cudaStreamWaitEvent(sB, ev[2], 0));
  { NoPdlScope side; B2_TRY(clip_layer_end(n, 2, rows, sB)); }
  B2_CHECK_CUDA(cudaStreamWaitEvent(sC, ev[2], 0));
  { NoPdlScope side; B2_TRY(bwd_op(n, fs, rows, kConv2Wgrad, sC)); }
  B2_TRY(bwd_op(n, fs, rows, kConv2Dgrad, st, true));
  B2_CHECK_CUDA(cudaEventRecord(ev[3], st));                 // dZ1 ready, W2 no longer needed
  B2_CHECK_CUDA(cudaStreamWaitEvent(sC, ev[3], 0));
  { NoPdlScope side; B2_TRY(clip_layer_end(n, 1, rows, sC)); }
  B2_TRY(bwd_op(n, fs, rows, kConv1Wgrad, st, true));
  NoPdlScope tail;   // the join and the fan-out use ordinary dependencies
  B2_TRY(clip_layer_end(n, 0, rows, st));
  B2_TRY(join_branches(n, st, br));   // every S_l partial is written
  B2_TRY(clip_scale(n, st));
  B2_CHECK_CUDA(cudaEventRecord(ev[9], st));                 // c32 ready
  for (cudaStream_t s : {sA, sB, sC, sN}) B2_CHECK_CUDA(cudaStreamWaitEvent(s, ev[9], 0));
  B2_TRY(clip_apply(n, 3, rows, sA));
  if (!fc2_on_sn) B2_TRY(clip_apply(n, 4, rows, sA));
  if (n->soft) B2_TRY(soft_update_layers(n, 3, fc2_on_sn ? 3 : 4, n->soft_c, n->soft_t, sA));
  B2_TRY(clip_apply(n, 2, rows, sB));
  if (n->soft) B2_TRY(soft_update_layers(n, 2, 2, n->soft_c, n->soft_t, sB));
  B2_TRY(clip_apply(n, 1, rows, sC));
  if (n->soft) B2_TRY(soft_update_layers(n, 1, 1, n->soft_c, n->soft_t, sC));
  if (fc2_on_sn) {
    B2_TRY(clip_apply(n, 4, rows, sN));
    if (n->soft) B2_TRY(soft_update_layers(n, 4, 4, n->soft_c, n->soft_t, sN));
  }
  if (n->iqn_n) {
    B2_TRY(clip_apply(n, kLayers, rows, sN));
    if (n->soft) B2_TRY(soft_update_extra(n, n->soft_c, n->soft_t, sN));
  }
  B2_TRY(clip_apply(n, 0, rows, st));
  if (n->soft) B2_TRY(soft_update_layers(n, 0, 0, n->soft_c, n->soft_t, st));
  return join_branches(n, st, br);
}

static int backward_and_update(b200dqn_net* n, const FrameSource& fs, int rows, cudaStream_t st, bool update) {
  if (update && n->world > 1 && !g_prof_on && n->use_branches && st != nullptr &&
      n->cfg.math_mode == B200DQN_MATH_TCGEN05)
    return backward_and_update_multi(n, fs, rows, st);
  // Under the event profiler the same kernels run, but every "branch" is the main stream (serialised).
  const bool branches = update && n->world == 1 && n->use_branches && (st != nullptr || g_prof_on);
  if (!branches) {
    for (int op = kFc1Wgrad; op <= kConv1Wgrad; ++op) {
      B2_TRY(bwd_op(n, fs, rows, BwdOp(op), st));
      if (op == kFc1Dgrad && n->iqn_n) B2_TRY(iqn_backward(n, rows, st, nullptr, update));
    }
    B2_TRY(cost_finish_on(n, rows, st));
    if (!update) return B200DQN_OK;
    if (n->world > 1) {
      B2_TRY(optimizer_range(n, 0, kLayers - 1, 1 | 2, rows, st, "grad_reduce"));
      B2_TRY(comm_allreduce_grads(n, st));
      B2_PROF("allreduce", st);
      B2_TRY(optimizer_range(n, 0, kLayers - 1, 4, rows, st, "optimizer"));
    } else {
      if (n->clip) B2_TRY(clip_step_serial(n, rows, st));
      else B2_TRY(update_range(n, 0, kLayers - 1, rows, st, "optimizer"));
      if (n->soft) {   // every layer is updated by now (the embedding and fraction layer in iqn_backward above)
        B2_TRY(soft_update_layers(n, 0, kLayers - 1, n->soft_c, n->soft_t, st));
        B2_TRY(soft_update_extra(n, n->soft_c, n->soft_t, st));
      }
    }
    return B200DQN_OK;
  }
  const StepBranches br{g_prof_on ? st : n->side[0], g_prof_on ? st : n->side[1], g_prof_on ? st : n->side[2],
                        g_prof_on ? st : n->side[3]};
  const auto [sA, sB, sC, sN] = br;
  cudaEvent_t* ev = n->ev;
  const bool tc = n->cfg.math_mode == B200DQN_MATH_TCGEN05;
  B2_CHECK_CUDA(cudaEventRecord(ev[0], st));                 // dZ4, the dW5 partials and the per-sample costs are ready
  B2_CHECK_CUDA(cudaStreamWaitEvent(sA, ev[0], 0));
  B2_CHECK_CUDA(cudaStreamWaitEvent(sN, ev[0], 0));
  {
    NoPdlScope side;
    B2_TRY(bwd_op(n, fs, rows, kFc1Wgrad, sA));             // overlaps fc1_dgrad (few CTAs)
    // fourth branch: the scalar cost and the 512 x A layer — nothing later in the step reads W5, and nothing here
    // sits in front of the fc1 optimizer any more (the SIMT engine's scalar fc2 rides with fc1 in opt_fc)
    B2_TRY(cost_finish_on(n, rows, sN));
    if (n->clip) {
      if (tc || n->fc2_block()) B2_TRY(clip_layer_end(n, 4, rows, sN));
    } else if (tc || n->fc2_block()) {
      B2_TRY(opt_fc2_small(n, rows, sN));
      if (n->soft) B2_TRY(soft_update_layers(n, 4, 4, n->soft_c, n->soft_t, sN));
    }
  }
  B2_TRY(bwd_op(n, fs, rows, kFc1Dgrad, st, true));
  if (n->iqn_n) {
    B2_TRY(iqn_backward(n, rows, st, sN, true));   // dZ3 is dpsi
    NoPdlScope side;
    if (n->clip) B2_TRY(clip_layer_end(n, kLayers, rows, sN));   // dWe, written by k_iqn_we on sN
    else if (n->soft)                                   // behind the embedding's and fraction layer's updates on sN
      B2_TRY(soft_update_extra(n, n->soft_c, n->soft_t, sN));
  }
  B2_CHECK_CUDA(cudaEventRecord(ev[1], st));                 // dZ3 ready, W4 no longer needed
  B2_CHECK_CUDA(cudaStreamWaitEvent(sA, ev[1], 0));
  if (n->clip) return clip_branches(n, fs, rows, st, br);
  {
    NoPdlScope side;
    if (tc && n->lt.splits[3] > 1) {                           // IQN: sum fc1's wgrad partials first
      B2_TRY(optimizer_range(n, 3, 3, 1 | 2, rows, sA, "reduce_fc1"));
      B2_TRY(umma_opt_fc1(n, rows, sA, true));
    } else if (tc) {
      B2_TRY(umma_opt_fc1(n, rows, sA));                       // smem-free: co-resides with the dgrad chain
    }
    else B2_TRY(optimizer_range(n, 3, n->fc2_block() ? 3 : 4, 1 | 4, rows, sA, "opt_fc"));
    // fc1's soft target update (with the SIMT engine's scalar fc2, which rides with it in opt_fc)
    if (n->soft) B2_TRY(soft_update_layers(n, 3, tc || n->fc2_block() ? 3 : 4, n->soft_c, n->soft_t, sA));
  }
  B2_CHECK_CUDA(cudaStreamWaitEvent(sB, ev[1], 0));
  { NoPdlScope side; B2_TRY(bwd_op(n, fs, rows, kConv3Wgrad, sB)); }
  B2_TRY(bwd_op(n, fs, rows, kConv3Dgrad, st, true));
  B2_CHECK_CUDA(cudaEventRecord(ev[2], st));                 // dZ2 ready, W3 no longer needed
  B2_CHECK_CUDA(cudaStreamWaitEvent(sB, ev[2], 0));
  { NoPdlScope side; B2_TRY(update_conv(n, 2, rows, sB)); }
  B2_CHECK_CUDA(cudaStreamWaitEvent(sC, ev[2], 0));
  { NoPdlScope side; B2_TRY(bwd_op(n, fs, rows, kConv2Wgrad, sC)); }
  B2_TRY(bwd_op(n, fs, rows, kConv2Dgrad, st, true));
  B2_CHECK_CUDA(cudaEventRecord(ev[3], st));                 // dZ1 ready, W2 no longer needed
  B2_CHECK_CUDA(cudaStreamWaitEvent(sC, ev[3], 0));
  { NoPdlScope side; B2_TRY(update_conv(n, 1, rows, sC)); }
  B2_TRY(bwd_op(n, fs, rows, kConv1Wgrad, st, true));
  B2_TRY(update_conv(n, 0, rows, st));
  return join_branches(n, st, br);
}

static int shift_draw(b200dqn_net* n, cudaStream_t s) {
  B2_CHECK_CUDA(launch_pdl(k_shift_draw, dim3(1), dim3(1024), 0, s, n->d_crop_ctr,
                           (unsigned long long)n->cfg.shift_seed, n->crop_pad, n->nb, n->d_crop,
                           ktrace_slot("shift_draw")));
  B2_PROF("shift_draw", s);
  return B200DQN_OK;
}

// The random-shift draw of a train step on its own branch from the head of the step (on a stream; the serial schedule
// draws in line, in shift_join).  It reads only the counter, so it overlaps the sampler.
static int shift_fork(b200dqn_net* n, cudaStream_t st) {
  if (!n->crop_pad || n->crop_forked || !branches_on(n, st)) return B200DQN_OK;
  cudaEvent_t done;
  B2_TRY(fork_branch(n, st, true, 1, 17, &done, [&](cudaStream_t sD) { return shift_draw(n, sD); }));
  n->crop_forked = true;
  return B200DQN_OK;
}

// The draw is complete on st from here on: its branch joins (the forward's first launch after it keeps its PDL), or it
// runs here, in line.
static int shift_join(b200dqn_net* n, cudaStream_t st) {
  if (!n->crop_forked) return shift_draw(n, st);
  n->crop_forked = false;
  return join_branch(st, n->ev[18]);
}

// One DeepQNetwork.train on device-resident inputs (the caller counts train_iterations, :168).
static int train_step(b200dqn_net* n, const FrameSource& fs_in, const uint8_t* actions, const int64_t* rewards,
                      const uint8_t* terminals, const int32_t* midx, cudaStream_t st) {
  const int rows = n->nb;
  FrameSource fs = fs_in;
  if (n->crop_pad) {   // random-shift augmentation: fresh crop offsets for the prestates (slot 0) and poststates
    B2_TRY(shift_fork(n, st));
    B2_TRY(shift_join(n, st));
    fs.crop[0] = n->d_crop;
    fs.crop[1] = n->d_crop + 2 * rows;
  }
  HeadTrainArgs td{1, actions, rewards, terminals, midx, n->cfg.discount_rate, n->cfg.min_reward, n->cfg.max_reward,
                   float(n->cfg.clip_error), n->d_delta, n->d_step, n->d_rowcost, n->d_dz4,
                   n->d_part + n->lt.part_off[4], nullptr, 0,
                   n->cfg.optimizer == B200DQN_OPT_ADAM ? n->d_optscal : nullptr, float(n->cfg.learning_rate), n->A,
                   reinterpret_cast<uint32_t*>(n->d_cost + kCostRing + 1), HeadPush{}};
  umma_dz4_planes(n, &td.dz4_hi, &td.dz4_lo_off);
  comm_head_push(n, st, &td.push);
  if (n->step_replay && n->step_replay->per_on) {   // a prioritized ring: weighted step, TD errors for the update
    td.isw = n->step_replay->d_isw + n->rank * n->nb;
    td.td_err = n->d_td_err;
  }
  td.nstep = n->step_replay ? n->step_replay->nstep : 1;   // host-staged minibatches are one-step
  // Double DQN adds the online network on the poststates as a third slot of the same launches.  With target_steps = 0
  // the target network IS the online network, so slot 1 already holds that forward and a* = argmax of the same row:
  // the vanilla step is the Double DQN step, bit for bit.
  const int nets = (n->double_q && n->d_tw != n->d_w) ? 3 : 2;
  cudaEvent_t join = nullptr;
  if (n->munchausen && n->d_tw != n->d_w) {
    // The Munchausen target needs the target network on the prestates.  The pass reads only weights and frames, so on
    // a stream it forks into its own branch here, after the sampler, overlaps the forward and joins before the head;
    // on the serial schedule it runs in line, ahead of the forward.
    B2_TRY(fork_branch(n, st, branches_on(n, st), 0, 15, &join,
                       [&](cudaStream_t sP) { return forward_target_pre(n, fs, rows, sP); }));
  }
  if (n->rem_k && !n->boot) {
    // The mixture draw reads only its counter, so on a stream it runs on its own branch from here and joins before the
    // head; on the serial schedule it runs in line, ahead of the forward.
    B2_TRY(fork_branch(n, st, branches_on(n, st), 0, 15, &join, [&](cudaStream_t sR) {
      B2_CHECK_CUDA(launch_pdl(k_rem_alpha, dim3(1), dim3(256), 0, sR, n->d_rem_ctr, (unsigned long long)n->cfg.rem_seed,
                               n->rem_k, n->d_rem_alpha, ktrace_slot("rem_alpha")));
      B2_PROF("rem_alpha", sR);
      return B200DQN_OK;
    }));
  }
  B2_TRY(forward(n, fs, nets, rows, st, td, join));
  return backward_and_update(n, fs, rows, st, true);
}

// ---------------------------------------------------------------- layout conversion (host)
// Neon layout <-> internal layout index map for one layer; returns internal linear index.
static inline int64_t neon_to_internal(int layer, int64_t i, int A, int hidden) {
  switch (layer) {
    case 0: return i;  // (c,r,s) x K: identical
    case 1: {          // neon rows (c,r,s), C=32,R=4 -> internal rows (r,s,c)
      const int64_t k = i % kC2, row = i / kC2;
      const int c = int(row / 16), r = int(row / 4) % 4, s = int(row % 4);
      return ((int64_t(r) * 4 + s) * kC1 + c) * kC2 + k;
    }
    case 2: {          // C=64, R=3
      const int64_t k = i % kC3, row = i / kC3;
      const int c = int(row / 9), r = int(row / 3) % 3, s = int(row % 3);
      return ((int64_t(r) * 3 + s) * kC2 + c) * kC3 + k;
    }
    case 3: {          // neon W[n][(c,p,q)] -> internal W[(p,q,c)][n], n < hidden
      const int64_t nn = i / kFlat, col = i % kFlat;
      const int c = int(col / 49), p = int(col / 7) % 7, q = int(col % 7);
      return ((int64_t(p) * 7 + q) * kC3 + c) * hidden + nn;
    }
    default: {         // neon W[a][k] -> internal W[k][a] (dueling: a = A is the value row)
      const int64_t a = i / kHidden, k = i % kHidden;
      return k * A + a;
    }
  }
}

}  // namespace b200

using namespace b200;

// ============================================================================ C ABI: network
extern "C" int b200dqn_net_config_default(b200dqn_net_config* cfg, int num_actions) {
  B2_REQUIRE(cfg, B200DQN_EINVAL, "null cfg");
  memset(cfg, 0, sizeof(*cfg));
  cfg->num_actions = num_actions;
  cfg->batch_size = 32;          // main.py:39
  cfg->history_length = 4;       // main.py:34
  cfg->screen_h = cfg->screen_w = 84;  // main.py:27-28
  cfg->discount_rate = 0.99;     // main.py:38
  cfg->learning_rate = 0.00025;  // main.py:37
  cfg->decay_rate = 0.95;        // main.py:41
  cfg->clip_error = 1.0;         // main.py:42
  cfg->min_reward = -1;          // main.py:43
  cfg->max_reward = 1;           // main.py:44
  cfg->target_steps = 10000;     // main.py:63
  cfg->math_mode = B200DQN_MATH_FP32_SIMT;
  cfg->optimizer = B200DQN_OPT_RMSPROP;   // main.py:40
  cfg->num_atoms = 0;            // scalar head; the distributional head's support defaults to [-10, 10]
  cfg->v_min = -10.0;
  cfg->v_max = 10.0;
  cfg->dueling = 0;              // one value stream
  cfg->num_quantiles = 0;        // no quantile-regression head
  cfg->munchausen = 0;           // the scalar head's target; the Munchausen constants are the paper's
  cfg->munchausen_alpha = 0.9;
  cfg->munchausen_tau = 0.03;
  cfg->munchausen_clip = -1.0;
  cfg->num_tau_samples = 0;      // no IQN head; Dopamine's K when it is on
  cfg->num_quantile_samples = 32;
  cfg->tau_seed = 0;
  cfg->random_shift = 0;         // no augmentation; DrQ's pad is 4
  cfg->shift_seed = 0;
  cfg->num_heads = 0;            // no random ensemble mixture head
  cfg->rem_seed = 0;
  cfg->num_fractions = 0;        // no FQF head
  cfg->fraction_lr = 2.5e-9;
  cfg->bootstrap_heads = 0;      // no bootstrapped heads; this project's mask probability when they are on
  cfg->bootstrap_p = 0.5;
  cfg->bootstrap_seed = 0;
  return B200DQN_OK;
}

static int double_q_alloc(b200dqn_net* n);

extern "C" int b200dqn_net_create(int device, const b200dqn_net_config* cfg, b200dqn_net** out) {
  B2_REQUIRE(cfg && out, B200DQN_EINVAL, "net_create: null argument");
  B2_REQUIRE(cfg->num_actions >= 1 && cfg->num_actions <= kMaxActions, B200DQN_EINVAL,
             "net_create: num_actions %d not in [1,%d]", cfg->num_actions, kMaxActions);
  B2_REQUIRE(cfg->batch_size >= 1 && cfg->batch_size <= 4096, B200DQN_EINVAL, "net_create: batch_size");
  B2_REQUIRE(cfg->history_length >= 1, B200DQN_EINVAL, "net_create: history_length %d < 1", cfg->history_length);
  B2_REQUIRE(cfg->screen_h == kFrameH && cfg->screen_w == kFrameW, B200DQN_ENOTIMPL,
             "net_create: only the reference's 84x84 Nature-DQN screen is implemented (got %dx%d)", cfg->screen_h,
             cfg->screen_w);
  B2_REQUIRE(cfg->history_length <= kMaxHist, B200DQN_ENOTIMPL,
             "net_create: history_length %d not implemented (history lengths 1..%d are)", cfg->history_length, kMaxHist);
  B2_REQUIRE(cfg->math_mode == B200DQN_MATH_FP32_SIMT || cfg->math_mode == B200DQN_MATH_TCGEN05, B200DQN_EINVAL,
             "net_create: unknown math_mode %d", cfg->math_mode);
  B2_REQUIRE(cfg->optimizer >= B200DQN_OPT_RMSPROP && cfg->optimizer <= B200DQN_OPT_ADADELTA, B200DQN_EINVAL,
             "net_create: unknown optimizer %d", cfg->optimizer);   // deepqnetwork.py:61 `assert false, "Unknown optimizer"`
  B2_REQUIRE(cfg->num_atoms == 0 || (cfg->num_atoms >= 2 && cfg->num_atoms <= kMaxAtoms), B200DQN_EINVAL,
             "net_create: num_atoms %d is neither 0 (scalar head) nor in [2,%d]", cfg->num_atoms, kMaxAtoms);
  B2_REQUIRE(cfg->num_atoms == 0 || (std::isfinite(cfg->v_min) && std::isfinite(cfg->v_max) && cfg->v_min < cfg->v_max),
             B200DQN_EINVAL, "net_create: the support needs finite v_min < v_max (got %g, %g)", cfg->v_min, cfg->v_max);
  B2_REQUIRE(cfg->dueling == 0 || cfg->dueling == 1, B200DQN_EINVAL, "net_create: dueling %d is neither 0 nor 1",
             cfg->dueling);
  B2_REQUIRE(!(cfg->dueling && cfg->num_atoms), B200DQN_ENOTIMPL,
             "net_create: a dueling net with a distributional head is not implemented");
  B2_REQUIRE(cfg->num_quantiles >= 0 && cfg->num_quantiles <= kMaxQuantiles, B200DQN_EINVAL,
             "net_create: num_quantiles %d is neither 0 (no quantile head) nor in [1,%d]", cfg->num_quantiles,
             kMaxQuantiles);
  B2_REQUIRE(!(cfg->num_quantiles && cfg->num_atoms), B200DQN_EINVAL,
             "net_create: num_quantiles and num_atoms both ask for a head; a net has one");
  B2_REQUIRE(!cfg->num_quantiles || std::isfinite(cfg->clip_error), B200DQN_EINVAL,
             "net_create: the quantile Huber threshold clip_error must be finite (got %g)", cfg->clip_error);
  B2_REQUIRE(!(cfg->dueling && cfg->num_quantiles), B200DQN_ENOTIMPL,
             "net_create: a dueling net with a quantile-regression head is not implemented");
  B2_REQUIRE(cfg->munchausen == 0 || cfg->munchausen == 1, B200DQN_EINVAL,
             "net_create: munchausen %d is neither 0 nor 1 (the Munchausen target)", cfg->munchausen);
  if (cfg->munchausen) {
    B2_REQUIRE(std::isfinite(cfg->munchausen_alpha) && cfg->munchausen_alpha >= 0, B200DQN_EINVAL,
               "net_create: the Munchausen alpha must be finite and >= 0 (got %g)", cfg->munchausen_alpha);
    B2_REQUIRE(std::isfinite(cfg->munchausen_tau) && cfg->munchausen_tau > 0, B200DQN_EINVAL,
               "net_create: the Munchausen tau must be finite and > 0 (got %g)", cfg->munchausen_tau);
    B2_REQUIRE(std::isfinite(cfg->munchausen_clip) && cfg->munchausen_clip <= 0, B200DQN_EINVAL,
               "net_create: the Munchausen clip l0 must be finite and <= 0 (got %g)", cfg->munchausen_clip);
    B2_REQUIRE(!cfg->dueling && !cfg->num_atoms && !cfg->num_quantiles, B200DQN_ENOTIMPL,
               "net_create: the Munchausen target with a dueling network, a distributional or a quantile head is not "
               "implemented");
  }
  B2_REQUIRE(cfg->num_tau_samples >= 0 && cfg->num_tau_samples <= kIqnMaxPer, B200DQN_EINVAL,
             "net_create: num_tau_samples %d is neither 0 (no IQN head) nor in [1,%d]", cfg->num_tau_samples, kIqnMaxPer);
  if (cfg->num_tau_samples) {
    B2_REQUIRE(cfg->num_quantile_samples >= 1 && cfg->num_quantile_samples <= kIqnMaxPer, B200DQN_EINVAL,
               "net_create: num_quantile_samples %d not in [1,%d]", cfg->num_quantile_samples, kIqnMaxPer);
    B2_REQUIRE(!cfg->num_atoms && !cfg->num_quantiles, B200DQN_EINVAL,
               "net_create: num_tau_samples with num_atoms or num_quantiles asks for two heads; a net has one");
    B2_REQUIRE(std::isfinite(cfg->clip_error), B200DQN_EINVAL,
               "net_create: the quantile Huber threshold clip_error must be finite (got %g)", cfg->clip_error);
    const int64_t xr = int64_t(cfg->batch_size) * std::max(cfg->num_tau_samples, cfg->num_quantile_samples);
    B2_REQUIRE(xr <= 4096, B200DQN_EINVAL,
               "net_create: the IQN head runs fc1 on batch_size x max(num_tau_samples, num_quantile_samples) = %lld rows; "
               "at most 4096 are supported", (long long)xr);
    B2_REQUIRE(!cfg->dueling && !cfg->munchausen, B200DQN_ENOTIMPL,
               "net_create: the IQN head with a dueling network or the Munchausen target is not implemented");
  }
  B2_REQUIRE(cfg->random_shift >= 0 && cfg->random_shift <= kMaxCropPad, B200DQN_EINVAL,
             "net_create: random_shift %d is neither 0 (no augmentation) nor in [1,%d]", cfg->random_shift, kMaxCropPad);
  B2_REQUIRE(cfg->num_heads >= 0 && cfg->num_heads <= kMaxRemHeads, B200DQN_EINVAL,
             "net_create: num_heads %d is neither 0 (no REM head) nor in [1,%d]", cfg->num_heads, kMaxRemHeads);
  if (cfg->num_heads) {
    B2_REQUIRE(!cfg->num_atoms && !cfg->num_quantiles && !cfg->num_tau_samples, B200DQN_EINVAL,
               "net_create: num_heads (REM) with num_atoms, num_quantiles or num_tau_samples asks for two heads; a net "
               "has one");
    B2_REQUIRE(!cfg->dueling && !cfg->munchausen, B200DQN_ENOTIMPL,
               "net_create: the REM head with a dueling network or the Munchausen target is not implemented");
  }
  B2_REQUIRE(cfg->num_fractions == 0 || (cfg->num_fractions >= 2 && cfg->num_fractions <= kFqfMaxN), B200DQN_EINVAL,
             "net_create: num_fractions %d is neither 0 (no FQF head) nor in [2,%d]", cfg->num_fractions, kFqfMaxN);
  if (cfg->num_fractions) {
    B2_REQUIRE(std::isfinite(cfg->fraction_lr) && cfg->fraction_lr >= 0, B200DQN_EINVAL,
               "net_create: fraction_lr must be finite and >= 0 (got %g)", cfg->fraction_lr);
    B2_REQUIRE(int64_t(cfg->batch_size) * cfg->num_fractions <= 4096, B200DQN_EINVAL,
               "net_create: the FQF head runs fc1 on batch_size x num_fractions = %lld rows; at most 4096 are supported",
               (long long)cfg->batch_size * cfg->num_fractions);
    B2_REQUIRE(!cfg->num_atoms && !cfg->num_quantiles && !cfg->num_tau_samples && !cfg->num_heads, B200DQN_EINVAL,
               "net_create: num_fractions with num_atoms, num_quantiles, num_tau_samples or num_heads asks for two "
               "heads; a net has one");
    B2_REQUIRE(std::isfinite(cfg->clip_error), B200DQN_EINVAL,
               "net_create: the quantile Huber threshold clip_error must be finite (got %g)", cfg->clip_error);
    B2_REQUIRE(!cfg->dueling && !cfg->munchausen, B200DQN_ENOTIMPL,
               "net_create: the FQF head with a dueling network or the Munchausen target is not implemented");
  }
  B2_REQUIRE(cfg->bootstrap_heads >= 0 && cfg->bootstrap_heads <= kMaxRemHeads, B200DQN_EINVAL,
             "net_create: bootstrap_heads %d is neither 0 (no bootstrapped heads) nor in [1,%d]", cfg->bootstrap_heads,
             kMaxRemHeads);
  if (cfg->bootstrap_heads) {
    B2_REQUIRE(std::isfinite(cfg->bootstrap_p) && cfg->bootstrap_p > 0 && cfg->bootstrap_p <= 1, B200DQN_EINVAL,
               "net_create: the bootstrap mask probability bootstrap_p must be in (0, 1] (got %g)", cfg->bootstrap_p);
    B2_REQUIRE(!cfg->num_atoms && !cfg->num_quantiles && !cfg->num_tau_samples && !cfg->num_heads &&
               !cfg->num_fractions, B200DQN_EINVAL,
               "net_create: bootstrap_heads with num_atoms, num_quantiles, num_tau_samples, num_heads or num_fractions "
               "asks for two heads; a net has one");
    B2_REQUIRE(!cfg->dueling && !cfg->munchausen, B200DQN_ENOTIMPL,
               "net_create: bootstrapped heads with a dueling network or the Munchausen target are not implemented");
  }
  B2_REQUIRE(std::isfinite(cfg->soft_target_tau) && cfg->soft_target_tau >= 0 && cfg->soft_target_tau <= 1,
             B200DQN_EINVAL, "net_create: the soft target update's soft_target_tau must be finite and in [0, 1] (got %g)",
             cfg->soft_target_tau);
  B2_REQUIRE(cfg->soft_target_tau == 0 || cfg->target_steps != 0, B200DQN_EINVAL,
             "net_create: a soft target update (soft_target_tau %g) needs a separate target network; target_steps = 0 "
             "makes the target the online network", cfg->soft_target_tau);
  B2_REQUIRE(std::isfinite(cfg->max_grad_norm) && cfg->max_grad_norm >= 0, B200DQN_EINVAL,
             "net_create: gradient-norm clipping's max_grad_norm must be finite and >= 0 (got %g)", cfg->max_grad_norm);
  DeviceGuard g(device);
  auto* n = new (std::nothrow) b200dqn_net();
  B2_REQUIRE(n, B200DQN_EINVAL, "out of host memory");
  n->n_states = cfg->optimizer == B200DQN_OPT_ADAM ? 2 : cfg->optimizer == B200DQN_OPT_ADADELTA ? 3 : 1;
  n->device = device;
  B2_CHECK_CUDA(cudaDeviceGetAttribute(&n->sm_count, cudaDevAttrMultiProcessorCount, device));
  n->cfg = *cfg;
  n->nb = cfg->batch_size;
  n->A = cfg->num_actions;
  n->atoms = cfg->num_atoms;
  n->quantiles = cfg->num_quantiles;
  n->rem_k = cfg->num_heads;
  if (cfg->bootstrap_heads) {   // the REM head's K-headed fc2 and buffers, trained per head
    n->rem_k = cfg->bootstrap_heads;
    n->boot = true;
  }
  n->dueling = cfg->dueling != 0;
  n->munchausen = cfg->munchausen != 0;
  if (cfg->soft_target_tau > 0) {
    n->soft = true;
    n->soft_c = float(1.0 - cfg->soft_target_tau);
    n->soft_t = float(cfg->soft_target_tau);
  }
  n->hidden = n->dueling ? kDuelHidden : kHidden;
  if (cfg->num_tau_samples) {
    n->iqn_n = cfg->num_tau_samples;
    n->iqn_k = cfg->num_quantile_samples;
    n->iqn_rows = cfg->batch_size * std::max(n->iqn_n, n->iqn_k);
  }
  if (cfg->num_fractions) {   // the IQN head's machinery at N = K = num_fractions rows per sample
    n->fqf_n = n->iqn_n = n->iqn_k = cfg->num_fractions;
    n->iqn_rows = cfg->batch_size * n->fqf_n;
  }
  if (n->atoms) n->dz = (cfg->v_max - cfg->v_min) / double(n->atoms - 1);
  const int nb = n->nb, A = n->A, hist = cfg->history_length;
  const int xr = n->iqn_n ? n->iqn_rows : nb;   // rows of fc1's and fc2's buffers (IQN: the expanded rows)
  LayerTable& lt = n->lt;
  const int rows_[kLayers] = {64 * hist, kK2, kK3, kFlat, kHidden};   // conv1: one 64-tap k-block per frame
  const int cols_[kLayers] = {kC1, kC2, kC3, n->hidden, n->fc2_cols()};
  lt.off[0] = 0;
  for (int l = 0; l < kLayers; ++l) {
    lt.rows[l] = rows_[l];
    lt.cols[l] = cols_[l];
    lt.off[l + 1] = lt.off[l] + int64_t(rows_[l]) * cols_[l];
  }
  n->n_params = lt.off[kLayers];
  B2_REQUIRE(n->n_params % 4 == 0, B200DQN_EINVAL, "parameter count must be a multiple of 4");
  const int kred[3] = {nb * kP1 * kP1, nb * kP2 * kP2, nb * kP3 * kP3};
  const int base[3] = {512, 96, 112};
  int64_t po = 0;
  for (int l = 0; l < kLayers; ++l) {
    if (l == 4)
      lt.splits[l] = nb;   // the head kernel leaves one dW5 partial per sample
    else if (cfg->math_mode == B200DQN_MATH_TCGEN05)
      lt.splits[l] = l < 3 ? umma_wgrad_splits(l, nb) : n->iqn_n ? int(cdiv(nb * n->iqn_n, kIqnWgradRows)) : 1;
    else
      lt.splits[l] = l < 3 ? int(cdiv(kred[l], wgrad_chunk(kred[l], base[l]))) : 1;
    lt.part_off[l] = po;
    if (l == 4 && n->fc2_block())   // distributional / quantile / IQN / REM head: the taken action's [512][block] per row
      po += int64_t(n->iqn_n ? n->iqn_rows : nb) * kHidden * n->fc2_block();
    else
      po += int64_t(lt.splits[l]) * (lt.off[l + 1] - lt.off[l]);
  }
  n->part_elems = po;

  auto fmalloc = [&](float** p, size_t elems) -> cudaError_t {
    cudaError_t e = cudaMalloc(p, elems * sizeof(float));
    if (e == cudaSuccess) e = cudaMemset(*p, 0, elems * sizeof(float));
    return e;
  };
  B2_CHECK_CUDA(fmalloc(&n->d_w, n->n_params));
  B2_CHECK_CUDA(fmalloc(&n->d_s, n->n_params * n->n_states));
  B2_CHECK_CUDA(fmalloc(&n->d_optscal, 4));
  if (cfg->target_steps) {
    B2_CHECK_CUDA(fmalloc(&n->d_tw, n->n_params));
    B2_CHECK_CUDA(fmalloc(&n->d_ts, n->n_params * n->n_states));
  } else {
    n->d_tw = n->d_w;  // deepqnetwork.py:72-73: the target model IS the online model
    n->d_ts = n->d_s;
  }
  // the gradient buffer is the one allocation peers map (comm.cu): their flag words sit behind it
  B2_CHECK_CUDA(fmalloc(&n->d_g, n->n_params + kXFlagWords));
  n->d_xflags = reinterpret_cast<uint32_t*>(n->d_g + n->n_params);
  constexpr int kXWords = kXChannels * kXMaxBlocks + 1 + 2 * kXChannels + 2 * kXPushChannels + 1;
  B2_CHECK_CUDA(cudaMalloc(&n->d_xepoch, kXWords * sizeof(uint32_t)));
  B2_CHECK_CUDA(cudaMemset(n->d_xepoch, 0, kXWords * sizeof(uint32_t)));
  n->d_xerr = n->d_xepoch + kXChannels * kXMaxBlocks;
  n->d_xll_epoch = n->d_xerr + 1;
  n->d_xpush_epoch = n->d_xll_epoch + 2 * kXChannels;
  B2_CHECK_CUDA(fmalloc(&n->d_part, n->part_elems));
  for (int z = 0; z < 2; ++z) {
    B2_CHECK_CUDA(fmalloc(&n->d_h1[z], size_t(nb) * kP1 * kP1 * kC1));
    B2_CHECK_CUDA(fmalloc(&n->d_h2[z], size_t(nb) * kP2 * kP2 * kC2));
    B2_CHECK_CUDA(fmalloc(&n->d_h3[z], size_t(nb) * kFlat));
    B2_CHECK_CUDA(fmalloc(&n->d_h4[z], size_t(xr) * n->hidden));
  }
  for (int z = 0; z < 3; ++z) B2_CHECK_CUDA(fmalloc(&n->d_q[z], size_t(nb) * A));
  B2_CHECK_CUDA(fmalloc(&n->d_fc1part, size_t(2) * kFc1Splits * xr * n->hidden));
  B2_CHECK_CUDA(fmalloc(&n->d_delta, size_t(nb) * A));
  B2_CHECK_CUDA(fmalloc(&n->d_dz4, size_t(xr) * n->hidden));
  B2_CHECK_CUDA(fmalloc(&n->d_dz3, size_t(nb) * kFlat));
  B2_CHECK_CUDA(fmalloc(&n->d_dz2, size_t(nb) * kP2 * kP2 * kC2));
  B2_CHECK_CUDA(fmalloc(&n->d_dz1, size_t(nb) * kP1 * kP1 * kC1));
  B2_CHECK_CUDA(fmalloc(&n->d_cost, kCostRing + 2));   // ring, "latest" slot, action-range flag word
  B2_CHECK_CUDA(cudaMalloc(&n->d_step, sizeof(uint32_t)));
  B2_CHECK_CUDA(cudaMemset(n->d_step, 0, sizeof(uint32_t)));
  B2_CHECK_CUDA(fmalloc(&n->d_rowcost, nb));
  if (n->atoms) {
    const size_t dist = size_t(nb) * A * n->atoms;
    B2_CHECK_CUDA(fmalloc(&n->d_logits, 3 * dist));
    B2_CHECK_CUDA(fmalloc(&n->d_probs, 3 * dist));
    B2_CHECK_CUDA(fmalloc(&n->d_tdist, size_t(nb) * n->atoms));
    B2_CHECK_CUDA(fmalloc(&n->d_lgrad, size_t(nb) * n->atoms));
    B2_CHECK_CUDA(cudaMalloc(&n->d_act_rows, nb * sizeof(int32_t)));
    B2_CHECK_CUDA(cudaMemset(n->d_act_rows, 0, nb * sizeof(int32_t)));
  }
  if (n->quantiles) {
    B2_CHECK_CUDA(fmalloc(&n->d_theta, size_t(3) * nb * A * n->quantiles));
    B2_CHECK_CUDA(fmalloc(&n->d_tquant, size_t(nb) * n->quantiles));
    B2_CHECK_CUDA(fmalloc(&n->d_qgrad, size_t(nb) * n->quantiles));
    B2_CHECK_CUDA(cudaMalloc(&n->d_act_rows, nb * sizeof(int32_t)));
    B2_CHECK_CUDA(cudaMemset(n->d_act_rows, 0, nb * sizeof(int32_t)));
  }
  if (n->rem_k) {
    B2_CHECK_CUDA(fmalloc(&n->d_theta, size_t(3) * nb * A * n->rem_k));
    B2_CHECK_CUDA(fmalloc(&n->d_rem_grad, size_t(nb) * n->rem_k));
    if (n->boot) {
      B2_CHECK_CUDA(cudaMalloc(&n->d_boot_mask, size_t(nb) * n->rem_k));
      B2_CHECK_CUDA(cudaMemset(n->d_boot_mask, 0, size_t(nb) * n->rem_k));
      B2_CHECK_CUDA(fmalloc(&n->d_boot_y, size_t(nb) * n->rem_k));
      B2_CHECK_CUDA(fmalloc(&n->d_boot_delta, size_t(nb) * n->rem_k));
      B2_CHECK_CUDA(cudaMalloc(&n->d_boot_head, sizeof(int32_t)));
      B2_CHECK_CUDA(cudaMemset(n->d_boot_head, 0xff, sizeof(int32_t)));   // -1: the mean over the heads
    } else {
      B2_CHECK_CUDA(fmalloc(&n->d_rem_alpha, n->rem_k));
      B2_CHECK_CUDA(cudaMalloc(&n->d_rem_ctr, sizeof(unsigned long long)));
      B2_CHECK_CUDA(cudaMemset(n->d_rem_ctr, 0, sizeof(unsigned long long)));
    }
    B2_CHECK_CUDA(cudaMalloc(&n->d_act_rows, nb * sizeof(int32_t)));
    B2_CHECK_CUDA(cudaMemset(n->d_act_rows, 0, nb * sizeof(int32_t)));
  }
  if (n->dueling) B2_CHECK_CUDA(fmalloc(&n->d_va, size_t(3) * nb * (A + 1)));
  if (n->munchausen) B2_CHECK_CUDA(fmalloc(&n->d_tdtarget, nb));
  if (cfg->max_grad_norm > 0) {   // S_l, N, c32, then k_grad_sq's partials of layers 0-4 and the embedding
    n->clip = true;
    for (int l = 0; l <= kLayers; ++l)
      n->sq_base[l + 1] = n->sq_base[l] + (l < kLayers || n->iqn_n ? cdiv(clip_layer_size(n, l), kSqChunk) : 0);
    B2_CHECK_CUDA(cudaMalloc(&n->d_clip, size_t(8 + n->sq_base[kLayers + 1]) * sizeof(double)));
    B2_CHECK_CUDA(cudaMemset(n->d_clip, 0, size_t(8 + n->sq_base[kLayers + 1]) * sizeof(double)));
  }
  if (cfg->random_shift) {
    n->crop_pad = cfg->random_shift;
    B2_CHECK_CUDA(cudaMalloc(&n->d_crop_ctr, sizeof(unsigned long long)));
    B2_CHECK_CUDA(cudaMemset(n->d_crop_ctr, 0, sizeof(unsigned long long)));
    B2_CHECK_CUDA(cudaMalloc(&n->d_crop, size_t(nb) * 4 * sizeof(int32_t)));
    B2_CHECK_CUDA(cudaMemset(n->d_crop, 0, size_t(nb) * 4 * sizeof(int32_t)));
  }
  if (n->iqn_n) {
    const size_t we = size_t(kIqnCos) * kFlat, R = size_t(xr);
    B2_CHECK_CUDA(fmalloc(&n->d_we, we));
    B2_CHECK_CUDA(fmalloc(&n->d_wes, we * n->n_states));
    if (cfg->target_steps) {
      B2_CHECK_CUDA(fmalloc(&n->d_twe, we));
      B2_CHECK_CUDA(fmalloc(&n->d_twes, we * n->n_states));
    } else {
      n->d_twe = n->d_we;
      n->d_twes = n->d_wes;
    }
    B2_CHECK_CUDA(fmalloc(&n->d_weg, we));
    if (!n->fqf_n) {   // the FQF head draws nothing
      B2_CHECK_CUDA(cudaMalloc(&n->d_tau_ctr, sizeof(unsigned long long)));
      B2_CHECK_CUDA(cudaMemset(n->d_tau_ctr, 0, sizeof(unsigned long long)));
    }
    B2_CHECK_CUDA(fmalloc(&n->d_tau, 2 * R));
    B2_CHECK_CUDA(fmalloc(&n->d_cos, 2 * R * kIqnCos));
    B2_CHECK_CUDA(fmalloc(&n->d_phi, 2 * R * kFlat));
    B2_CHECK_CUDA(fmalloc(&n->d_x, 2 * R * kFlat));
    B2_CHECK_CUDA(fmalloc(&n->d_iqn_theta, 2 * R * A));
    B2_CHECK_CUDA(fmalloc(&n->d_iqn_tq, size_t(nb) * n->iqn_n));
    B2_CHECK_CUDA(fmalloc(&n->d_iqn_qgrad, size_t(nb) * n->iqn_n));
    B2_CHECK_CUDA(fmalloc(&n->d_dx, R * kFlat));
    B2_CHECK_CUDA(fmalloc(&n->d_dphi, R * kFlat));
    B2_CHECK_CUDA(cudaMalloc(&n->d_act_rows, R * sizeof(int32_t)));
    B2_CHECK_CUDA(cudaMemset(n->d_act_rows, 0, R * sizeof(int32_t)));
    if (cfg->math_mode == B200DQN_MATH_TCGEN05) {
      B2_CHECK_CUDA(cudaMalloc(&n->d_x16, 4 * R * kFlat * sizeof(__half)));
      B2_CHECK_CUDA(cudaMemset(n->d_x16, 0, 4 * R * kFlat * sizeof(__half)));
    }
  }
  if (n->fqf_n) {
    const size_t N = size_t(n->fqf_n), wf = N * kFlat, Rb = size_t(nb) * (N - 1);
    B2_CHECK_CUDA(fmalloc(&n->d_wf, wf));
    B2_CHECK_CUDA(fmalloc(&n->d_wfs, wf * n->n_states));
    if (cfg->target_steps) {
      B2_CHECK_CUDA(fmalloc(&n->d_twf, wf));
      B2_CHECK_CUDA(fmalloc(&n->d_twfs, wf * n->n_states));
    } else {
      n->d_twf = n->d_wf;
      n->d_twfs = n->d_wfs;
    }
    B2_CHECK_CUDA(fmalloc(&n->d_wfg, wf));
    B2_CHECK_CUDA(fmalloc(&n->d_fl, size_t(nb) * N));
    B2_CHECK_CUDA(fmalloc(&n->d_fq, size_t(nb) * N));
    B2_CHECK_CUDA(fmalloc(&n->d_ftau, size_t(nb) * (N + 1)));
    B2_CHECK_CUDA(fmalloc(&n->d_fg, size_t(nb) * (N - 1)));
    B2_CHECK_CUDA(fmalloc(&n->d_fdl, size_t(nb) * N));
    B2_CHECK_CUDA(fmalloc(&n->d_btau, Rb));
    B2_CHECK_CUDA(fmalloc(&n->d_bcos, Rb * kIqnCos));
    B2_CHECK_CUDA(fmalloc(&n->d_bphi, Rb * kFlat));
    B2_CHECK_CUDA(fmalloc(&n->d_bx, Rb * kFlat));
    B2_CHECK_CUDA(fmalloc(&n->d_bh4, Rb * kHidden));
    B2_CHECK_CUDA(fmalloc(&n->d_btheta, Rb * A));
    if (cfg->math_mode == B200DQN_MATH_TCGEN05) {
      B2_CHECK_CUDA(cudaMalloc(&n->d_bx16, 2 * Rb * kFlat * sizeof(__half)));
      B2_CHECK_CUDA(cudaMemset(n->d_bx16, 0, 2 * Rb * kFlat * sizeof(__half)));
    }
  }
  const size_t state_bytes = size_t(nb) * hist * kFrameBytes;
  B2_CHECK_CUDA(cudaMalloc(&n->d_pre, state_bytes + 256));
  B2_CHECK_CUDA(cudaMalloc(&n->d_post, state_bytes + 256));
  B2_CHECK_CUDA(cudaMalloc(&n->d_act, nb));
  B2_CHECK_CUDA(cudaMalloc(&n->d_term, nb));
  B2_CHECK_CUDA(cudaMalloc(&n->d_rew, nb * sizeof(int64_t)));
  B2_CHECK_CUDA(cudaMalloc(&n->d_iota1, nb * sizeof(int32_t)));
  B2_CHECK_CUDA(cudaMalloc(&n->d_iota4, nb * sizeof(int32_t)));
  k_iota<<<cdiv(nb, 128), 128>>>(n->d_iota1, n->d_iota4, nb, hist);
  B2_LAUNCH_CHECK();
  n->pin_bytes = 2 * state_bytes + size_t(nb) * 16 + size_t(nb) * A * sizeof(float) + 256;
  B2_CHECK_CUDA(cudaMallocHost(&n->h_pin, n->pin_bytes));
  {
    void* m = nullptr;
    B2_CHECK_CUDA(cudaHostAlloc(&m, 4096, cudaHostAllocMapped));
    memset(m, 0, 4096);
    n->h_res = static_cast<volatile uint32_t*>(m);
  }
  {
    int prio_lo = 0, prio_hi = 0;   // numerically larger = lower priority
    B2_CHECK_CUDA(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
    for (int i = 0; i < 4; ++i)   // the three wgrad/optimizer branches low, the collective stream high
      B2_CHECK_CUDA(cudaStreamCreateWithPriority(&n->side[i], cudaStreamNonBlocking, i < 3 ? prio_lo : prio_hi));
  }
  for (auto& e : n->ev) B2_CHECK_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  n->use_graph = getenv("B200DQN_NO_GRAPH") == nullptr;
  n->use_branches = getenv("B200DQN_NO_BRANCHES") == nullptr;
  int rc = umma_net_init(n);
  if (rc) return rc;
  if (n->munchausen && n->d_tw != n->d_w && (rc = double_q_alloc(n))) return rc;   // the target pass's third slot
  B2_CHECK_CUDA(cudaDeviceSynchronize());
  *out = n;
  return B200DQN_OK;
}

extern "C" int b200dqn_net_destroy(b200dqn_net* n) {
  if (!n) return B200DQN_OK;
  DeviceGuard g(n->device);
  cudaDeviceSynchronize();
  comm_destroy(n);
  umma_net_destroy(n);
  destroy_step_graphs(n);
  n->graph_predict.drop();
  for (auto& sd : n->side) if (sd) cudaStreamDestroy(sd);
  for (auto& e : n->ev) if (e) cudaEventDestroy(e);
  if (n->d_tw != n->d_w) { cudaFree(n->d_tw); cudaFree(n->d_ts); }
  cudaFree(n->d_optscal);
  cudaFree(n->d_w); cudaFree(n->d_s); cudaFree(n->d_g); cudaFree(n->d_part); cudaFree(n->d_xepoch);
  for (int z = 0; z < 3; ++z) {
    cudaFree(n->d_h1[z]); cudaFree(n->d_h2[z]); cudaFree(n->d_h3[z]); cudaFree(n->d_q[z]);
  }
  for (int z = 0; z < 2; ++z) cudaFree(n->d_h4[z]);
  cudaFree(n->d_fc1part); cudaFree(n->d_delta); cudaFree(n->d_dz4); cudaFree(n->d_dz3); cudaFree(n->d_dz2);
  cudaFree(n->d_dz1); cudaFree(n->d_cost); cudaFree(n->d_step); cudaFree(n->d_rowcost); cudaFree(n->d_pre); cudaFree(n->d_post);
  cudaFree(n->d_act); cudaFree(n->d_term); cudaFree(n->d_rew); cudaFree(n->d_iota1); cudaFree(n->d_iota4);
  cudaFree(n->d_td_err);
  cudaFree(n->d_logits); cudaFree(n->d_probs); cudaFree(n->d_tdist); cudaFree(n->d_lgrad); cudaFree(n->d_act_rows);
  cudaFree(n->d_va);
  cudaFree(n->d_theta); cudaFree(n->d_tquant); cudaFree(n->d_qgrad);
  cudaFree(n->d_rem_ctr); cudaFree(n->d_rem_alpha); cudaFree(n->d_rem_grad);
  cudaFree(n->d_boot_mask); cudaFree(n->d_boot_y); cudaFree(n->d_boot_delta); cudaFree(n->d_boot_head);
  cudaFree(n->d_tdtarget);
  if (n->d_twe != n->d_we) { cudaFree(n->d_twe); cudaFree(n->d_twes); }
  cudaFree(n->d_crop_ctr); cudaFree(n->d_crop);
  cudaFree(n->d_clip);
  cudaFree(n->d_we); cudaFree(n->d_wes); cudaFree(n->d_weg); cudaFree(n->d_tau_ctr); cudaFree(n->d_tau);
  cudaFree(n->d_cos); cudaFree(n->d_phi); cudaFree(n->d_x); cudaFree(n->d_iqn_theta); cudaFree(n->d_iqn_tq);
  cudaFree(n->d_iqn_qgrad); cudaFree(n->d_dx); cudaFree(n->d_dphi); cudaFree(n->d_x16);
  if (n->d_twf != n->d_wf) { cudaFree(n->d_twf); cudaFree(n->d_twfs); }
  cudaFree(n->d_wf); cudaFree(n->d_wfs); cudaFree(n->d_wfg); cudaFree(n->d_fl); cudaFree(n->d_fq); cudaFree(n->d_ftau);
  cudaFree(n->d_fg); cudaFree(n->d_fdl); cudaFree(n->d_btau); cudaFree(n->d_bcos); cudaFree(n->d_bphi); cudaFree(n->d_bx);
  cudaFree(n->d_bh4); cudaFree(n->d_btheta); cudaFree(n->d_bx16);
  cudaFreeHost(n->h_pin);
  cudaFreeHost(const_cast<uint32_t*>(n->h_res));
  delete n;
  return B200DQN_OK;
}

// ABI layer 5, the IQN embedding: Neon W[n][i], n = fc1's input column in (c, p, q) order, i < 64 <-> internal
// We[i][(p, q, c)].  These take over the five-layer entry points' work for it.
static int xfer_we(b200dqn_net* n, float* dev_base, float* host, bool to_device, cudaStream_t st) {
  const int64_t cnt = int64_t(kIqnCos) * kFlat;
  std::vector<float> tmp(cnt);
  auto at = [](int64_t i) {
    const int nn = int(i / kIqnCos), f = int(i % kIqnCos);
    const int c = nn / 49, p = (nn / 7) % 7, q = nn % 7;
    return int64_t(f) * kFlat + (p * 7 + q) * kC3 + c;
  };
  if (to_device) {
    for (int64_t i = 0; i < cnt; ++i) tmp[at(i)] = host[i];
    B2_CHECK_CUDA(cudaMemcpyAsync(dev_base, tmp.data(), cnt * sizeof(float), cudaMemcpyHostToDevice, st));
    B2_CHECK_CUDA(cudaStreamSynchronize(st));
  } else {
    B2_CHECK_CUDA(cudaMemcpyAsync(tmp.data(), dev_base, cnt * sizeof(float), cudaMemcpyDeviceToHost, st));
    B2_CHECK_CUDA(cudaStreamSynchronize(st));
    for (int64_t i = 0; i < cnt; ++i) host[i] = tmp[at(i)];
  }
  return B200DQN_OK;
}

static bool is_we(const b200dqn_net* n, int layer) { return layer == kLayers && n->iqn_n; }

// ABI layer 6, the FQF fraction layer: Neon W_f[k][n], n = fc1's input column in (c, p, q) order <-> internal
// W_f[k][(p, q, c)]
static int xfer_wf(b200dqn_net* n, float* dev_base, float* host, bool to_device, cudaStream_t st) {
  const int64_t cnt = int64_t(n->fqf_n) * kFlat;
  std::vector<float> tmp(cnt);
  auto at = [](int64_t i) {
    const int k = int(i / kFlat), nn = int(i % kFlat);
    const int c = nn / 49, p = (nn / 7) % 7, q = nn % 7;
    return int64_t(k) * kFlat + (p * 7 + q) * kC3 + c;
  };
  if (to_device) {
    for (int64_t i = 0; i < cnt; ++i) tmp[at(i)] = host[i];
    B2_CHECK_CUDA(cudaMemcpyAsync(dev_base, tmp.data(), cnt * sizeof(float), cudaMemcpyHostToDevice, st));
    B2_CHECK_CUDA(cudaStreamSynchronize(st));
  } else {
    B2_CHECK_CUDA(cudaMemcpyAsync(tmp.data(), dev_base, cnt * sizeof(float), cudaMemcpyDeviceToHost, st));
    B2_CHECK_CUDA(cudaStreamSynchronize(st));
    for (int64_t i = 0; i < cnt; ++i) host[i] = tmp[at(i)];
  }
  return B200DQN_OK;
}

static bool is_wf(const b200dqn_net* n, int layer) { return layer == kLayers + 1 && n->fqf_n; }
// a layer index valid on this net: the five of every net, the embedding (IQN, FQF), the fraction layer (FQF)
static bool layer_ok(const b200dqn_net* n, int layer) { return layer >= 0 && (layer < kLayers || is_we(n, layer) || is_wf(n, layer)); }

extern "C" int b200dqn_net_layer_shape(const b200dqn_net* n, int layer, int* rows, int* cols) {
  B2_REQUIRE(n && layer_ok(n, layer), B200DQN_EINVAL, "net_layer_shape: bad layer");
  if (layer == kLayers + 1) {
    if (rows) *rows = n->fqf_n;
    if (cols) *cols = kFlat;
    return B200DQN_OK;
  }
  if (layer == kLayers) {
    if (rows) *rows = kFlat;
    if (cols) *cols = kIqnCos;
    return B200DQN_OK;
  }
  // NEON shapes: conv (C*R*S, K); linear (nout, nin)
  const int r[kLayers] = {n->lt.rows[0], kK2, kK3, n->hidden, n->fc2_cols()};
  const int c[kLayers] = {kC1, kC2, kC3, kFlat, kHidden};
  if (rows) *rows = r[layer];
  if (cols) *cols = c[layer];
  return B200DQN_OK;
}

static int xfer_params(b200dqn_net* n, float* dev_base, int layer, float* host, bool to_device, cudaStream_t st) {
  const int64_t off = n->lt.off[layer], cnt = n->lt.off[layer + 1] - off;
  std::vector<float> tmp(cnt);
  if (to_device) {
    for (int64_t i = 0; i < cnt; ++i) tmp[neon_to_internal(layer, i, n->fc2_cols(), n->hidden)] = host[i];
    B2_CHECK_CUDA(cudaMemcpyAsync(dev_base + off, tmp.data(), cnt * sizeof(float), cudaMemcpyHostToDevice, st));
    B2_CHECK_CUDA(cudaStreamSynchronize(st));
  } else {
    B2_CHECK_CUDA(cudaMemcpyAsync(tmp.data(), dev_base + off, cnt * sizeof(float), cudaMemcpyDeviceToHost, st));
    B2_CHECK_CUDA(cudaStreamSynchronize(st));
    for (int64_t i = 0; i < cnt; ++i) host[i] = tmp[neon_to_internal(layer, i, n->fc2_cols(), n->hidden)];
  }
  return B200DQN_OK;
}

extern "C" int b200dqn_net_set_weights(b200dqn_net* n, int which, int layer, const float* host_W,
                                       const float* host_S, void* stream) {
  B2_REQUIRE(n && host_W && layer_ok(n, layer) && (which == 0 || which == 1), B200DQN_EINVAL,
             "net_set_weights: bad argument");
  DeviceGuard g(n->device);
  cudaStream_t st = as_stream(stream);
  if (layer == kLayers + 1) {
    B2_TRY(xfer_wf(n, which ? n->d_twf : n->d_wf, const_cast<float*>(host_W), true, st));
    if (host_S) B2_TRY(xfer_wf(n, which ? n->d_twfs : n->d_wfs, const_cast<float*>(host_S), true, st));
    return B200DQN_OK;
  }
  if (layer == kLayers) {
    B2_TRY(xfer_we(n, which ? n->d_twe : n->d_we, const_cast<float*>(host_W), true, st));
    if (host_S) B2_TRY(xfer_we(n, which ? n->d_twes : n->d_wes, const_cast<float*>(host_S), true, st));
    return B200DQN_OK;
  }
  int rc = xfer_params(n, which ? n->d_tw : n->d_w, layer, const_cast<float*>(host_W), true, st);
  if (rc) return rc;
  if (host_S && (rc = xfer_params(n, which ? n->d_ts : n->d_s, layer, const_cast<float*>(host_S), true, st))) return rc;
  return umma_weights_changed(n, st);
}

extern "C" int b200dqn_net_get_weights(b200dqn_net* n, int which, int layer, float* host_W, float* host_S,
                                       void* stream) {
  B2_REQUIRE(n && layer_ok(n, layer) && (which == 0 || which == 1), B200DQN_EINVAL, "net_get_weights: bad argument");
  DeviceGuard g(n->device);
  cudaStream_t st = as_stream(stream);
  if (layer == kLayers + 1) {
    if (host_W) B2_TRY(xfer_wf(n, which ? n->d_twf : n->d_wf, host_W, false, st));
    if (host_S) B2_TRY(xfer_wf(n, which ? n->d_twfs : n->d_wfs, host_S, false, st));
    return B200DQN_OK;
  }
  if (layer == kLayers) {
    if (host_W) B2_TRY(xfer_we(n, which ? n->d_twe : n->d_we, host_W, false, st));
    if (host_S) B2_TRY(xfer_we(n, which ? n->d_twes : n->d_wes, host_S, false, st));
    return B200DQN_OK;
  }
  int rc;
  if (host_W && (rc = xfer_params(n, which ? n->d_tw : n->d_w, layer, host_W, false, st))) return rc;
  if (host_S && (rc = xfer_params(n, which ? n->d_ts : n->d_s, layer, host_S, false, st))) return rc;
  return B200DQN_OK;
}

extern "C" int b200dqn_net_num_states(const b200dqn_net* n, int* count) {
  B2_REQUIRE(n && count, B200DQN_EINVAL, "net_num_states: null argument");
  *count = n->n_states;
  return B200DQN_OK;
}

extern "C" int b200dqn_net_set_state(b200dqn_net* n, int which, int layer, int k, const float* host_S, void* stream) {
  B2_REQUIRE(n && host_S && layer_ok(n, layer) && (which == 0 || which == 1) && k >= 0 && k < n->n_states,
             B200DQN_EINVAL, "net_set_state: bad argument");
  DeviceGuard g(n->device);
  if (layer == kLayers + 1)
    return xfer_wf(n, (which ? n->d_twfs : n->d_wfs) + int64_t(k) * n->fqf_n * kFlat, const_cast<float*>(host_S), true,
                   as_stream(stream));
  if (layer == kLayers)
    return xfer_we(n, (which ? n->d_twes : n->d_wes) + int64_t(k) * kIqnCos * kFlat, const_cast<float*>(host_S), true,
                   as_stream(stream));
  return xfer_params(n, (which ? n->d_ts : n->d_s) + int64_t(k) * n->n_params, layer, const_cast<float*>(host_S), true,
                     as_stream(stream));
}

extern "C" int b200dqn_net_get_state(b200dqn_net* n, int which, int layer, int k, float* host_S, void* stream) {
  B2_REQUIRE(n && host_S && layer_ok(n, layer) && (which == 0 || which == 1) && k >= 0 && k < n->n_states,
             B200DQN_EINVAL, "net_get_state: bad argument");
  DeviceGuard g(n->device);
  if (layer == kLayers + 1)
    return xfer_wf(n, (which ? n->d_twfs : n->d_wfs) + int64_t(k) * n->fqf_n * kFlat, host_S, false, as_stream(stream));
  if (layer == kLayers)
    return xfer_we(n, (which ? n->d_twes : n->d_wes) + int64_t(k) * kIqnCos * kFlat, host_S, false, as_stream(stream));
  return xfer_params(n, (which ? n->d_ts : n->d_s) + int64_t(k) * n->n_params, layer, host_S, false, as_stream(stream));
}

extern "C" int b200dqn_net_sync_target(b200dqn_net* n, void* stream) {
  B2_REQUIRE(n, B200DQN_EINVAL, "null net");
  if (n->d_tw == n->d_w) return B200DQN_OK;  // target_steps == 0: alias
  DeviceGuard g(n->device);
  cudaStream_t st = as_stream(stream);
  B2_CHECK_CUDA(cudaMemcpyAsync(n->d_tw, n->d_w, n->n_params * sizeof(float), cudaMemcpyDeviceToDevice, st));
  B2_CHECK_CUDA(cudaMemcpyAsync(n->d_ts, n->d_s, n->n_params * n->n_states * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (n->iqn_n) {   // the embedding is a layer of each network
    const size_t we = size_t(kIqnCos) * kFlat * sizeof(float);
    B2_CHECK_CUDA(cudaMemcpyAsync(n->d_twe, n->d_we, we, cudaMemcpyDeviceToDevice, st));
    B2_CHECK_CUDA(cudaMemcpyAsync(n->d_twes, n->d_wes, we * n->n_states, cudaMemcpyDeviceToDevice, st));
  }
  if (n->fqf_n) {   // and so is the fraction layer
    const size_t wf = size_t(n->fqf_n) * kFlat * sizeof(float);
    B2_CHECK_CUDA(cudaMemcpyAsync(n->d_twf, n->d_wf, wf, cudaMemcpyDeviceToDevice, st));
    B2_CHECK_CUDA(cudaMemcpyAsync(n->d_twfs, n->d_wfs, wf * n->n_states, cudaMemcpyDeviceToDevice, st));
  }
  return umma_target_synced(n, st);
}

extern "C" int b200dqn_net_soft_update_target(b200dqn_net* n, double tau, void* stream) {
  B2_REQUIRE(n, B200DQN_EINVAL, "null net");
  B2_REQUIRE(std::isfinite(tau) && tau > 0 && tau <= 1, B200DQN_EINVAL,
             "net_soft_update_target: tau must be finite and in (0, 1] (got %g)", tau);
  B2_REQUIRE(n->d_tw != n->d_w, B200DQN_EINVAL,
             "net_soft_update_target: target_steps = 0 makes the target the online network; there is nothing to blend");
  DeviceGuard g(n->device);
  cudaStream_t st = as_stream(stream);
  const float c = float(1.0 - tau), t = float(tau);
  B2_TRY(soft_update_layers(n, 0, kLayers - 1, c, t, st));
  return soft_update_extra(n, c, t, st);
}

// Captures what enqueue() puts on key.stream into a CUDA graph held by c, unless c already holds one captured at key.
template <class F>
static int graph_cached(GraphCache& c, const GraphKey& key, F&& enqueue) {
  if (c.exec && c.key == key) return B200DQN_OK;
  c.drop();
  cudaGraph_t graph = nullptr;
  B2_CHECK_CUDA(cudaStreamBeginCapture(key.stream, cudaStreamCaptureModeThreadLocal));
  const int rc = enqueue();
  cudaError_t e = cudaStreamEndCapture(key.stream, &graph);
  if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
  B2_CHECK_CUDA(e);
  B2_CHECK_CUDA(cudaGraphInstantiate(&c.exec, graph, 0));
  cudaGraphDestroy(graph);
  c.key = key;
  return B200DQN_OK;
}

extern "C" int b200dqn_net_predict_device(b200dqn_net* n, const uint8_t* dev_states, int live_rows, float* dev_q,
                                          void* stream) {
  B2_REQUIRE(n && dev_states && dev_q && live_rows >= 1 && live_rows <= n->nb, B200DQN_EINVAL,
             "net_predict_device: bad argument");
  DeviceGuard g(n->device);
  cudaStream_t st = as_stream(stream);
  FrameSource fs{{dev_states, dev_states}, {n->d_iota4, n->d_iota4}, {0, 0}};
  HeadTrainArgs no_td{};
  int rc = forward(n, fs, 1, live_rows, st, no_td);
  if (rc) return rc;
  if (dev_q != n->d_q[0])
    B2_CHECK_CUDA(cudaMemcpyAsync(dev_q, n->d_q[0], size_t(live_rows) * n->A * sizeof(float),
                                  cudaMemcpyDeviceToDevice, st));
  if (live_rows < n->nb) {
    k_zero_rows<<<cdiv((n->nb - live_rows) * n->A, 128), 128, 0, st>>>(dev_q, live_rows, n->nb, n->A);
    B2_LAUNCH_CHECK();
  }
  return B200DQN_OK;
}

// Q rows of a fast-path predict -> host-mapped memory: data, system fence, sequence number
__global__ void k_publish_q_counter(const float* __restrict__ q, int count, volatile uint32_t* host_res, uint32_t* counter) {
  for (int i = threadIdx.x; i < count; i += blockDim.x) host_res[kHostQ + i] = __float_as_uint(q[i]);
  __syncthreads();
  if (threadIdx.x == 0) {
    const uint32_t seq = *counter + 1;     // device-resident count of fast-path predicts: the graph replays unchanged
    *counter = seq;
    __threadfence_system();
    host_res[2] = seq;
  }
}

// agent.py:55-61 on a device-resident state window (StateBuffer): the forward pass for the live rows, captured once
// into a CUDA graph (one launch per env step), Q rows back through host-mapped memory (no memcpy, polled).
// host_q receives (batch, A); rows >= live_rows are padding and come back as exact zeros.
extern "C" int b200dqn_net_predict_device_host(b200dqn_net* n, const uint8_t* dev_states, int live_rows, float* host_q,
                                               void* stream) {
  B2_REQUIRE(n && dev_states && host_q && live_rows >= 1 && live_rows <= n->nb, B200DQN_EINVAL,
             "net_predict_device_host: bad argument");
  DeviceGuard g(n->device);
  cudaStream_t st = as_stream(stream);
  const int count = live_rows * n->A;
  if (count > kHostQFloats || st == nullptr || !n->use_graph || g_prof_on) {   // general path: device predict + copy
    int rc = b200dqn_net_predict_device(n, dev_states, live_rows, n->d_q[0], stream);
    if (rc) return rc;
    B2_CHECK_CUDA(cudaMemcpyAsync(host_q, n->d_q[0], size_t(n->nb) * n->A * sizeof(float), cudaMemcpyDeviceToHost, st));
    B2_CHECK_CUDA(cudaStreamSynchronize(st));
    return B200DQN_OK;
  }
  GraphKey key;
  key.src = dev_states; key.rows = live_rows; key.stream = st;
  B2_TRY(graph_cached(n->graph_predict, key, [&] {
    FrameSource fs{{dev_states, dev_states}, {n->d_iota4, n->d_iota4}, {0, 0}};
    HeadTrainArgs no_td{};
    int rc = forward(n, fs, 1, live_rows, st, no_td);
    if (!rc) {
      k_publish_q_counter<<<1, 64, 0, st>>>(n->d_q[0], count, n->h_res, n->d_optscal_u32());
      if (cudaGetLastError() != cudaSuccess) rc = B200DQN_ECUDA;
    }
    return rc;
  }));
  B2_CHECK_CUDA(cudaGraphLaunch(n->graph_predict.exec, st));
  n->predicts_launched += 1;
  int rc = poll_mapped_seq(n->h_res + 2, n->predicts_launched, st, "predict result");
  if (rc) return rc;
  for (int i = 0; i < count; ++i) {
    const uint32_t bits = n->h_res[kHostQ + i];
    memcpy(host_q + i, &bits, sizeof(float));
  }
  memset(host_q + count, 0, (size_t(n->nb) * n->A - count) * sizeof(float));
  return B200DQN_OK;
}

extern "C" int b200dqn_net_predict(b200dqn_net* n, const uint8_t* host_states, float* host_q, void* stream) {
  B2_REQUIRE(n && host_states && host_q, B200DQN_EINVAL, "net_predict: null argument");
  DeviceGuard g(n->device);
  cudaStream_t st = as_stream(stream);
  const size_t state_bytes = size_t(n->nb) * n->cfg.history_length * kFrameBytes;
  memcpy(n->h_pin, host_states, state_bytes);
  B2_CHECK_CUDA(cudaMemcpyAsync(n->d_pre, n->h_pin, state_bytes, cudaMemcpyHostToDevice, st));
  int rc = b200dqn_net_predict_device(n, n->d_pre, n->nb, n->d_q[0], stream);
  if (rc) return rc;
  float* hq = reinterpret_cast<float*>(n->h_pin + 2 * state_bytes + size_t(n->nb) * 16);
  B2_CHECK_CUDA(cudaMemcpyAsync(hq, n->d_q[0], size_t(n->nb) * n->A * sizeof(float), cudaMemcpyDeviceToHost, st));
  B2_CHECK_CUDA(cudaStreamSynchronize(st));
  memcpy(host_q, hq, size_t(n->nb) * n->A * sizeof(float));
  return B200DQN_OK;
}

// A host-supplied minibatch names its rows 0..nb-1, not ring slots, so it has no bootstrap mask of its own; at p = 1
// every mask is 1 and the rows need none.
static int check_host_rows_maskable(const b200dqn_net* n, const char* who) {
  B2_REQUIRE(!n->boot || n->cfg.bootstrap_p >= 1.0, B200DQN_ENOTIMPL,
             "%s: bootstrapped heads with bootstrap_p = %g < 1 mask each transition by its ring slot; a host-supplied "
             "minibatch has none (train from the replay ring)", who, n->cfg.bootstrap_p);
  return B200DQN_OK;
}

extern "C" int b200dqn_net_train_device(b200dqn_net* n, const uint8_t* dev_pre, const uint8_t* dev_actions,
                                        const int64_t* dev_rewards, const uint8_t* dev_post,
                                        const uint8_t* dev_terminals, void* stream) {
  B2_REQUIRE(n && dev_pre && dev_actions && dev_rewards && dev_post && dev_terminals, B200DQN_EINVAL,
             "net_train_device: null argument");
  B2_TRY(check_host_rows_maskable(n, "net_train_device"));
  DeviceGuard g(n->device);
  FrameSource fs{{dev_pre, dev_post}, {n->d_iota4, n->d_iota4}, {0, 0}};
  B2_TRY(train_step(n, fs, dev_actions, dev_rewards, dev_terminals, n->d_iota1, as_stream(stream)));
  n->train_iterations += 1;
  return B200DQN_OK;
}

extern "C" int b200dqn_net_train(b200dqn_net* n, const uint8_t* host_pre, const uint8_t* host_actions,
                                 const int64_t* host_rewards, const uint8_t* host_post, const uint8_t* host_terminals,
                                 float* host_cost, void* stream) {
  B2_REQUIRE(n && host_pre && host_actions && host_rewards && host_post && host_terminals, B200DQN_EINVAL,
             "net_train: null argument");
  B2_TRY(check_host_rows_maskable(n, "net_train"));
  for (int i = 0; i < n->nb; ++i)
    B2_REQUIRE(host_actions[i] < n->A, B200DQN_EINVAL, "net_train: action %d >= num_actions %d", host_actions[i], n->A);
  DeviceGuard g(n->device);
  cudaStream_t st = as_stream(stream);
  const size_t sb = size_t(n->nb) * n->cfg.history_length * kFrameBytes;
  uint8_t* p = n->h_pin;
  memcpy(p, host_pre, sb);
  memcpy(p + sb, host_post, sb);
  uint8_t* meta = p + 2 * sb;
  memcpy(meta, host_rewards, n->nb * 8);
  memcpy(meta + n->nb * 8, host_actions, n->nb);
  memcpy(meta + n->nb * 9, host_terminals, n->nb);
  B2_CHECK_CUDA(cudaMemcpyAsync(n->d_pre, p, sb, cudaMemcpyHostToDevice, st));
  B2_CHECK_CUDA(cudaMemcpyAsync(n->d_post, p + sb, sb, cudaMemcpyHostToDevice, st));
  B2_CHECK_CUDA(cudaMemcpyAsync(n->d_rew, meta, n->nb * 8, cudaMemcpyHostToDevice, st));
  B2_CHECK_CUDA(cudaMemcpyAsync(n->d_act, meta + n->nb * 8, n->nb, cudaMemcpyHostToDevice, st));
  B2_CHECK_CUDA(cudaMemcpyAsync(n->d_term, meta + n->nb * 9, n->nb, cudaMemcpyHostToDevice, st));
  int rc = b200dqn_net_train_device(n, n->d_pre, n->d_act, n->d_rew, n->d_post, n->d_term, stream);
  if (rc) return rc;
  if (host_cost) return b200dqn_net_read_costs(n, 1, host_cost, stream);
  B2_CHECK_CUDA(cudaStreamSynchronize(st));
  return B200DQN_OK;
}

static int check_fusable(b200dqn_net* n, b200dqn_replay* r) {
  B2_REQUIRE(r->device == n->device, B200DQN_EINVAL, "train_fused: replay and net live on different devices");
  B2_REQUIRE(r->h == kFrameH && r->w == kFrameW && r->hist == n->cfg.history_length, B200DQN_EINVAL,
             "train_fused: replay geometry (%dx%dx%d) differs from the network's (%dx%dx%d)", r->h, r->w, r->hist,
             kFrameH, kFrameW, n->cfg.history_length);
  B2_REQUIRE(r->batch == n->nb * n->world, B200DQN_EINVAL,
             "train_fused: replay batch (%d) must equal the global minibatch %d x %d", r->batch, n->nb, n->world);
  if (r->per_on) {
    B2_REQUIRE(n->world == 1 && !n->nccl_comm, B200DQN_ENOTIMPL,
               "prioritized replay is implemented for a single learner only (comm_init has run)");
    if (!n->d_td_err) {   // the first step on a prioritized ring (before any graph capture)
      DeviceGuard g(n->device);
      B2_CHECK_CUDA(cudaMalloc(&n->d_td_err, n->nb * sizeof(float)));
      B2_CHECK_CUDA(cudaMemset(n->d_td_err, 0, n->nb * sizeof(float)));
    }
  }
  if (r->nstep > 1) {
    B2_REQUIRE(n->world == 1 && !n->nccl_comm, B200DQN_ENOTIMPL,
               "n-step returns are implemented for a single learner only (comm_init has run)");
  }
  n->ring_nstep = r->nstep;
  return B200DQN_OK;
}

static int train_on_ring(b200dqn_net* n, b200dqn_replay* r, cudaStream_t st) {
  const int32_t* my_idx = r->d_idx + n->rank * n->nb;  // this rank's slice of the global minibatch
  // prestates = frames index-H .. index-1, poststates = index-H+N .. index+N-1 (src/replay_memory.py:71-72 at N = 1)
  const int hist = n->cfg.history_length;
  FrameSource fs{{r->d_screens, r->d_screens}, {my_idx, my_idx}, {-hist, -hist + r->nstep}};
  n->step_replay = r;
  const int rc = train_step(n, fs, r->d_actions, r->d_rewards, r->d_terminals, my_idx, st);
  n->step_replay = nullptr;
  return rc;
}

// what a step graph on ring r and stream st is captured at
static GraphKey step_graph_key(const b200dqn_net* n, const b200dqn_replay* r, cudaStream_t st) {
  GraphKey k;
  k.src = r; k.serial = r->serial; k.stream = st; k.world = n->world; k.trace_gen = g_ktrace_gen;
  k.per_gen = r->per_gen; k.nstep = r->nstep;
  return k;
}

// train_on_ring through a cached CUDA graph (the sampler is NOT part of it: the indexes are already in r)
static int train_sampled_launch(b200dqn_net* n, b200dqn_replay* r, cudaStream_t st) {
  const bool use_graph = n->use_graph && !g_prof_on && st != nullptr;
  if (!use_graph) return train_on_ring(n, r, st);
  B2_TRY(graph_cached(n->graph_train, step_graph_key(n, r, st), [&] { return train_on_ring(n, r, st); }));
  B2_CHECK_CUDA(cudaGraphLaunch(n->graph_train.exec, st));
  return B200DQN_OK;
}

extern "C" int b200dqn_net_train_sampled(b200dqn_net* n, b200dqn_replay* r, void* stream) {
  B2_REQUIRE(n && r, B200DQN_EINVAL, "net_train_sampled: null argument");
  int rc = check_fusable(n, r);
  if (rc) return rc;
  DeviceGuard g(n->device);
  B2_TRY(replay_flush(r, as_stream(stream)));   // pending add()s reach the ring first (not part of the graph)
  B2_TRY(train_sampled_launch(n, r, as_stream(stream)));
  n->train_iterations += 1;
  return B200DQN_OK;
}

// wait for train step number `want` (1-based count of steps run by this net) and fetch its cost from the mapped block
static int wait_step_cost(b200dqn_net* n, cudaStream_t st, uint32_t want, float* cost) {
  int rc = poll_mapped_seq(n->h_res, want, st, "train step result");
  if (rc) return rc;
  B2_REQUIRE(n->h_res[1] == 0, B200DQN_EINVAL,
             "train: a sampled action is >= num_actions %d (IndexError at deepqnetwork.py:141 in the reference)", n->A);
  if (cost) {
    const uint32_t bits = n->h_res[4 + (want - 1) % kHostCosts];
    memcpy(cost, &bits, sizeof(float));
  }
  return B200DQN_OK;
}

extern "C" int b200dqn_net_train_sampled_cost(b200dqn_net* n, b200dqn_replay* r, float* host_cost, void* stream) {
  B2_REQUIRE(host_cost, B200DQN_EINVAL, "net_train_sampled_cost: null argument");
  int rc = b200dqn_net_train_sampled(n, r, stream);
  if (rc) return rc;
  return wait_step_cost(n, as_stream(stream), uint32_t(n->train_iterations), host_cost);
}

// The head of a fused step: the trace tick, the random-shift draw's fork and the sampler.  The sampler must not start
// ahead of the tick.
static int sample_step_head(b200dqn_net* n, b200dqn_replay* r, cudaStream_t st) {
  auto head = [&] {
    int rc = shift_fork(n, st);
    if (!rc) rc = launch_sample(r, st);
    if (rc) n->crop_forked = false;
    return rc;
  };
  if (!ktrace_tick(st)) return head();
  NoPdlScope after_tick;
  return head();
}

extern "C" int b200dqn_net_train_fused(b200dqn_net* n, b200dqn_replay* r, int nsteps, void* stream) {
  B2_REQUIRE(n && r && nsteps >= 1, B200DQN_EINVAL, "net_train_fused: bad argument");
  int rc = check_fusable(n, r);
  if (rc) return rc;
  B2_REQUIRE(r->count >= r->hist + r->nstep, B200DQN_ESTATE,
             "getMinibatch: count must be at least history_length + n_step");
  B2_REQUIRE(r->rng_set, B200DQN_ESTATE, "net_train_fused: call b200dqn_replay_set_rng first");
  DeviceGuard g(n->device);
  cudaStream_t st = as_stream(stream);
  B2_TRY(replay_flush(r, st));
  // The whole step (sampler + 15 kernels, three side branches) is captured once into a CUDA graph
  // and replayed: one graph launch per step instead of ~17 stream operations.
  const bool use_graph = n->use_graph && !g_prof_on && st != nullptr;
  if (use_graph) {
    B2_TRY(graph_cached(n->graph_step, step_graph_key(n, r, st), [&] {
      const long long launches_before = g_launch_count;
      int rc = sample_step_head(n, r, st);
      if (!rc) rc = train_on_ring(n, r, st);
      n->graph_launches = int(g_launch_count - launches_before);
      return rc;
    }));
    for (int i = 0; i < nsteps; ++i) B2_CHECK_CUDA(cudaGraphLaunch(n->graph_step.exec, st));
  } else {
    for (int i = 0; i < nsteps; ++i) {
      B2_TRY(sample_step_head(n, r, st));
      B2_TRY(train_on_ring(n, r, st));
    }
  }
  n->train_iterations += nsteps;
  r->samples_launched += uint32_t(nsteps);
  return B200DQN_OK;
}

// agent.py:102-114 as ONE call (see include/b200dqn.h)
extern "C" int b200dqn_net_step_host(b200dqn_net* n, b200dqn_replay* r, int nframes, const uint8_t* host_actions,
                                     const int64_t* host_rewards, const uint8_t* host_frames,
                                     const uint8_t* host_terminals, int train_repeat, const uint32_t* host_key624,
                                     uint32_t host_pos, float* host_costs, uint32_t* host_words_consumed, void* stream) {
  B2_REQUIRE(n && r && nframes >= 0 && train_repeat >= 0 && train_repeat <= kHostCosts, B200DQN_EINVAL,
             "net_step_host: bad argument");
  B2_REQUIRE(nframes == 0 || (host_actions && host_rewards && host_frames && host_terminals), B200DQN_EINVAL,
             "net_step_host: null frame arrays");
  for (int i = 0; i < nframes; ++i) {     // ReplayMemory.add x nframes (replay_memory.py:26-34): pinned bank, deferred
    int rc = b200dqn_replay_add(r, host_actions[i], host_rewards[i], host_frames + size_t(i) * r->frame_bytes,
                                host_terminals[i], stream);
    if (rc) return rc;
  }
  if (train_repeat == 0) return B200DQN_OK;
  DeviceGuard g(n->device);
  cudaStream_t st = as_stream(stream);
  int rc;
  if (host_key624 && (rc = replay_set_rng_async(r, host_key624, host_pos, st))) return rc;   // the host stream moved
  uint32_t words_before = 0;
  if (host_words_consumed) {              // running totals: exact across several samplings, once earlier ones are in
    if ((rc = replay_wait_words(r, st))) return rc;
    words_before = r->h_words[2];
  }
  rc = b200dqn_net_train_fused(n, r, train_repeat, stream);
  if (rc) return rc;
  if (!host_costs && !host_words_consumed) return B200DQN_OK;      // asynchronous
  float last = 0.f;
  rc = wait_step_cost(n, st, uint32_t(n->train_iterations), &last);   // the last step's cost is published last
  if (rc) return rc;
  if (host_costs)
    for (int i = 0; i < train_repeat; ++i) {
      const uint32_t bits = n->h_res[4 + (uint32_t(n->train_iterations) - train_repeat + i) % kHostCosts];
      memcpy(host_costs + i, &bits, sizeof(float));
    }
  if (host_words_consumed) {
    rc = replay_wait_words(r, st);
    if (rc) return rc;
    *host_words_consumed = r->h_words[2] - words_before;   // running totals: exact across several samplings
  }
  return B200DQN_OK;
}

extern "C" int b200dqn_net_read_costs(b200dqn_net* n, int count, float* host_costs, void* stream) {
  B2_REQUIRE(n && host_costs && count >= 1 && count <= kCostRing, B200DQN_EINVAL, "net_read_costs: bad argument");
  DeviceGuard g(n->device);
  cudaStream_t st = as_stream(stream);
  float* ring = reinterpret_cast<float*>(n->h_pin);
  uint32_t step = 0;
  // the pinned block is reused: wait for anything in flight first
  B2_CHECK_CUDA(cudaStreamSynchronize(st));
  B2_CHECK_CUDA(cudaMemcpyAsync(ring, n->d_cost, (kCostRing + 2) * sizeof(float), cudaMemcpyDeviceToHost, st));
  B2_CHECK_CUDA(cudaMemcpyAsync(&step, n->d_step, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  B2_CHECK_CUDA(cudaStreamSynchronize(st));
  B2_REQUIRE(reinterpret_cast<uint32_t*>(ring)[kCostRing + 1] == 0, B200DQN_EINVAL,
             "train: a sampled action is >= num_actions %d (IndexError at deepqnetwork.py:141 in the reference)", n->A);
  B2_REQUIRE(uint32_t(count) <= step, B200DQN_ESTATE, "net_read_costs: only %u steps have run", step);
  for (int i = 0; i < count; ++i) host_costs[i] = ring[(step - count + i) % kCostRing];
  return B200DQN_OK;
}

extern "C" int b200dqn_net_train_iterations(const b200dqn_net* n, int64_t* iters) {
  B2_REQUIRE(n && iters, B200DQN_EINVAL, "null argument");
  *iters = n->train_iterations;
  return B200DQN_OK;
}

extern "C" int b200dqn_net_device_ptr(b200dqn_net* n, int which, void** dev_ptr, size_t* bytes) {
  B2_REQUIRE(n && dev_ptr, B200DQN_EINVAL, "net_device_ptr: null argument");
  void* p = nullptr;
  size_t b = 0;
  switch (which) {
    case B200DQN_NET_PTR_Q_ONLINE: p = n->d_q[0]; b = size_t(n->nb) * n->A * 4; break;
    case B200DQN_NET_PTR_Q_TARGET: p = n->d_q[1]; b = size_t(n->nb) * n->A * 4; break;
    case B200DQN_NET_PTR_DELTAS:
      B2_REQUIRE(!n->atoms, B200DQN_EINVAL, "net_device_ptr: a distributional head has no scalar delta");
      B2_REQUIRE(!n->quantiles, B200DQN_EINVAL, "net_device_ptr: a quantile-regression head has no scalar delta");
      B2_REQUIRE(!n->iqn_n, B200DQN_EINVAL, "net_device_ptr: an IQN head has no scalar delta");
      B2_REQUIRE(!n->boot, B200DQN_EINVAL, "net_device_ptr: bootstrapped heads have no scalar delta per action");
      B2_REQUIRE(!n->rem_k, B200DQN_EINVAL, "net_device_ptr: a REM head has no scalar delta per action");
      p = n->d_delta;
      b = size_t(n->nb) * n->A * 4;
      break;
    case B200DQN_NET_PTR_GRADS: p = n->d_g; b = n->n_params * 4; break;
    case B200DQN_NET_PTR_WEIGHTS: p = n->d_w; b = n->n_params * 4; break;
    case B200DQN_NET_PTR_COST: p = n->d_cost; b = kCostRing * 4; break;
    case B200DQN_NET_PTR_H1: p = n->d_h1[0]; b = size_t(n->nb) * kP1 * kP1 * kC1 * 4; break;
    case B200DQN_NET_PTR_H2: p = n->d_h2[0]; b = size_t(n->nb) * kP2 * kP2 * kC2 * 4; break;
    case B200DQN_NET_PTR_H3: p = n->d_h3[0]; b = size_t(n->nb) * kFlat * 4; break;
    case B200DQN_NET_PTR_H4: p = n->d_h4[0]; b = size_t(n->iqn_n ? n->iqn_rows : n->nb) * n->hidden * 4; break;
    case B200DQN_NET_PTR_DZ4: p = n->d_dz4; b = size_t(n->iqn_n ? n->iqn_rows : n->nb) * n->hidden * 4; break;
    case B200DQN_NET_PTR_DZ3: p = n->d_dz3; b = size_t(n->nb) * kFlat * 4; break;
    case B200DQN_NET_PTR_DZ2: p = n->d_dz2; b = size_t(n->nb) * kP2 * kP2 * kC2 * 4; break;
    case B200DQN_NET_PTR_DZ1: p = n->d_dz1; b = size_t(n->nb) * kP1 * kP1 * kC1 * 4; break;
    case B200DQN_NET_PTR_Q_ONLINE_POST:   // target_steps = 0: the target forward is the online one (train_step)
      p = n->d_tw == n->d_w ? n->d_q[1] : n->d_q[2];
      b = size_t(n->nb) * n->A * 4;
      break;
    case B200DQN_NET_PTR_TD_ERRORS:
      B2_REQUIRE(n->d_td_err, B200DQN_EINVAL, "net_device_ptr: no train step on a prioritized ring has run");
      p = n->d_td_err;
      b = size_t(n->nb) * 4;
      break;
    case B200DQN_NET_PTR_ROW_COSTS: p = n->d_rowcost; b = size_t(n->nb) * 4; break;
    case B200DQN_NET_PTR_LOGITS:
    case B200DQN_NET_PTR_PROBS:
    case B200DQN_NET_PTR_TARGET_DIST:
    case B200DQN_NET_PTR_LOGIT_GRADS:
      B2_REQUIRE(n->atoms, B200DQN_EINVAL, "net_device_ptr: selector %d needs a distributional head", which);
      p = which == B200DQN_NET_PTR_LOGITS ? n->d_logits : which == B200DQN_NET_PTR_PROBS ? n->d_probs
        : which == B200DQN_NET_PTR_TARGET_DIST ? n->d_tdist : n->d_lgrad;
      b = (which <= B200DQN_NET_PTR_PROBS ? size_t(3) * n->nb * n->A : size_t(n->nb)) * n->atoms * 4;
      break;
    case B200DQN_NET_PTR_DZ4_PLANES: {
      __half* hi = nullptr;
      int64_t lo_off = 0;
      umma_dz4_planes(n, &hi, &lo_off);
      B2_REQUIRE(n->cfg.math_mode == B200DQN_MATH_TCGEN05 && hi, B200DQN_EINVAL,
                 "net_device_ptr: the dZ4 planes exist on the tensor-core engine only");
      p = hi;
      b = size_t(lo_off + int64_t(n->nb) * n->hidden) * 2;
      break;
    }
    case B200DQN_NET_PTR_DUELING_VA:
      B2_REQUIRE(n->dueling, B200DQN_EINVAL, "net_device_ptr: selector %d needs a dueling net", which);
      p = n->d_va;
      b = size_t(3) * n->nb * (n->A + 1) * 4;
      break;
    case B200DQN_NET_PTR_QUANTILES:
    case B200DQN_NET_PTR_TARGET_QUANTILES:
    case B200DQN_NET_PTR_QUANTILE_GRADS:
      B2_REQUIRE(n->quantiles, B200DQN_EINVAL, "net_device_ptr: selector %d needs a quantile-regression head", which);
      p = which == B200DQN_NET_PTR_QUANTILES ? n->d_theta : which == B200DQN_NET_PTR_TARGET_QUANTILES ? n->d_tquant
                                                                                                       : n->d_qgrad;
      b = (which == B200DQN_NET_PTR_QUANTILES ? size_t(3) * n->nb * n->A : size_t(n->nb)) * n->quantiles * 4;
      break;
    case B200DQN_NET_PTR_Q_TARGET_PRE:
    case B200DQN_NET_PTR_TD_TARGETS:
      B2_REQUIRE(n->munchausen, B200DQN_EINVAL, "net_device_ptr: selector %d needs the Munchausen target", which);
      if (which == B200DQN_NET_PTR_TD_TARGETS) {
        p = n->d_tdtarget;
        b = size_t(n->nb) * 4;
      } else {   // target_steps = 0: the target network is the online one, and so is its Q row of the prestates
        p = n->d_tw == n->d_w ? n->d_q[0] : n->d_q[2];
        b = size_t(n->nb) * n->A * 4;
      }
      break;
    case B200DQN_NET_PTR_IQN_TAUS:
    case B200DQN_NET_PTR_IQN_COS:
    case B200DQN_NET_PTR_IQN_PHI:
    case B200DQN_NET_PTR_IQN_X:
    case B200DQN_NET_PTR_IQN_QUANTILES:
    case B200DQN_NET_PTR_IQN_TARGET_QUANTILES:
    case B200DQN_NET_PTR_IQN_QUANTILE_GRADS:
    case B200DQN_NET_PTR_IQN_DX:
    case B200DQN_NET_PTR_IQN_DPHI:
    case B200DQN_NET_PTR_IQN_TAU_COUNTER: {
      B2_REQUIRE(n->iqn_n, B200DQN_EINVAL, "net_device_ptr: selector %d needs an IQN head", which);
      B2_REQUIRE(!(n->fqf_n && which == B200DQN_NET_PTR_IQN_TAU_COUNTER), B200DQN_EINVAL,
                 "net_device_ptr: the FQF head draws nothing and has no counter");
      const size_t R = size_t(n->iqn_rows), nbn = size_t(n->nb) * n->iqn_n;
      switch (which) {
        case B200DQN_NET_PTR_IQN_TAUS: p = n->d_tau; b = 2 * R * 4; break;
        case B200DQN_NET_PTR_IQN_COS: p = n->d_cos; b = 2 * R * kIqnCos * 4; break;
        case B200DQN_NET_PTR_IQN_PHI: p = n->d_phi; b = 2 * R * kFlat * 4; break;
        case B200DQN_NET_PTR_IQN_X: p = n->d_x; b = 2 * R * kFlat * 4; break;
        case B200DQN_NET_PTR_IQN_QUANTILES: p = n->d_iqn_theta; b = 2 * R * n->A * 4; break;
        case B200DQN_NET_PTR_IQN_TARGET_QUANTILES: p = n->d_iqn_tq; b = nbn * 4; break;
        case B200DQN_NET_PTR_IQN_QUANTILE_GRADS: p = n->d_iqn_qgrad; b = nbn * 4; break;
        case B200DQN_NET_PTR_IQN_DX: p = n->d_dx; b = R * kFlat * 4; break;
        case B200DQN_NET_PTR_IQN_DPHI: p = n->d_dphi; b = R * kFlat * 4; break;
        default: p = n->d_tau_ctr; b = sizeof(unsigned long long); break;
      }
      break;
    }
    case B200DQN_NET_PTR_SHIFT_OFFSETS:
    case B200DQN_NET_PTR_SHIFT_DRAWS:
      B2_REQUIRE(n->crop_pad, B200DQN_EINVAL, "net_device_ptr: selector %d needs random_shift > 0", which);
      if (which == B200DQN_NET_PTR_SHIFT_OFFSETS) {
        p = n->d_crop;
        b = size_t(n->nb) * 4 * sizeof(int32_t);
      } else {
        p = n->d_crop_ctr;
        b = sizeof(unsigned long long);
      }
      break;
    case B200DQN_NET_PTR_REM_HEADS:
    case B200DQN_NET_PTR_REM_ALPHAS:
    case B200DQN_NET_PTR_REM_GRADS:
    case B200DQN_NET_PTR_REM_COUNTER:
      B2_REQUIRE(n->rem_k, B200DQN_EINVAL, "net_device_ptr: selector %d needs a REM head", which);
      B2_REQUIRE(!n->boot || which == B200DQN_NET_PTR_REM_HEADS || which == B200DQN_NET_PTR_REM_GRADS, B200DQN_EINVAL,
                 "net_device_ptr: bootstrapped heads draw no REM mixture (selector %d)", which);
      switch (which) {
        case B200DQN_NET_PTR_REM_HEADS: p = n->d_theta; b = size_t(3) * n->nb * n->A * n->rem_k * 4; break;
        case B200DQN_NET_PTR_REM_ALPHAS: p = n->d_rem_alpha; b = size_t(n->rem_k) * 4; break;
        case B200DQN_NET_PTR_REM_GRADS: p = n->d_rem_grad; b = size_t(n->nb) * n->rem_k * 4; break;
        default: p = n->d_rem_ctr; b = sizeof(unsigned long long); break;
      }
      break;
    case B200DQN_NET_PTR_FQF_LOGITS:
    case B200DQN_NET_PTR_FQF_PROBS:
    case B200DQN_NET_PTR_FQF_FRACTIONS:
    case B200DQN_NET_PTR_FQF_BOUNDARY_QUANTILES:
    case B200DQN_NET_PTR_FQF_FRACTION_GRADS:
    case B200DQN_NET_PTR_FQF_LOGIT_GRADS: {
      B2_REQUIRE(n->fqf_n, B200DQN_EINVAL, "net_device_ptr: selector %d needs an FQF head", which);
      const size_t nb = size_t(n->nb), N = size_t(n->fqf_n);
      switch (which) {
        case B200DQN_NET_PTR_FQF_LOGITS: p = n->d_fl; b = nb * N * 4; break;
        case B200DQN_NET_PTR_FQF_PROBS: p = n->d_fq; b = nb * N * 4; break;
        case B200DQN_NET_PTR_FQF_FRACTIONS: p = n->d_ftau; b = nb * (N + 1) * 4; break;
        case B200DQN_NET_PTR_FQF_BOUNDARY_QUANTILES: p = n->d_btheta; b = nb * (N - 1) * n->A * 4; break;
        case B200DQN_NET_PTR_FQF_FRACTION_GRADS: p = n->d_fg; b = nb * (N - 1) * 4; break;
        default: p = n->d_fdl; b = nb * N * 4; break;
      }
      break;
    }
    case B200DQN_NET_PTR_BOOT_MASKS:
    case B200DQN_NET_PTR_BOOT_TARGETS:
    case B200DQN_NET_PTR_BOOT_DELTAS:
    case B200DQN_NET_PTR_BOOT_ACTIVE_HEAD: {
      B2_REQUIRE(n->boot, B200DQN_EINVAL, "net_device_ptr: selector %d needs bootstrapped heads", which);
      const size_t nk = size_t(n->nb) * n->rem_k;
      switch (which) {
        case B200DQN_NET_PTR_BOOT_MASKS: p = n->d_boot_mask; b = nk; break;
        case B200DQN_NET_PTR_BOOT_TARGETS: p = n->d_boot_y; b = nk * 4; break;
        case B200DQN_NET_PTR_BOOT_DELTAS: p = n->d_boot_delta; b = nk * 4; break;
        default: p = n->d_boot_head; b = sizeof(int32_t); break;
      }
      break;
    }
    case B200DQN_NET_PTR_GRAD_SQ:
    case B200DQN_NET_PTR_GRAD_NORM:
    case B200DQN_NET_PTR_CLIP_SCALE:
      B2_REQUIRE(n->clip, B200DQN_EINVAL, "net_device_ptr: selector %d needs gradient-norm clipping", which);
      switch (which) {
        case B200DQN_NET_PTR_GRAD_SQ: p = n->d_clip; b = 6 * sizeof(double); break;
        case B200DQN_NET_PTR_GRAD_NORM: p = n->d_clip + 6; b = sizeof(double); break;
        default: p = n->d_clip_c(); b = sizeof(float); break;
      }
      break;
    default: B2_REQUIRE(false, B200DQN_EINVAL, "net_device_ptr: unknown selector %d", which);
  }
  *dev_ptr = p;
  if (bytes) *bytes = b;
  return B200DQN_OK;
}

extern "C" int b200dqn_net_set_keep_grads(b200dqn_net* n, int keep) {
  B2_REQUIRE(n, B200DQN_EINVAL, "null net");
  n->keep_grads = keep != 0;
  destroy_step_graphs(n);   // parameters are baked in
  return B200DQN_OK;
}

// Buffers of the third network slot, made the first time Double DQN is switched on: the fc1 split-K partials grow to
// three slots, the SIMT engine gets fp32 activations for slot 2 and the tensor-core engine fp16 planes.
static int double_q_alloc(b200dqn_net* n) {
  if (n->double_q_alloc) return B200DQN_OK;
  DeviceGuard g(n->device);
  B2_CHECK_CUDA(cudaDeviceSynchronize());   // no step or predict in flight still reads the old partial buffer
  const size_t nb = size_t(n->nb);
  float* part = nullptr;
  B2_CHECK_CUDA(cudaMalloc(&part, size_t(3) * kFc1Splits * nb * n->hidden * sizeof(float)));
  B2_CHECK_CUDA(cudaMemset(part, 0, size_t(3) * kFc1Splits * nb * n->hidden * sizeof(float)));
  cudaFree(n->d_fc1part);
  n->d_fc1part = part;
  n->graph_predict.drop();
  if (n->cfg.math_mode == B200DQN_MATH_TCGEN05) {
    int rc = umma_double_q_alloc(n);
    if (rc) return rc;
  } else {
    const size_t elems[3] = {nb * kP1 * kP1 * kC1, nb * kP2 * kP2 * kC2, nb * kFlat};
    float** dst[3] = {&n->d_h1[2], &n->d_h2[2], &n->d_h3[2]};
    for (int i = 0; i < 3; ++i) {
      B2_CHECK_CUDA(cudaMalloc(dst[i], elems[i] * sizeof(float)));
      B2_CHECK_CUDA(cudaMemset(*dst[i], 0, elems[i] * sizeof(float)));
    }
  }
  n->double_q_alloc = true;
  return B200DQN_OK;
}

extern "C" int b200dqn_net_set_double_q(b200dqn_net* n, int on) {
  B2_REQUIRE(n, B200DQN_EINVAL, "null net");
  if (on) {
    B2_REQUIRE(!n->munchausen, B200DQN_EINVAL,
               "net_set_double_q: the Munchausen target makes no greedy choice for Double DQN to change");
    B2_REQUIRE(!n->fqf_n, B200DQN_ENOTIMPL, "net_set_double_q: the Double DQN target with the FQF head is not implemented");
    B2_REQUIRE(!n->iqn_n, B200DQN_ENOTIMPL, "net_set_double_q: the Double DQN target with the IQN head is not implemented");
    B2_REQUIRE(!n->nccl_comm, B200DQN_ENOTIMPL,
               "net_set_double_q: the Double DQN target is implemented for a single learner only (comm_init has run)");
    B2_TRY(double_q_alloc(n));
  }
  n->double_q = on != 0;
  destroy_step_graphs(n);   // the number of network slots is baked in
  return B200DQN_OK;
}

extern "C" int b200dqn_net_set_active_head(b200dqn_net* n, int h, void* stream) {
  B2_REQUIRE(n, B200DQN_EINVAL, "null net");
  B2_REQUIRE(n->boot, B200DQN_EINVAL, "net_set_active_head: the net has no bootstrapped heads");
  B2_REQUIRE(h >= -1 && h < n->rem_k, B200DQN_EINVAL, "net_set_active_head: head %d not in [-1,%d]", h, n->rem_k - 1);
  DeviceGuard g(n->device);
  k_boot_set_head<<<1, 1, 0, as_stream(stream)>>>(n->d_boot_head, h);
  B2_LAUNCH_CHECK();
  return B200DQN_OK;
}

extern "C" int b200dqn_net_get_grads(b200dqn_net* n, int layer, float* host_dW, void* stream) {
  B2_REQUIRE(n && host_dW && layer_ok(n, layer), B200DQN_EINVAL, "net_get_grads: bad argument");
  DeviceGuard g(n->device);
  cudaStream_t st = as_stream(stream);
  if (layer == kLayers + 1) return xfer_wf(n, n->d_wfg, host_dW, false, st);   // written whole by k_fqf_wf
  if (layer == kLayers) return xfer_we(n, n->d_weg, host_dW, false, st);   // written whole by k_iqn_we
  const int64_t n4 = n->n_params / 4;
  if (n->world == 1) {  // partials of the last step are still in scratch; sum them into d_g
    // a distributional or quantile fc2 is summed by its own kernel
    const int64_t e4 = n->fc2_block() ? n->lt.off[4] / 4 : n4;
    k_optimizer<<<cdiv(e4, 256), 256, 0, st>>>(n->lt, n->d_part, n->d_g, n->d_w, n->d_s, 0, e4, 1 | 2, OptArgs{},
                                               KTrace{nullptr, 0});
    B2_LAUNCH_CHECK();
    if (n->fc2_block()) {
      NoPdlScope plain;
      B2_TRY(opt_fc2_dist(n, n->nb, 2, st, "grads_fc2_dist"));
    }
  } else if (n->xchg_ok && n->xchg_sched == 2 && n->d_xbuf && layer == 3) {
    // gather schedule: fc1's global gradient was computed locally and never passed through d_g
    const int64_t b4 = n->lt.off[3] / 4, e4 = n->lt.off[4] / 4;
    k_optimizer<<<cdiv(e4 - b4, 256), 256, 0, st>>>(n->lt, n->d_part, n->d_g, n->d_w, n->d_s, b4, e4, 1 | 2, OptArgs{},
                                                    KTrace{nullptr, 0});
    B2_LAUNCH_CHECK();
  }
  return xfer_params(n, n->d_g, layer, host_dW, false, st);
}

extern "C" int b200dqn_net_launches_per_step(const b200dqn_net* n, int* launches) {
  B2_REQUIRE(n && launches, B200DQN_EINVAL, "null argument");
  // Counted at the launch sites while the step was captured into its CUDA graph; before the first
  // fused step: the static schedule (sample, 4 forward, head, 7 backward GEMMs, per-layer optimizers).
  if (n->graph_launches > 0) {
    *launches = n->graph_launches;
  } else {
    const bool tc = n->cfg.math_mode == B200DQN_MATH_TCGEN05;
    // a distributional or quantile head adds k_fc2_dist, and on the SIMT engine fc2's own update; the Munchausen
    // target with a separate target network repeats the forward's launches for its pass
    // an IQN head adds the tau draw, the embedding, the modulation, its backward and the embedding's gradient;
    // random-shift augmentation and the REM head add their draws (bootstrapped heads draw nothing); an FQF head replaces the tau draw by the fraction
    // proposal and adds the boundary pass (phi, the modulation, fc1 and fc2) and the fraction layer's gradient
    // a soft target update adds one blend per update launch: conv1, conv2, conv3, fc1 (with the SIMT engine's scalar
    // fc2), fc2 where it is updated on its own, the embedding and the fraction layer
    *launches = 1 + 4 + 1 + 7 + (n->world > 1 ? (tc ? 7 : 2) : (tc ? 6 : 4)) + (n->fc2_block() ? (tc ? 1 : 2) : 0) +
                (n->munchausen && n->d_tw != n->d_w ? 4 : 0) + (n->iqn_n ? 5 : 0) + (n->fqf_n ? 5 : 0) +
                (n->crop_pad ? 1 : 0) +
                (n->rem_k && !n->boot ? 1 : 0) +
                (tc && n->lt.splits[3] > 1 ? n->lt.splits[3] : 0) +   // IQN: the chunked fc1 wgrad and its reduction
                (n->soft ? 4 + (tc || n->fc2_block() ? 1 : 0) + (n->iqn_n ? 1 : 0) + (n->fqf_n ? 1 : 0) : 0) +
                // gradient-norm clipping: a reduce per layer whose update read partials (not the tensor-core fc1's
                // single partial), a sum of squares per layer, clip_scale, and one update launch per layer in place
                // of the per-branch ones (tensor-core conv layers: plus their 5 image packs); the embedding adds its
                // sum of squares and its update
                (n->clip ? (tc ? 15 : n->fc2_block() ? 11 : 12) + (n->iqn_n ? 2 : 0) : 0);
  }
  return B200DQN_OK;
}
