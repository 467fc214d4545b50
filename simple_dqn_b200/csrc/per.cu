// per.cu — proportional prioritized experience replay on the device ring (Schaul et al., 2016; the variant of OpenAI
// baselines' PrioritizedReplayBuffer): a 32-ary fp64 sum tree and min tree over the ring, the stratified tree-descent
// sampler, the importance weights and the priority update after a train step.
//
// The tree is a pure function of its leaves: a node is always recomputed from its 32 children by the same fixed-order
// warp reduction (xor butterfly 16, 8, 4, 2, 1), never updated by adding a delta, and nothing uses atomics.  Leaf i is
// the stored priority of slot i if getMinibatch would accept i as an index (src/replay_memory.py:59-65), else 0, so a
// draw never retries.  All fp64 arithmetic uses the _rn intrinsics: no contraction, so tests/per_oracle.py restates
// every node and every draw bit for bit.
#include <math.h>

#include <new>

#include "replay.cuh"

namespace b200 {

struct PerView {
  double* prio;
  double* sum;
  double* mn;                 // min levels 1..: node j of level l at mn[off[l] - off[1] + j]
  const uint8_t* terminals;
  const int64_t* cursor;      // {count, current}
  int64_t off[b200dqn_replay::kPerMaxLevels + 1];
  int64_t n[b200dqn_replay::kPerMaxLevels];
  int nlev, hist, nstep;
  int64_t size;
};

static PerView per_view(const b200dqn_replay* r) {
  PerView v{};
  v.prio = r->d_prio; v.sum = r->d_sum; v.mn = r->d_min;
  v.terminals = r->d_terminals; v.cursor = r->d_cursor;
  for (int l = 0; l <= b200dqn_replay::kPerMaxLevels; ++l) v.off[l] = r->per_off[l];
  for (int l = 0; l < b200dqn_replay::kPerMaxLevels; ++l) v.n[l] = r->per_n[l];
  v.nlev = r->per_nlev; v.hist = r->hist; v.nstep = r->nstep; v.size = r->size;
  return v;
}

// the acceptance test of getMinibatch (src/replay_memory.py:59-65) for slot i, with the window of n-step returns
// [i - hist, i + nstep - 1] (sample_block)
__device__ __forceinline__ bool per_valid(const PerView& v, int64_t i, int64_t count, int64_t current) {
  if (i < v.hist || i > count - v.nstep) return false;
  if (i + v.nstep - 1 >= current && i - v.hist < current) return false;
  unsigned any = 0;
  for (int j = 1; j <= v.hist; ++j) any |= v.terminals[i - j];
  return any == 0;
}

__device__ __forceinline__ void per_set_leaf(const PerView& v, int64_t i, int64_t count, int64_t current) {
  v.sum[i] = per_valid(v, i, count, current) ? v.prio[i] : 0.0;
}

// one warp: node j of level l >= 1 from its 32 children
__device__ __forceinline__ void per_node(const PerView& v, int l, int64_t j, int lane) {
  const int64_t c = j * 32 + lane;
  double s = 0.0, m = __longlong_as_double(0x7ff0000000000000ll);   // +inf
  if (c < v.n[l - 1]) {
    s = v.sum[v.off[l - 1] + c];
    m = l == 1 ? (s > 0.0 ? s : m) : v.mn[v.off[l - 1] - v.off[1] + c];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s = __dadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
    m = fmin(m, __shfl_xor_sync(0xffffffffu, m, o));
  }
  if (lane == 0) {
    v.sum[v.off[l] + j] = s;
    v.mn[v.off[l] - v.off[1] + j] = m;
  }
}

// beta = beta0 + (1 - beta0) * min(1, k / beta_steps), k = samplings done
__device__ __forceinline__ double per_beta(uint32_t k, double beta0, double beta_steps) {
  const double frac = beta_steps > 0.0 ? fmin(1.0, __ddiv_rn(double(k), beta_steps)) : 1.0;
  return __dadd_rn(beta0, __dmul_rn(__dsub_rn(1.0, beta0), frac));
}

// w = (N P)^-beta / (N P_min)^-beta with P = leaf / total, P_min = min / total (baselines), rounded once to fp32
__device__ __forceinline__ float per_weight(double leaf, double total, double minv, double count, double beta) {
  const double num = pow(__dmul_rn(count, __ddiv_rn(leaf, total)), -beta);
  const double den = pow(__dmul_rn(count, __ddiv_rn(minv, total)), -beta);
  return static_cast<float>(__ddiv_rn(num, den));
}

// ------------------------------------------------------------------------------------------ tree maintenance
__global__ void k_per_fill(double* prio, const double* maxp, double alpha, int64_t from, int64_t n, int64_t size) {
  const int64_t t = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
  if (t < n) prio[(from + t) % size] = pow(*maxp, alpha);
}

__global__ void k_per_init(double* prio, double* maxp, int64_t size) {
  const int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
  if (i < size) prio[i] = 1.0;
  if (i == 0) *maxp = 1.0;
}

__global__ void k_per_leaves(const PerView v) {
  const int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
  if (i < v.size) per_set_leaf(v, i, v.cursor[0], v.cursor[1]);
}

__global__ void k_per_level(const PerView v, int l) {
  const int64_t j = (blockIdx.x * int64_t(blockDim.x) + threadIdx.x) >> 5;
  if (j < v.n[l]) per_node(v, l, j, threadIdx.x & 31);
}

// A flush of n deferred add()s at pos0: those slots get max_priority^alpha, and the leaves of
// [pos0 - (nstep - 1), pos0 + n + hist) (mod size) are re-derived: the written slots, the slots whose window
// [i - hist, i + nstep - 1] held the old write pointer or holds the new one, and the slots that became drawable as
// count grew past i + nstep - 1.  No other slot's acceptance can change.  Then their ancestors, level by level.  One
// CTA.
constexpr int kPerAddThreads = 256;
__global__ void __launch_bounds__(kPerAddThreads) k_per_add(const PerView v, const double* maxp, double alpha,
                                                            int64_t pos0, int n) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t touched = min(int64_t(n) + v.hist + v.nstep - 1, v.size);
  const int64_t first = pos0 - (v.nstep - 1) + v.size;   // + size: the leaves before pos0 may lie across the wrap
  const int64_t count = v.cursor[0], current = v.cursor[1];
  const double p = pow(*maxp, alpha);
  for (int t = tid; t < n; t += kPerAddThreads) v.prio[(pos0 + t) % v.size] = p;
  __syncthreads();
  for (int64_t t = tid; t < touched; t += kPerAddThreads) per_set_leaf(v, (first + t) % v.size, count, current);
  __syncthreads();
  for (int l = 1; l < v.nlev; ++l) {
    for (int64_t t = warp; t < touched; t += kPerAddThreads / 32) per_node(v, l, ((first + t) % v.size) >> (5 * l), lane);
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------ sampler
// Stratified proportional draw: sample i takes mass = random.random() * (total/batch) + i * (total/batch) and descends
// from the root.  random.random() is CPython's: two MT19937 words, ((w0 >> 5) * 2^26 + (w1 >> 6)) / 2^53, so a draw
// consumes exactly 2 * batch words and the words-consumed channel keeps the host stream in lock-step unchanged.
// One warp per sample (one 256-byte read and one warp scan per level); kPerWarps samples per CTA.  Every CTA reads
// the same state slot and runs the stream forward to its own words; the CTA with the last samples leaves the
// advanced state in the other slot, and the last CTA to arrive (ticket) advances the counters.
constexpr int kPerWarps = 8;
__global__ void __launch_bounds__(kPerWarps * 32)
k_sample_per(const PerView v, uint32_t* __restrict__ mt_state, int batch, int32_t* __restrict__ idx_out,
             float* __restrict__ isw, uint32_t* __restrict__ words, uint32_t* __restrict__ ticket, double beta0,
             double beta_steps, const KTrace kt) {
  __shared__ uint32_t mt[kMtN + 1];
  __shared__ uint32_t w[2 * kPerWarps];
  constexpr int kThreads = kPerWarps * 32;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  kt_begin(kt);
  pdl_wait();
  pdl_launch_dependents();
  const uint32_t k = words[2];
  const uint32_t* cur = mt_state + (k & 1u) * kMtSlot;
  for (int i = tid; i < kMtN + 1; i += kThreads) mt[i] = cur[i];
  __syncthreads();
  if (tid == 0) {   // every CTA has read k and the state: the last one to get here may advance the counters
    __threadfence();
    if (atomicInc(ticket, gridDim.x - 1) == gridDim.x - 1) {
      words[0] = 2u * batch;
      words[1] += 2u * batch;
      words[2] = k + 1;
    }
  }
  const int s0 = blockIdx.x * kPerWarps;
  const int ns = min(kPerWarps, batch - s0);
  int pos = static_cast<int>(mt[kMtN]);
  int skip = 2 * s0, got = 0;
  while (got < 2 * ns) {
    if (pos >= kMtN) {
      __syncthreads();
      mt_regenerate(mt, tid, kThreads);
      pos = 0;
    }
    if (skip > 0) {
      const int adv = min(skip, kMtN - pos);
      pos += adv;
      skip -= adv;
      continue;
    }
    const int take = min(2 * ns - got, kMtN - pos);
    if (tid < take) w[got + tid] = mt_temper(mt[pos + tid]);
    pos += take;
    got += take;
  }
  __syncthreads();
  if (blockIdx.x == gridDim.x - 1) {
    uint32_t* nxt = mt_state + ((k + 1u) & 1u) * kMtSlot;
    for (int i = tid; i < kMtN; i += kThreads) nxt[i] = mt[i];
    if (tid == 0) nxt[kMtN] = static_cast<uint32_t>(pos);
  }
  if (warp < ns) {
    const int s = s0 + warp;
    const int top = v.nlev - 1;
    const double total = v.sum[v.off[top]];
    if (!(total > 0.0)) {   // no drawable slot: sticky error, a harmless index, zero weight (the reference would spin)
      if (lane == 0) {
        words[3] = 1u;
        idx_out[s] = v.hist;
        isw[s] = 0.f;
      }
    } else {
      const double seg = __ddiv_rn(total, double(batch));
      const double a = double(w[2 * warp] >> 5), b = double(w[2 * warp + 1] >> 6);
      const double rnd = __dmul_rn(__dadd_rn(__dmul_rn(a, 67108864.0), b), 1.0 / 9007199254740992.0);
      double mass = __dadd_rn(__dmul_rn(rnd, seg), __dmul_rn(double(s), seg));
      int64_t node = 0;
      double leaf = 0.0;
      for (int l = top - 1; l >= 0; --l) {
        const double x = v.sum[v.off[l] + node * 32 + lane];   // the padding of a level is zero
        double incl = x;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const double up = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl = __dadd_rn(incl, up);
        }
        const unsigned gt = __ballot_sync(0xffffffffu, incl > mass);
        int pick;
        if (gt) {
          pick = __ffs(gt) - 1;
        } else {   // rounding left no prefix above the mass: the last child with a positive sum
          const unsigned pz = __ballot_sync(0xffffffffu, x > 0.0);
          pick = pz ? 31 - __clz(pz) : 0;
        }
        const double before = __shfl_sync(0xffffffffu, incl, pick > 0 ? pick - 1 : 0);
        leaf = __shfl_sync(0xffffffffu, x, pick);
        if (pick > 0) mass = __dsub_rn(mass, before);
        node = node * 32 + pick;
      }
      if (lane == 0) {
        const double minv = v.mn[v.off[top] - v.off[1]];
        idx_out[s] = static_cast<int32_t>(node);
        isw[s] = per_weight(leaf, total, minv, double(v.cursor[0]), per_beta(k, beta0, beta_steps));
      }
    }
  }
  kt_end(kt);
}

// importance weights of caller-chosen indexes (set_indexes), from their stored priorities, at the current beta
__global__ void k_per_weights(const PerView v, const int32_t* __restrict__ idx, int batch, float* __restrict__ isw,
                              const uint32_t* __restrict__ words, double beta0, double beta_steps) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= batch) return;
  const int top = v.nlev - 1;
  isw[i] = per_weight(v.prio[idx[i]], v.sum[v.off[top]], v.mn[v.off[top] - v.off[1]], double(v.cursor[0]),
                      per_beta(words[2], beta0, beta_steps));
}

// ------------------------------------------------------------------------------------------ priority update
// After the head: slot idx[b] gets (|delta_b| + eps)^alpha, the last occurrence winning when a slot is in the
// minibatch twice (baselines' sequential update_priorities); max_priority = max(max_priority, |delta_b| + eps); then
// the ancestors of the written leaves, level by level.  One CTA: it runs on a side branch of the step.
constexpr int kPerUpdThreads = 1024, kPerUpdMaxRows = 4096;
__global__ void __launch_bounds__(kPerUpdThreads)
k_per_update(const PerView v, const int32_t* __restrict__ idx, const float* __restrict__ td_err, int rows,
             double alpha, double eps, double* maxp, const KTrace kt) {
  __shared__ int32_t s_idx[kPerUpdMaxRows];
  __shared__ double s_max[kPerUpdThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  kt_begin(kt);
  pdl_wait();
  const int64_t count = v.cursor[0], current = v.cursor[1];
  for (int b = tid; b < rows; b += kPerUpdThreads) s_idx[b] = idx[b];
  __syncthreads();
  double mx = 0.0;
  for (int b = tid; b < rows; b += kPerUpdThreads) {
    const int32_t slot = s_idx[b];
    bool last = true;
    for (int b2 = b + 1; b2 < rows && last; ++b2) last = s_idx[b2] != slot;
    const double a = __dadd_rn(fabs(double(td_err[b])), eps);
    mx = fmax(mx, a);
    if (last) {
      const double p = pow(a, alpha);
      v.prio[slot] = p;
      v.sum[slot] = per_valid(v, slot, count, current) ? p : 0.0;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (lane == 0) s_max[warp] = mx;
  __syncthreads();
  if (tid == 0) {
    double m = *maxp;
    for (int i = 0; i < kPerUpdThreads / 32; ++i) m = fmax(m, s_max[i]);
    *maxp = m;
  }
  for (int l = 1; l < v.nlev; ++l) {
    for (int b = warp; b < rows; b += kPerUpdThreads / 32) per_node(v, l, int64_t(s_idx[b]) >> (5 * l), lane);
    __syncthreads();
  }
  kt_end(kt);
}

// ------------------------------------------------------------------------------------------ host side
static inline unsigned cdiv64(int64_t a, int64_t b) { return unsigned((a + b - 1) / b); }

int per_rebuild(b200dqn_replay* r, int64_t fill_from, int64_t fill_n, bool init, cudaStream_t st) {
  const PerView v = per_view(r);
  if (init) {
    k_per_init<<<cdiv64(r->size, 256), 256, 0, st>>>(r->d_prio, r->d_maxp, r->size);
    B2_LAUNCH_CHECK();
  }
  if (fill_n > 0) {
    const int64_t n = fill_n < r->size ? fill_n : r->size;
    k_per_fill<<<cdiv64(n, 256), 256, 0, st>>>(r->d_prio, r->d_maxp, r->per_alpha, fill_from, n, r->size);
    B2_LAUNCH_CHECK();
  }
  k_per_leaves<<<cdiv64(r->size, 256), 256, 0, st>>>(v);
  B2_LAUNCH_CHECK();
  for (int l = 1; l < r->per_nlev; ++l) {
    k_per_level<<<cdiv64(r->per_n[l] * 32, 256), 256, 0, st>>>(v, l);
    B2_LAUNCH_CHECK();
  }
  return B200DQN_OK;
}

int per_after_add(b200dqn_replay* r, int64_t pos0, int64_t n, cudaStream_t st) {
  k_per_add<<<1, kPerAddThreads, 0, st>>>(per_view(r), r->d_maxp, r->per_alpha, pos0, int(n));
  B2_LAUNCH_CHECK();
  return B200DQN_OK;
}

int launch_sample_per(b200dqn_replay* r, cudaStream_t st) {
  B2_CHECK_CUDA(launch_pdl(k_sample_per, dim3(cdiv64(r->batch, kPerWarps)), dim3(kPerWarps * 32), 0, st, per_view(r),
                           r->d_mt, r->batch, r->d_idx, r->d_isw, r->d_words, r->d_per_ticket, r->per_beta0,
                           r->per_beta_steps, ktrace_slot("sample_per")));
  B2_PROF("sample_per", st);
  return B200DQN_OK;
}

int per_weights_of_indexes(b200dqn_replay* r, cudaStream_t st) {
  k_per_weights<<<cdiv64(r->batch, 128), 128, 0, st>>>(per_view(r), r->d_idx, r->batch, r->d_isw, r->d_words,
                                                       r->per_beta0, r->per_beta_steps);
  B2_LAUNCH_CHECK();
  return B200DQN_OK;
}

int launch_per_update(b200dqn_replay* r, const int32_t* idx, const float* td_err, int rows, cudaStream_t st) {
  NoPdlScope side;   // off the critical chain: ordinary dependencies
  B2_CHECK_CUDA(launch_pdl(k_per_update, dim3(1), dim3(kPerUpdThreads), 0, st, per_view(r), idx, td_err, rows,
                           r->per_alpha, r->per_eps, r->d_maxp, ktrace_slot("per_update")));
  B2_PROF("per_update", st);
  return B200DQN_OK;
}

static int per_alloc(b200dqn_replay* r) {
  if (r->d_sum) return B200DQN_OK;
  int nlev = 0;
  int64_t n = r->size, off = 0;
  while (true) {
    B2_REQUIRE(nlev < b200dqn_replay::kPerMaxLevels, B200DQN_EINVAL, "replay_set_prioritized: ring too large");
    r->per_n[nlev] = n;
    r->per_off[nlev] = off;
    off += (n + 31) / 32 * 32;
    ++nlev;
    if (n == 1) break;
    n = (n + 31) / 32;
  }
  r->per_off[nlev] = off;
  r->per_nlev = nlev;
  B2_CHECK_CUDA(cudaMalloc(&r->d_prio, r->size * sizeof(double)));
  B2_CHECK_CUDA(cudaMalloc(&r->d_sum, off * sizeof(double)));
  B2_CHECK_CUDA(cudaMalloc(&r->d_min, (off - r->per_off[1]) * sizeof(double)));
  B2_CHECK_CUDA(cudaMalloc(&r->d_maxp, sizeof(double)));
  B2_CHECK_CUDA(cudaMalloc(&r->d_isw, r->batch * sizeof(float)));
  B2_CHECK_CUDA(cudaMalloc(&r->d_per_ticket, sizeof(uint32_t)));
  B2_CHECK_CUDA(cudaMemset(r->d_sum, 0, off * sizeof(double)));      // the padding of every level stays zero
  B2_CHECK_CUDA(cudaMemset(r->d_min, 0, (off - r->per_off[1]) * sizeof(double)));
  B2_CHECK_CUDA(cudaMemset(r->d_isw, 0, r->batch * sizeof(float)));
  B2_CHECK_CUDA(cudaMemset(r->d_per_ticket, 0, sizeof(uint32_t)));
  return B200DQN_OK;
}

void per_free(b200dqn_replay* r) {
  cudaFree(r->d_prio); cudaFree(r->d_sum); cudaFree(r->d_min); cudaFree(r->d_maxp); cudaFree(r->d_isw);
  cudaFree(r->d_per_ticket);
}

}  // namespace b200

using namespace b200;

extern "C" int b200dqn_replay_set_prioritized(b200dqn_replay* r, int on, double alpha, double beta0, double beta_steps,
                                              double eps) {
  B2_REQUIRE(r, B200DQN_EINVAL, "null replay");
  B2_REQUIRE(!on || (alpha >= 0.0 && beta0 >= 0.0 && beta0 <= 1.0 && beta_steps >= 0.0 && eps > 0.0), B200DQN_EINVAL,
             "replay_set_prioritized: need alpha >= 0, 0 <= beta0 <= 1, beta_steps >= 0, eps > 0");
  B2_REQUIRE(!on || r->batch <= kPerUpdMaxRows, B200DQN_EINVAL, "replay_set_prioritized: batch > %d", kPerUpdMaxRows);
  DeviceGuard g(r->device);
  B2_CHECK_CUDA(cudaDeviceSynchronize());
  { int frc = replay_flush(r, nullptr); if (frc) return frc; }
  if (on) {
    int rc = per_alloc(r);
    if (rc) return rc;
    r->per_alpha = alpha; r->per_beta0 = beta0; r->per_beta_steps = beta_steps; r->per_eps = eps;
    if ((rc = per_rebuild(r, 0, 0, true, nullptr))) return rc;
    B2_CHECK_CUDA(cudaMemset(r->d_words + 3, 0, sizeof(uint32_t)));   // clear a sticky empty-ring error
  }
  r->per_on = on != 0;
  r->per_gen += 1;
  B2_CHECK_CUDA(cudaDeviceSynchronize());
  r->h_words[3] = 0;
  return B200DQN_OK;
}
