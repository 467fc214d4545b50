// replay.cuh — device-resident replay ring and state window (object layouts).
#pragma once
#include "common.cuh"

struct b200dqn_replay {
  // process-wide creation number, never reused (a ring created after another is destroyed may get its address):
  // what a net's cached step graphs, which bake in this ring's buffers and shape, are keyed by
  uint64_t serial = 0;
  int device = 0;
  int64_t size = 0;
  int h = 0, w = 0, hist = 0, batch = 0;
  int64_t frame_bytes = 0;
  int gather_smem = 0;   // dynamic shared memory k_gather may use on this device: larger frames take its byte loop
  // host mirror of the cursor (src/replay_memory.py:17-18)
  int64_t count = 0, current = 0;

  // HBM
  uint8_t* d_screens = nullptr;    // [size][h][w]
  uint8_t* d_actions = nullptr;    // [size]
  int64_t* d_rewards = nullptr;    // [size]
  uint8_t* d_terminals = nullptr;  // [size] 0/1
  int64_t* d_cursor = nullptr;     // {count, current} — read by the sampler, graph-safe
  // MT19937 state: 624 key words + position (CPython random.getstate()[1]), DOUBLE-BUFFERED: sampling number k
  // (0-based count of samplings done) reads slot k & 1 and leaves the advanced state in slot (k + 1) & 1, so that
  // the many CTAs of the prioritized sampler (per.cu::k_sample_per) can all read the state while one of them writes
  // its successor
  uint32_t* d_mt = nullptr;        // [2][kMtSlot]
  uint32_t* mt_slot_ptr() const { return d_mt + (samples_launched & 1u) * 640; }   // host view: current slot
  int32_t* d_idx = nullptr;        // [batch] accepted indexes, acceptance order
  uint32_t* d_words = nullptr;     // [0] words consumed by the last sample() call, [1] running total
  // host-mapped mirror written by the sampler: [0] samplings completed (published last), [1] words of the last
  // one, [2] running total
  volatile uint32_t* h_words = nullptr;
  uint32_t samples_launched = 0;   // host count of sampler launches (= the sequence number the next wait expects)
  // pinned staging for asynchronous MT19937 state uploads (the host stream moved since the last sampling)
  static constexpr int kMtSlots = 4;
  uint32_t* h_mt = nullptr;        // [kMtSlots][640]
  cudaEvent_t mt_done[kMtSlots] = {};
  int mt_slot = 0;
  uint8_t* d_pre = nullptr;        // [batch][hist][h][w]
  uint8_t* d_post = nullptr;       // [batch][hist][h][w]
  uint8_t* d_mb_actions = nullptr;
  int64_t* d_mb_rewards = nullptr;   // [batch][nstep]: rewards[index .. index + nstep - 1]
  uint8_t* d_mb_terminals = nullptr; // [batch][nstep]
  // n-step returns (b200dqn_replay_set_n_step): a sample is the window [index - hist, index + nstep - 1]; the
  // poststate is getState(index + nstep - 1).  Step graphs capture it (shifts, head), so they compare it.
  int nstep = 1;

  // pinned staging slots (small host<->device landing pads)
  static constexpr int kSlots = 16;
  uint8_t* h_stage = nullptr;
  cudaEvent_t slot_done[kSlots] = {};
  int next_slot = 0;
  bool rng_set = false;

  // add() is deferred: frames + scalars collect in one of two pinned banks and reach HBM in ONE
  // transfer + one tiny kernel when somebody needs the ring (sample / gather / getState / train) or
  // the bank is full.  The host cursor mirror is always current.
  static constexpr int kPend = 8;
  uint8_t* h_bank[2] = {};            // [kPend][frame_bytes] frames, then the scalar arrays
  cudaEvent_t bank_done[2] = {};
  int bank = 0, npend = 0;
  int64_t pend_pos0 = 0;              // ring slot of the first pending frame
  int64_t* bank_rewards(int b) const { return reinterpret_cast<int64_t*>(h_bank[b] + size_t(kPend) * frame_bytes); }
  uint8_t* bank_actions(int b) const { return reinterpret_cast<uint8_t*>(bank_rewards(b) + kPend); }
  uint8_t* bank_terminals(int b) const { return bank_actions(b) + kPend; }

  // Proportional prioritized replay (per.cu; Schaul et al. 2016), off by default.  Allocated the first time it is
  // switched on.  The 32-ary fp64 sum tree holds the leaves (level 0: stored priority of a drawable slot, else 0) and
  // every level above them; the min tree holds levels 1.. (a leaf's min value is itself if positive, else +inf).
  // Each level starts on a 32-node boundary; the padding stays zero.
  static constexpr int kPerMaxLevels = 8;
  bool per_on = false;
  uint32_t per_gen = 0;               // bumped by every switch: step graphs that sample from this ring are stale
  double per_alpha = 0.6, per_beta0 = 0.4, per_beta_steps = 1.0, per_eps = 1e-6;
  int per_nlev = 0;                   // levels including the leaves; the root is level per_nlev - 1
  int64_t per_n[kPerMaxLevels] = {};  // nodes per level
  int64_t per_off[kPerMaxLevels + 1] = {};
  double* d_prio = nullptr;           // [size] stored priorities p^alpha
  double* d_sum = nullptr;            // [per_off[nlev]]
  double* d_min = nullptr;            // [per_off[nlev] - per_off[1]]
  double* d_maxp = nullptr;           // [1] max_priority (not raised to alpha)
  float* d_isw = nullptr;             // [batch] importance weights of the last draw / set_indexes
  uint32_t* d_per_ticket = nullptr;   // [1] CTA arrival counter of the prioritized sampler
};

struct b200dqn_statebuf {
  int device = 0;
  int h = 0, w = 0, hist = 0, batch = 0;
  int64_t frame_bytes = 0;
  uint8_t* d_buf = nullptr;  // [batch][hist][h][w]; only row 0 ever non-zero
  static constexpr int kSlots = 16;
  uint8_t* h_stage = nullptr;
  cudaEvent_t slot_done[kSlots] = {};
  int next_slot = 0;
};

namespace b200 {
// Launches used by the fused train step (net.cu).
int launch_sample(b200dqn_replay* r, cudaStream_t st);
// push the pending add()s to HBM (no-op when there are none); call before anything reads the ring
int replay_flush(b200dqn_replay* r, cudaStream_t st);
int replay_wait_words(b200dqn_replay* r, cudaStream_t st);
int replay_publish_words(b200dqn_replay* r, cudaStream_t st);   // device counters -> host-mapped mirror (tiny kernel)
#ifdef __CUDACC__
// ---- the sampling loop of getMinibatch (src/replay_memory.py:55-69) as a CTA-wide device function, run by the
// sampler kernel (replay.cu::k_sample).  See k_sample for the formulation (one MT19937 word per trial; accepted
// indexes = the first `batch` stream words passing all three tests, in stream order).
constexpr int kMtN = 624, kMtM = 397, kMtSlot = 640;
struct SampleShared {
  uint32_t mt[kMtN + 1];
  int warp_cnt[12];
  int cut;
};
__device__ __forceinline__ uint32_t mt_mix(uint32_t cur, uint32_t nxt, uint32_t far) {
  uint32_t y = (cur & 0x80000000u) | (nxt & 0x7fffffffu);
  return far ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
}
__device__ __forceinline__ uint32_t mt_temper(uint32_t y) {
  y ^= (y >> 11);
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  y ^= (y >> 18);
  return y;
}
// genrand_uint32's regeneration of the whole 624-word key in shared memory, CTA-wide (every thread calls it; the
// caller has synchronised since the last read of the old key).  Three dependency-free segments, then word 623.  Word i
// of a segment reads the OLD word i + 1, which another warp's thread rewrites in the same segment: every thread reads
// its operands, the CTA synchronises, and only then are the new words stored.
__device__ __forceinline__ void mt_regenerate(uint32_t* mt, int tid, int nthreads) {
#pragma unroll 1
  for (int seg = 0; seg < 3; ++seg) {
    const int lo = seg * 227, hi = seg == 2 ? 623 : lo + 227, far = seg == 0 ? kMtM : -227;
    for (int base = lo; base < hi; base += nthreads) {   // one pass when nthreads >= 227
      const int i = base + tid;
      const uint32_t v = i < hi ? mt_mix(mt[i], mt[i + 1], mt[i + far]) : 0u;
      __syncthreads();
      if (i < hi) mt[i] = v;
      __syncthreads();
    }
  }
  if (tid == 0) mt[623] = mt_mix(mt[623], mt[0], mt[396]);
  __syncthreads();
}

// Every thread of the CTA calls this (nthreads = blockDim.x, a multiple of 32, <= 384; __syncthreads inside).  sh.mt
// holds the state on entry and the advanced state (position in [624]) on return; accepted indexes go to idx_out
// (shared or global), in acceptance order.  Returns the number of 32-bit words consumed.
// n-step returns (nstep = N >= 1; count >= hist + N): the trial is randint(hist, count - N), and a sample is rejected
// when its window [index - hist, index + N - 1] straddles the write pointer; at N = 1 this is :59 and :61 exactly.
__device__ __forceinline__ uint32_t sample_block(SampleShared& sh, const uint8_t* __restrict__ terminals, int64_t count,
                                                 int64_t current, int hist, int nstep, int batch, int32_t* idx_out,
                                                 int tid, int nthreads) {
  const int lane = tid & 31, wid = tid >> 5, nwarps = nthreads >> 5;
  uint32_t* mt = sh.mt;
  const uint32_t n = static_cast<uint32_t>(count - hist - nstep + 1);  // width of randrange(hist, count - N + 1)
  const int kbits = 32 - __clz(n);                         // n.bit_length(), n >= 1
  int pos = static_cast<int>(mt[kMtN]);
  int accepted = 0;
  uint32_t words = 0;
  while (accepted < batch) {
    if (pos >= kMtN) {  // genrand_uint32: regenerate the whole key, position 0
      mt_regenerate(mt, tid, nthreads);
      pos = 0;
    }
    const int avail = min(kMtN - pos, nthreads);
    bool ok = false;
    int index = 0;
    if (tid < avail) {
      const uint32_t r = mt_temper(mt[pos + tid]) >> (32 - kbits);
      if (r < n) {
        index = hist + static_cast<int>(r);
        ok = !(index + nstep - 1 >= current && index - hist < current);  // :61 wraps over the write pointer
        // :65 episode end — all `hist` bytes are requested at once (no short-circuit: one memory latency, not four)
        unsigned any = 0;
        for (int j = 1; j <= hist; ++j) any |= terminals[index - j];
        ok = ok && any == 0;
      }
    }
    const unsigned ballot = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) sh.warp_cnt[wid] = __popc(ballot);
    if (tid == 0) sh.cut = -1;
    __syncthreads();
    int before = 0, total = 0;
    for (int wi = 0; wi < nwarps; ++wi) {
      const int c = sh.warp_cnt[wi];
      if (wi < wid) before += c;
      total += c;
    }
    const int rank = accepted + before + __popc(ballot & ((1u << lane) - 1u));
    if (ok && rank < batch) {
      idx_out[rank] = index;
      if (rank == batch - 1) sh.cut = tid;  // the word that completed the minibatch
    }
    __syncthreads();
    if (accepted + total >= batch) {
      const int used = sh.cut + 1;
      pos += used;
      words += used;
      accepted = batch;
    } else {
      accepted += total;
      pos += avail;
      words += avail;
    }
    __syncthreads();
  }
  if (tid == 0) mt[kMtN] = static_cast<uint32_t>(pos);
  __syncthreads();
  return words;
}

// [0] samplings completed (published last), [1] words of the last one, [2] running total, [3] sticky error of the
// prioritized sampler (a draw from a ring with no drawable slot)
__device__ __forceinline__ void publish_words(const uint32_t* __restrict__ words, volatile uint32_t* host_words) {
  host_words[1] = words[0];
  host_words[2] = words[1];
  host_words[3] = words[3];
  __threadfence_system();
  host_words[0] = words[2];
}
#endif
// adopt a host MT19937 state (624 key words + position) without synchronising the stream
int replay_set_rng_async(b200dqn_replay* r, const uint32_t* key624, uint32_t pos, cudaStream_t st);

// ---- prioritized replay (per.cu)
int launch_sample_per(b200dqn_replay* r, cudaStream_t st);
// leaves and ancestors of the slots written by a flush of n deferred add()s starting at pos0
int per_after_add(b200dqn_replay* r, int64_t pos0, int64_t n, cudaStream_t st);
// every leaf and node from the stored priorities (fill_from/fill_n: slots that get max_priority^alpha first)
int per_rebuild(b200dqn_replay* r, int64_t fill_from, int64_t fill_n, bool init, cudaStream_t st);
// importance weights of the indexes in d_idx (set_indexes on a prioritized ring)
int per_weights_of_indexes(b200dqn_replay* r, cudaStream_t st);
// priority update after a train step: td_err[rows] of the indexes idx[rows]
int launch_per_update(b200dqn_replay* r, const int32_t* idx, const float* td_err, int rows, cudaStream_t st);
void per_free(b200dqn_replay* r);
}  // namespace b200
