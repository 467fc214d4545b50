// replay.cu — replay ring in HBM: add / getState / device MT19937 sampler / TMA-bulk gather,
// and the device-side StateBuffer.  Replaces src/replay_memory.py and src/state_buffer.py of
// the reference (file:line cited per function in include/b200dqn.h).
#include <atomic>
#include <new>

#include "replay.cuh"

namespace b200 {

// ------------------------------------------------------------------------------------------
// K8a: metadata write of ReplayMemory.add (src/replay_memory.py:29-34).  The frame itself is a
// plain async H2D copy; the scalars ride in the kernel arguments, the cursor is mirrored to
// device memory so graph-captured samplers always see the live count/current.
// ------------------------------------------------------------------------------------------
__global__ void k_add_meta(uint8_t* actions, int64_t* rewards, uint8_t* terminals, int64_t* cursor,
                           int64_t pos, int action, int64_t reward, int terminal, int64_t new_count,
                           int64_t new_current) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    actions[pos] = static_cast<uint8_t>(action);
    rewards[pos] = reward;
    terminals[pos] = terminal ? 1 : 0;
    cursor[0] = new_count;
    cursor[1] = new_current;
  }
}

__global__ void k_set_cursor(int64_t* cursor, int64_t count, int64_t current) {
  cursor[0] = count;
  cursor[1] = current;
}

// metadata of up to kPend deferred add()s; the scalar arrays are read straight from pinned host memory
__global__ void k_add_meta_batch(uint8_t* actions, int64_t* rewards, uint8_t* terminals, int64_t* cursor,
                                 int64_t pos0, int64_t size, int n, const uint8_t* __restrict__ h_actions,
                                 const int64_t* __restrict__ h_rewards, const uint8_t* __restrict__ h_terminals,
                                 int64_t new_count, int64_t new_current) {
  const int i = threadIdx.x;
  if (i < n) {
    const int64_t pos = (pos0 + i) % size;
    actions[pos] = h_actions[i];
    rewards[pos] = h_rewards[i];
    terminals[pos] = h_terminals[i] ? 1 : 0;
  }
  if (i == 0) {
    cursor[0] = new_count;
    cursor[1] = new_current;
  }
}

// ------------------------------------------------------------------------------------------
// K1a: the sampling loop of getMinibatch (src/replay_memory.py:55-69) on the device.
//
// CPython-3 randint(hist, count-1) = hist + _randbelow(n), n = count - hist, and every trial
// (including the r >= n retry of _randbelow and the two rejections of :61/:65) consumes exactly
// one MT19937 output word.  Hence: accepted indexes = the first `batch` stream words that pass
// all three tests, in stream order.  One CTA evaluates up to 256 consecutive words per round,
// compacts the survivors in order with ballot + prefix counts, and regenerates the 624-word
// state in three dependency-free segments when the position reaches 624 (see
// oracle/mt19937.py::twist_segmented for the proof-by-test of that formulation).
// ------------------------------------------------------------------------------------------
constexpr int kSampleThreads = 256;

__global__ void __launch_bounds__(kSampleThreads, 1)
k_sample(uint32_t* __restrict__ mt_state, const uint8_t* __restrict__ terminals,
         const int64_t* __restrict__ cursor, int hist, int nstep, int batch, int32_t* __restrict__ idx_out,
         uint32_t* __restrict__ words_out, const KTrace kt) {
  __shared__ SampleShared sh;
  const int tid = threadIdx.x;
  kt_begin(kt);
  pdl_wait();
  pdl_launch_dependents();
  const uint32_t k = words_out[2];                      // samplings done so far: selects the state slot
  const uint32_t* cur = mt_state + (k & 1u) * kMtSlot;
  uint32_t* nxt = mt_state + ((k + 1u) & 1u) * kMtSlot;
  for (int i = tid; i < kMtN + 1; i += kSampleThreads) sh.mt[i] = cur[i];
  __syncthreads();
  const uint32_t words =
      sample_block(sh, terminals, cursor[0], cursor[1], hist, nstep, batch, idx_out, tid, kSampleThreads);
  for (int i = tid; i < kMtN + 1; i += kSampleThreads) nxt[i] = sh.mt[i];
  if (tid == 0) {
    words_out[0] = words;
    words_out[1] += words;
    words_out[2] = k + 1;         // samplings completed
  }
  kt_end(kt);
}

// Host-mapped mirror of the sampler's counters: data, system fence, then the sequence number the host polls.  Kept
// OUT of k_sample (a system-scope fence on the critical chain costs ~2 us): the fused step publishes from its
// off-chain cost kernel, a stand-alone sampling from this one-thread kernel.
__global__ void k_publish_words(const uint32_t* __restrict__ words, volatile uint32_t* host_words) {
  publish_words(words, host_words);
}

int replay_publish_words(b200dqn_replay* r, cudaStream_t st) {
  k_publish_words<<<1, 1, 0, st>>>(r->d_words, r->h_words);
  B2_LAUNCH_CHECK();
  return B200DQN_OK;
}

int replay_flush(b200dqn_replay* r, cudaStream_t st) {
  if (r->npend == 0) return B200DQN_OK;
  const int b = r->bank, n = r->npend;
  const int64_t pos0 = r->pend_pos0;
  const int64_t first = (r->size - pos0) < n ? (r->size - pos0) : n;   // frames before the ring wraps
  B2_CHECK_CUDA(cudaMemcpyAsync(r->d_screens + pos0 * r->frame_bytes, r->h_bank[b], first * r->frame_bytes,
                                cudaMemcpyHostToDevice, st));
  if (first < n)
    B2_CHECK_CUDA(cudaMemcpyAsync(r->d_screens, r->h_bank[b] + first * r->frame_bytes, (n - first) * r->frame_bytes,
                                  cudaMemcpyHostToDevice, st));
  k_add_meta_batch<<<1, 32, 0, st>>>(r->d_actions, r->d_rewards, r->d_terminals, r->d_cursor, pos0, r->size, n,
                                     r->bank_actions(b), r->bank_rewards(b), r->bank_terminals(b), r->count,
                                     r->current);
  B2_LAUNCH_CHECK();
  if (r->per_on) {
    int rc = per_after_add(r, pos0, n, st);
    if (rc) return rc;
  }
  B2_CHECK_CUDA(cudaEventRecord(r->bank_done[b], st));
  r->bank ^= 1;
  r->npend = 0;
  B2_CHECK_CUDA(cudaEventSynchronize(r->bank_done[r->bank]));   // the other bank must have drained (it has, long ago)
  return B200DQN_OK;
}

// wait (polling host-mapped memory) until every sampler launched so far has published its word count
int replay_wait_words(b200dqn_replay* r, cudaStream_t st) {
  const int rc = poll_mapped_seq(r->h_words, r->samples_launched, st, "sampler result");
  if (rc) return rc;
  B2_REQUIRE(r->h_words[3] == 0, B200DQN_ESTATE,
             "prioritized getMinibatch: the ring has no slot the sampler may draw (every leaf of the sum tree is 0)");
  return B200DQN_OK;
}

int replay_set_rng_async(b200dqn_replay* r, const uint32_t* key624, uint32_t pos, cudaStream_t st) {
  B2_REQUIRE(pos <= 624, B200DQN_EINVAL, "MT19937 position %u > 624", pos);
  const int slot = r->mt_slot;
  r->mt_slot = (slot + 1) % b200dqn_replay::kMtSlots;
  B2_CHECK_CUDA(cudaEventSynchronize(r->mt_done[slot]));   // the copy that last used this slot (long finished)
  uint32_t* pin = r->h_mt + size_t(slot) * 640;
  memcpy(pin, key624, 624 * sizeof(uint32_t));
  pin[624] = pos;
  B2_CHECK_CUDA(cudaMemcpyAsync(r->mt_slot_ptr(), pin, 625 * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  B2_CHECK_CUDA(cudaEventRecord(r->mt_done[slot], st));
  r->rng_set = true;
  return B200DQN_OK;
}

int launch_sample(b200dqn_replay* r, cudaStream_t st) {
  int frc = replay_flush(r, st);
  if (frc) return frc;
  if (r->per_on) return launch_sample_per(r, st);
  B2_CHECK_CUDA(launch_pdl(k_sample, dim3(1), dim3(kSampleThreads), 0, st, r->d_mt, (const uint8_t*)r->d_terminals,
                           (const int64_t*)r->d_cursor, r->hist, r->nstep, r->batch, r->d_idx, r->d_words,
                           ktrace_slot("sample")));
  B2_PROF("sample", st);
  return B200DQN_OK;
}

// ------------------------------------------------------------------------------------------
// K1b: the copy half of getMinibatch (src/replay_memory.py:71-78).  Per sample the hist+1 frames
// index-hist .. index are one contiguous span of the ring; CTA (k, f) pulls frame f of sample k
// into shared memory with one TMA bulk copy (UBLKCP) and pushes it back out with bulk stores to
// the prestates slot f (f < hist) and the poststates slot f-1 (f >= 1): each ring byte is read
// from HBM exactly once.  Frame sizes that are not a multiple of 16 B take the byte-loop path.
// n-step returns (nstep = N): the span is index-hist .. index+N-1 (hist+N frames), frame f goes to the prestates if
// f < hist and to poststate slot f-N if f >= N, and the rewards and terminals of index .. index+N-1 are staged as
// [batch][N].  A CTA whose frame is in neither state (hist <= f < N) has nothing to copy.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
k_gather(const uint8_t* __restrict__ screens, const uint8_t* __restrict__ actions,
         const int64_t* __restrict__ rewards, const uint8_t* __restrict__ terminals,
         const int32_t* __restrict__ idx, int hist, int nstep, uint32_t frame_bytes, uint8_t* __restrict__ pre,
         uint8_t* __restrict__ post, uint8_t* __restrict__ mb_actions, int64_t* __restrict__ mb_rewards,
         uint8_t* __restrict__ mb_terminals, int use_tma) {
  extern __shared__ __align__(128) uint8_t s_frame[];
  __shared__ __align__(8) uint64_t bar;
  const int k = blockIdx.x, f = blockIdx.y;
  const int64_t index = idx[k];
  const uint8_t* src = screens + (index - hist + f) * static_cast<int64_t>(frame_bytes);
  uint8_t* dst_pre = pre + (static_cast<int64_t>(k) * hist + f) * frame_bytes;
  uint8_t* dst_post = post + (static_cast<int64_t>(k) * hist + (f - nstep)) * frame_bytes;

  if (f == 0 && threadIdx.x == 32) mb_actions[k] = actions[index];
  if (f == 0 && threadIdx.x >= 32 && threadIdx.x < 64) {
    for (int j = threadIdx.x - 32; j < nstep; j += 32) {
      mb_rewards[int64_t(k) * nstep + j] = rewards[index + j];
      mb_terminals[int64_t(k) * nstep + j] = terminals[index + j];
    }
  }
  const bool to_pre = f < hist, to_post = f >= nstep;
  if (!to_pre && !to_post) return;
  if (use_tma) {
    if (threadIdx.x == 0) {
      mbar_init(&bar, 1);
      mbar_fence_init();
      mbar_arrive_expect_tx(&bar, frame_bytes);
      tma_bulk_g2s(s_frame, src, frame_bytes, &bar);
      mbar_wait(&bar, 0);
      if (to_pre) tma_bulk_s2g(dst_pre, s_frame, frame_bytes);
      if (to_post) tma_bulk_s2g(dst_post, s_frame, frame_bytes);
      tma_bulk_commit();
      tma_bulk_wait_read_all();  // smem may be released once the reads are done
    }
  } else {
    for (uint32_t i = threadIdx.x; i < frame_bytes; i += blockDim.x) {
      const uint8_t v = src[i];
      if (to_pre) dst_pre[i] = v;
      if (to_post) dst_post[i] = v;
    }
  }
}

// StateBuffer.add (src/state_buffer.py:15-18): each thread owns one 16-byte (or 1-byte) column of
// the four frames of row 0, so the in-place shift has no cross-thread hazard.
template <typename T>
__global__ void k_statebuf_shift(T* __restrict__ row0, const T* __restrict__ fresh, int hist, int64_t n_per_frame) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n_per_frame) return;
  for (int f = 0; f + 1 < hist; ++f) row0[f * n_per_frame + i] = row0[(f + 1) * n_per_frame + i];
  row0[(hist - 1) * n_per_frame + i] = fresh[i];
}

}  // namespace b200

using namespace b200;

// b200dqn_replay::serial of the next ring created in this process (0 names no ring)
static std::atomic<uint64_t> g_replay_serial{1};

// ============================================================================ C ABI: replay
extern "C" int b200dqn_replay_create(int device, int64_t size, int screen_h, int screen_w, int history_length,
                                     int batch_size, b200dqn_replay** out) {
  B2_REQUIRE(out && size > 0 && screen_h > 0 && screen_w > 0 && history_length > 0 && batch_size > 0,
             B200DQN_EINVAL, "replay_create: bad argument");
  B2_REQUIRE(size < (int64_t(1) << 31), B200DQN_EINVAL, "replay_create: size must fit int32 indexes");
  B2_REQUIRE(size >= b200dqn_replay::kPend, B200DQN_EINVAL,
             "replay_create: size %lld is smaller than the %d-frame ingestion bank (a deferred flush may wrap at most once)",
             (long long)size, b200dqn_replay::kPend);
  DeviceGuard g(device);
  auto* r = new (std::nothrow) b200dqn_replay();
  B2_REQUIRE(r, B200DQN_EINVAL, "out of host memory");
  r->device = device;
  r->size = size;
  r->h = screen_h;
  r->w = screen_w;
  r->hist = history_length;
  r->batch = batch_size;
  r->frame_bytes = int64_t(screen_h) * screen_w;
  const size_t state_bytes = size_t(batch_size) * history_length * r->frame_bytes;
  // the ring gets hist frames of slack so that vector loads of the last sample never run off the end
  B2_CHECK_CUDA(cudaMalloc(&r->d_screens, size_t(size) * r->frame_bytes + 256));
  B2_CHECK_CUDA(cudaMalloc(&r->d_actions, size));
  B2_CHECK_CUDA(cudaMalloc(&r->d_rewards, size * sizeof(int64_t)));
  B2_CHECK_CUDA(cudaMalloc(&r->d_terminals, size));
  B2_CHECK_CUDA(cudaMalloc(&r->d_cursor, 2 * sizeof(int64_t)));
  B2_CHECK_CUDA(cudaMalloc(&r->d_mt, 2 * 640 * sizeof(uint32_t)));
  B2_CHECK_CUDA(cudaMalloc(&r->d_idx, batch_size * sizeof(int32_t)));
  B2_CHECK_CUDA(cudaMalloc(&r->d_words, 4 * sizeof(uint32_t)));
  B2_CHECK_CUDA(cudaMalloc(&r->d_pre, state_bytes));
  B2_CHECK_CUDA(cudaMalloc(&r->d_post, state_bytes));
  B2_CHECK_CUDA(cudaMalloc(&r->d_mb_actions, batch_size));
  B2_CHECK_CUDA(cudaMalloc(&r->d_mb_rewards, batch_size * sizeof(int64_t)));
  B2_CHECK_CUDA(cudaMalloc(&r->d_mb_terminals, batch_size));
  // np.empty in the reference leaves garbage; zero is a valid instance of garbage and keeps
  // terminal tests on never-written slots deterministic.
  B2_CHECK_CUDA(cudaMemset(r->d_actions, 0, size));
  B2_CHECK_CUDA(cudaMemset(r->d_rewards, 0, size * sizeof(int64_t)));
  B2_CHECK_CUDA(cudaMemset(r->d_terminals, 0, size));
  B2_CHECK_CUDA(cudaMemset(r->d_cursor, 0, 2 * sizeof(int64_t)));
  B2_CHECK_CUDA(cudaMemset(r->d_mt, 0, 2 * 640 * sizeof(uint32_t)));
  B2_CHECK_CUDA(cudaMemset(r->d_idx, 0, batch_size * sizeof(int32_t)));
  B2_CHECK_CUDA(cudaMemset(r->d_words, 0, 4 * sizeof(uint32_t)));
  B2_CHECK_CUDA(cudaMallocHost(&r->h_stage, size_t(b200dqn_replay::kSlots) * r->frame_bytes));
  B2_CHECK_CUDA(cudaMallocHost(&r->h_mt, size_t(b200dqn_replay::kMtSlots) * 640 * sizeof(uint32_t)));
  for (auto& e : r->mt_done) B2_CHECK_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  {
    void* m = nullptr;
    B2_CHECK_CUDA(cudaHostAlloc(&m, 64, cudaHostAllocMapped));
    memset(m, 0, 64);
    r->h_words = static_cast<volatile uint32_t*>(m);
  }
  for (int b = 0; b < 2; ++b) {
    B2_CHECK_CUDA(cudaMallocHost(&r->h_bank[b], size_t(b200dqn_replay::kPend) * (r->frame_bytes + 16)));
    B2_CHECK_CUDA(cudaEventCreateWithFlags(&r->bank_done[b], cudaEventDisableTiming));
  }
  for (int i = 0; i < b200dqn_replay::kSlots; ++i)
    B2_CHECK_CUDA(cudaEventCreateWithFlags(&r->slot_done[i], cudaEventDisableTiming));
  // k_gather stages one frame in dynamic shared memory.  Its limit is raised to all that one block may opt into, the
  // same for every ring on the device, so that creating a ring of smaller frames never lowers it under another
  // ring's; frames larger than that take the byte loop (b200dqn_replay_gather).
  {
    int optin = 0;
    cudaFuncAttributes fa{};
    B2_CHECK_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
    B2_CHECK_CUDA(cudaFuncGetAttributes(&fa, k_gather));
    r->gather_smem = optin - int(fa.sharedSizeBytes);
    B2_CHECK_CUDA(cudaFuncSetAttribute(k_gather, cudaFuncAttributeMaxDynamicSharedMemorySize, r->gather_smem));
  }
  r->serial = g_replay_serial.fetch_add(1, std::memory_order_relaxed);
  *out = r;
  return B200DQN_OK;
}

extern "C" int b200dqn_replay_destroy(b200dqn_replay* r) {
  if (!r) return B200DQN_OK;
  DeviceGuard g(r->device);
  cudaDeviceSynchronize();
  cudaFree(r->d_screens); cudaFree(r->d_actions); cudaFree(r->d_rewards); cudaFree(r->d_terminals);
  cudaFree(r->d_cursor); cudaFree(r->d_mt); cudaFree(r->d_idx); cudaFree(r->d_words);
  cudaFree(r->d_pre); cudaFree(r->d_post); cudaFree(r->d_mb_actions); cudaFree(r->d_mb_rewards);
  cudaFree(r->d_mb_terminals);
  per_free(r);
  cudaFreeHost(r->h_stage);
  cudaFreeHost(const_cast<uint32_t*>(r->h_words));
  cudaFreeHost(r->h_mt);
  for (auto& e : r->mt_done) if (e) cudaEventDestroy(e);
  for (int b = 0; b < 2; ++b) { cudaFreeHost(r->h_bank[b]); if (r->bank_done[b]) cudaEventDestroy(r->bank_done[b]); }
  for (auto& e : r->slot_done) if (e) cudaEventDestroy(e);
  delete r;
  return B200DQN_OK;
}

extern "C" int b200dqn_replay_add(b200dqn_replay* r, int action, int64_t reward, const uint8_t* host_screen,
                                  int terminal, void* stream) {
  B2_REQUIRE(r && host_screen, B200DQN_EINVAL, "replay_add: null argument");
  DeviceGuard g(r->device);
  const int b = r->bank, i = r->npend;
  const int64_t pos = r->current;
  if (i == 0) r->pend_pos0 = pos;
  memcpy(r->h_bank[b] + size_t(i) * r->frame_bytes, host_screen, r->frame_bytes);
  r->bank_actions(b)[i] = static_cast<uint8_t>(action);
  r->bank_rewards(b)[i] = reward;
  r->bank_terminals(b)[i] = terminal ? 1 : 0;
  r->npend = i + 1;
  r->count = r->count > pos + 1 ? r->count : pos + 1;   // :33
  r->current = (pos + 1) % r->size;                      // :34
  if (r->npend == b200dqn_replay::kPend) return replay_flush(r, as_stream(stream));
  return B200DQN_OK;
}

extern "C" int b200dqn_replay_add_batch(b200dqn_replay* r, int64_t n, const uint8_t* host_actions,
                                        const int64_t* host_rewards, const uint8_t* host_screens,
                                        const uint8_t* host_terminals, void* stream) {
  B2_REQUIRE(r && n >= 0 && host_actions && host_rewards && host_screens && host_terminals, B200DQN_EINVAL,
             "replay_add_batch: bad argument");
  DeviceGuard g(r->device);
  cudaStream_t st = as_stream(stream);
  { int frc = replay_flush(r, st); if (frc) return frc; }
  const int64_t pos_first = r->current;
  int64_t done = 0;
  while (done < n) {
    const int64_t pos = r->current;
    const int64_t seg = (n - done) < (r->size - pos) ? (n - done) : (r->size - pos);
    B2_CHECK_CUDA(cudaMemcpyAsync(r->d_screens + pos * r->frame_bytes, host_screens + done * r->frame_bytes,
                                  seg * r->frame_bytes, cudaMemcpyHostToDevice, st));
    B2_CHECK_CUDA(cudaMemcpyAsync(r->d_actions + pos, host_actions + done, seg, cudaMemcpyHostToDevice, st));
    B2_CHECK_CUDA(cudaMemcpyAsync(r->d_rewards + pos, host_rewards + done, seg * sizeof(int64_t),
                                  cudaMemcpyHostToDevice, st));
    B2_CHECK_CUDA(cudaMemcpyAsync(r->d_terminals + pos, host_terminals + done, seg, cudaMemcpyHostToDevice, st));
    r->count = r->count > pos + seg ? r->count : pos + seg;
    r->current = (pos + seg) % r->size;
    done += seg;
  }
  k_set_cursor<<<1, 1, 0, st>>>(r->d_cursor, r->count, r->current);
  B2_LAUNCH_CHECK();
  if (r->per_on) {   // the written slots get max_priority^alpha; every leaf and node is re-derived
    int rc = per_rebuild(r, pos_first, n, false, st);
    if (rc) return rc;
  }
  B2_CHECK_CUDA(cudaStreamSynchronize(st));  // host arrays may be reused by the caller
  return B200DQN_OK;
}

extern "C" int b200dqn_replay_get_cursor(const b200dqn_replay* r, int64_t* count, int64_t* current) {
  B2_REQUIRE(r, B200DQN_EINVAL, "null replay");
  if (count) *count = r->count;
  if (current) *current = r->current;
  return B200DQN_OK;
}

extern "C" int b200dqn_replay_set_cursor(b200dqn_replay* r, int64_t count, int64_t current) {
  B2_REQUIRE(r && count >= 0 && count <= r->size && current >= 0 && current < r->size, B200DQN_EINVAL,
             "replay_set_cursor: out of range");
  DeviceGuard g(r->device);
  { int frc = replay_flush(r, nullptr); if (frc) return frc; }
  r->count = count;
  r->current = current;
  k_set_cursor<<<1, 1>>>(r->d_cursor, count, current);
  B2_LAUNCH_CHECK();
  if (r->per_on) {   // the drawable set follows the cursor
    int rc = per_rebuild(r, 0, 0, false, nullptr);
    if (rc) return rc;
  }
  B2_CHECK_CUDA(cudaDeviceSynchronize());
  return B200DQN_OK;
}

extern "C" int b200dqn_replay_get_state(b200dqn_replay* r, int64_t index, uint8_t* host_out, void* stream) {
  B2_REQUIRE(r && host_out, B200DQN_EINVAL, "replay_get_state: null argument");
  B2_REQUIRE(r->count > 0, B200DQN_ESTATE, "replay memory is empy, use at least --random_steps 1");  // :38
  DeviceGuard g(r->device);
  cudaStream_t st = as_stream(stream);
  { int frc = replay_flush(r, st); if (frc) return frc; }
  index = ((index % r->count) + r->count) % r->count;  // python modulo (:40)
  if (index >= r->hist - 1) {
    B2_CHECK_CUDA(cudaMemcpyAsync(host_out, r->d_screens + (index - (r->hist - 1)) * r->frame_bytes,
                                  r->hist * r->frame_bytes, cudaMemcpyDeviceToHost, st));
  } else {
    for (int j = 0; j < r->hist; ++j) {  // :46-47, oldest first
      const int i = r->hist - 1 - j;
      const int64_t src = (((index - i) % r->count) + r->count) % r->count;
      B2_CHECK_CUDA(cudaMemcpyAsync(host_out + j * r->frame_bytes, r->d_screens + src * r->frame_bytes,
                                    r->frame_bytes, cudaMemcpyDeviceToHost, st));
    }
  }
  B2_CHECK_CUDA(cudaStreamSynchronize(st));
  return B200DQN_OK;
}

extern "C" int b200dqn_replay_set_rng(b200dqn_replay* r, const uint32_t host_mt625[625], void* stream) {
  B2_REQUIRE(r && host_mt625, B200DQN_EINVAL, "replay_set_rng: null argument");
  B2_REQUIRE(host_mt625[624] <= 624, B200DQN_EINVAL, "replay_set_rng: MT19937 position %u > 624", host_mt625[624]);
  DeviceGuard g(r->device);
  cudaStream_t st = as_stream(stream);
  B2_CHECK_CUDA(cudaMemcpyAsync(r->mt_slot_ptr(), host_mt625, 625 * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  B2_CHECK_CUDA(cudaStreamSynchronize(st));
  r->rng_set = true;
  return B200DQN_OK;
}

extern "C" int b200dqn_replay_set_rng_parts(b200dqn_replay* r, const uint32_t* host_key624, uint32_t host_pos,
                                            void* stream) {
  B2_REQUIRE(r && host_key624, B200DQN_EINVAL, "replay_set_rng_parts: null argument");
  DeviceGuard g(r->device);
  return replay_set_rng_async(r, host_key624, host_pos, as_stream(stream));
}

extern "C" int b200dqn_replay_get_rng(b200dqn_replay* r, uint32_t host_mt625[625], void* stream) {
  B2_REQUIRE(r && host_mt625, B200DQN_EINVAL, "replay_get_rng: null argument");
  DeviceGuard g(r->device);
  cudaStream_t st = as_stream(stream);
  B2_CHECK_CUDA(cudaMemcpyAsync(host_mt625, r->mt_slot_ptr(), 625 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  B2_CHECK_CUDA(cudaStreamSynchronize(st));
  return B200DQN_OK;
}

extern "C" int b200dqn_replay_sample(b200dqn_replay* r, void* stream) {
  B2_REQUIRE(r, B200DQN_EINVAL, "null replay");
  B2_REQUIRE(r->count >= r->hist + r->nstep, B200DQN_ESTATE,
             "getMinibatch: count (%lld) must be at least history_length (%d) + n_step (%d)", (long long)r->count,
             r->hist, r->nstep);  // :52 at n_step 1
  B2_REQUIRE(r->rng_set, B200DQN_ESTATE, "replay_sample: call b200dqn_replay_set_rng first");
  DeviceGuard g(r->device);
  int rc = launch_sample(r, as_stream(stream));
  if (!rc) r->samples_launched += 1;
  return rc;
}

extern "C" int b200dqn_replay_sample_sync(b200dqn_replay* r, uint32_t* host_words_consumed, void* stream) {
  B2_REQUIRE(host_words_consumed, B200DQN_EINVAL, "replay_sample_sync: null argument");
  int rc = b200dqn_replay_sample(r, stream);
  if (rc) return rc;
  if ((rc = replay_publish_words(r, as_stream(stream)))) return rc;
  rc = replay_wait_words(r, as_stream(stream));
  if (rc) return rc;
  *host_words_consumed = r->h_words[1];
  return B200DQN_OK;
}

extern "C" int b200dqn_replay_set_indexes(b200dqn_replay* r, const int32_t* host_indexes, void* stream) {
  B2_REQUIRE(r && host_indexes, B200DQN_EINVAL, "replay_set_indexes: null argument");
  for (int i = 0; i < r->batch; ++i)
    B2_REQUIRE(host_indexes[i] >= r->hist && host_indexes[i] <= r->size - r->nstep, B200DQN_EINVAL,
               "replay_set_indexes: index %d out of [hist, size - n_step]", host_indexes[i]);
  DeviceGuard g(r->device);
  cudaStream_t st = as_stream(stream);
  B2_CHECK_CUDA(cudaMemcpyAsync(r->d_idx, host_indexes, r->batch * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  if (r->per_on) {   // a prioritized ring trains these indexes exactly as if they had been drawn
    { int frc = replay_flush(r, st); if (frc) return frc; }
    int rc = per_weights_of_indexes(r, st);
    if (rc) return rc;
  }
  B2_CHECK_CUDA(cudaStreamSynchronize(st));
  return B200DQN_OK;
}

extern "C" int b200dqn_replay_gather(b200dqn_replay* r, void* stream) {
  B2_REQUIRE(r, B200DQN_EINVAL, "null replay");
  DeviceGuard g(r->device);
  { int frc = replay_flush(r, as_stream(stream)); if (frc) return frc; }
  const int use_tma = (r->frame_bytes % 16 == 0 && r->frame_bytes <= r->gather_smem) ? 1 : 0;
  dim3 grid(r->batch, r->hist + r->nstep);
  k_gather<<<grid, 128, use_tma ? r->frame_bytes : 0, as_stream(stream)>>>(
      r->d_screens, r->d_actions, r->d_rewards, r->d_terminals, r->d_idx, r->hist, r->nstep, uint32_t(r->frame_bytes),
      r->d_pre, r->d_post, r->d_mb_actions, r->d_mb_rewards, r->d_mb_terminals, use_tma);
  B2_LAUNCH_CHECK();
  B2_PROF("gather", as_stream(stream));
  return B200DQN_OK;
}

extern "C" int b200dqn_replay_read_minibatch(b200dqn_replay* r, uint8_t* host_pre, uint8_t* host_actions,
                                             int64_t* host_rewards, uint8_t* host_post, uint8_t* host_terminals,
                                             int32_t* host_indexes, uint32_t* host_words_consumed, void* stream) {
  B2_REQUIRE(r, B200DQN_EINVAL, "null replay");
  DeviceGuard g(r->device);
  cudaStream_t st = as_stream(stream);
  const size_t state_bytes = size_t(r->batch) * r->hist * r->frame_bytes;
  if (host_pre) B2_CHECK_CUDA(cudaMemcpyAsync(host_pre, r->d_pre, state_bytes, cudaMemcpyDeviceToHost, st));
  if (host_post) B2_CHECK_CUDA(cudaMemcpyAsync(host_post, r->d_post, state_bytes, cudaMemcpyDeviceToHost, st));
  if (host_actions) B2_CHECK_CUDA(cudaMemcpyAsync(host_actions, r->d_mb_actions, r->batch, cudaMemcpyDeviceToHost, st));
  const size_t nmb = size_t(r->batch) * r->nstep;   // (batch, n_step) rewards and terminals
  if (host_rewards)
    B2_CHECK_CUDA(cudaMemcpyAsync(host_rewards, r->d_mb_rewards, nmb * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  if (host_terminals)
    B2_CHECK_CUDA(cudaMemcpyAsync(host_terminals, r->d_mb_terminals, nmb, cudaMemcpyDeviceToHost, st));
  if (host_indexes)
    B2_CHECK_CUDA(cudaMemcpyAsync(host_indexes, r->d_idx, r->batch * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  if (host_words_consumed)
    B2_CHECK_CUDA(cudaMemcpyAsync(host_words_consumed, r->d_words, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  B2_CHECK_CUDA(cudaStreamSynchronize(st));
  return B200DQN_OK;
}

extern "C" int b200dqn_replay_set_n_step(b200dqn_replay* r, int n) {
  B2_REQUIRE(r, B200DQN_EINVAL, "null replay");
  B2_REQUIRE(n >= 1 && int64_t(r->hist) + n <= r->size, B200DQN_EINVAL,
             "replay_set_n_step: need 1 <= n_step and history_length (%d) + n_step (%d) <= size (%lld)", r->hist, n,
             (long long)r->size);
  if (n == r->nstep) return B200DQN_OK;
  DeviceGuard g(r->device);
  B2_CHECK_CUDA(cudaDeviceSynchronize());   // nothing in flight reads the staged rewards and terminals
  { int frc = replay_flush(r, nullptr); if (frc) return frc; }
  int64_t* rew = nullptr;
  uint8_t* term = nullptr;
  B2_CHECK_CUDA(cudaMalloc(&rew, size_t(r->batch) * n * sizeof(int64_t)));
  B2_CHECK_CUDA(cudaMalloc(&term, size_t(r->batch) * n));
  B2_CHECK_CUDA(cudaMemset(rew, 0, size_t(r->batch) * n * sizeof(int64_t)));
  B2_CHECK_CUDA(cudaMemset(term, 0, size_t(r->batch) * n));
  cudaFree(r->d_mb_rewards);
  cudaFree(r->d_mb_terminals);
  r->d_mb_rewards = rew;
  r->d_mb_terminals = term;
  r->nstep = n;   // the nets' step graphs compare it
  if (r->per_on) {   // the drawable set follows the window
    int rc = per_rebuild(r, 0, 0, false, nullptr);
    if (rc) return rc;
  }
  B2_CHECK_CUDA(cudaDeviceSynchronize());
  return B200DQN_OK;
}

extern "C" int b200dqn_replay_device_ptr(b200dqn_replay* r, int which, void** dev_ptr, size_t* bytes) {
  B2_REQUIRE(r && dev_ptr, B200DQN_EINVAL, "replay_device_ptr: null argument");
  { DeviceGuard g(r->device); int frc = replay_flush(r, nullptr); if (frc) return frc; cudaStreamSynchronize(nullptr); }
  const size_t state_bytes = size_t(r->batch) * r->hist * r->frame_bytes;
  void* p = nullptr;
  size_t b = 0;
  switch (which) {
    case B200DQN_PTR_SCREENS: p = r->d_screens; b = size_t(r->size) * r->frame_bytes; break;
    case B200DQN_PTR_ACTIONS: p = r->d_actions; b = r->size; break;
    case B200DQN_PTR_REWARDS: p = r->d_rewards; b = r->size * sizeof(int64_t); break;
    case B200DQN_PTR_TERMINALS: p = r->d_terminals; b = r->size; break;
    case B200DQN_PTR_PRESTATES: p = r->d_pre; b = state_bytes; break;
    case B200DQN_PTR_POSTSTATES: p = r->d_post; b = state_bytes; break;
    case B200DQN_PTR_MB_ACTIONS: p = r->d_mb_actions; b = r->batch; break;
    case B200DQN_PTR_MB_REWARDS: p = r->d_mb_rewards; b = size_t(r->batch) * r->nstep * sizeof(int64_t); break;
    case B200DQN_PTR_MB_TERMINALS: p = r->d_mb_terminals; b = size_t(r->batch) * r->nstep; break;
    case B200DQN_PTR_INDEXES: p = r->d_idx; b = r->batch * sizeof(int32_t); break;
    case B200DQN_PTR_WORDS_CONSUMED: p = r->d_words; b = 2 * sizeof(uint32_t); break;
    case B200DQN_PTR_MT_STATE: p = r->mt_slot_ptr(); b = 625 * sizeof(uint32_t); break;
    case B200DQN_PTR_PRIORITIES: p = r->d_prio; b = r->d_prio ? r->size * sizeof(double) : 0; break;
    case B200DQN_PTR_SUM_TREE: p = r->d_sum; b = r->d_sum ? r->per_off[r->per_nlev] * sizeof(double) : 0; break;
    case B200DQN_PTR_IS_WEIGHTS: p = r->d_isw; b = r->d_isw ? r->batch * sizeof(float) : 0; break;
    case B200DQN_PTR_MAX_PRIORITY: p = r->d_maxp; b = r->d_maxp ? sizeof(double) : 0; break;
    case B200DQN_PTR_MIN_TREE:
      p = r->d_min;
      b = r->d_min ? (r->per_off[r->per_nlev] - r->per_off[1]) * sizeof(double) : 0;
      break;
    default: B2_REQUIRE(false, B200DQN_EINVAL, "replay_device_ptr: unknown selector %d", which);
  }
  *dev_ptr = p;
  if (bytes) *bytes = b;
  return B200DQN_OK;
}

// ============================================================================ C ABI: state window
extern "C" int b200dqn_statebuf_create(int device, int screen_h, int screen_w, int history_length, int batch_size,
                                       b200dqn_statebuf** out) {
  B2_REQUIRE(out && screen_h > 0 && screen_w > 0 && history_length > 0 && batch_size > 0, B200DQN_EINVAL,
             "statebuf_create: bad argument");
  DeviceGuard g(device);
  auto* s = new (std::nothrow) b200dqn_statebuf();
  B2_REQUIRE(s, B200DQN_EINVAL, "out of host memory");
  s->device = device;
  s->h = screen_h;
  s->w = screen_w;
  s->hist = history_length;
  s->batch = batch_size;
  s->frame_bytes = int64_t(screen_h) * screen_w;
  const size_t bytes = size_t(batch_size) * history_length * s->frame_bytes;
  B2_CHECK_CUDA(cudaMalloc(&s->d_buf, bytes + size_t(b200dqn_statebuf::kSlots) * s->frame_bytes));
  B2_CHECK_CUDA(cudaMemset(s->d_buf, 0, bytes));
  B2_CHECK_CUDA(cudaMallocHost(&s->h_stage, size_t(b200dqn_statebuf::kSlots) * s->frame_bytes));
  for (int i = 0; i < b200dqn_statebuf::kSlots; ++i)
    B2_CHECK_CUDA(cudaEventCreateWithFlags(&s->slot_done[i], cudaEventDisableTiming));
  *out = s;
  return B200DQN_OK;
}

extern "C" int b200dqn_statebuf_destroy(b200dqn_statebuf* s) {
  if (!s) return B200DQN_OK;
  DeviceGuard g(s->device);
  cudaDeviceSynchronize();
  cudaFree(s->d_buf);
  cudaFreeHost(s->h_stage);
  for (auto& e : s->slot_done) if (e) cudaEventDestroy(e);
  delete s;
  return B200DQN_OK;
}

extern "C" int b200dqn_statebuf_add(b200dqn_statebuf* s, const uint8_t* host_screen, void* stream) {
  B2_REQUIRE(s && host_screen, B200DQN_EINVAL, "statebuf_add: null argument");
  DeviceGuard g(s->device);
  cudaStream_t st = as_stream(stream);
  const int slot = s->next_slot;
  s->next_slot = (slot + 1) % b200dqn_statebuf::kSlots;
  B2_CHECK_CUDA(cudaEventSynchronize(s->slot_done[slot]));
  uint8_t* stage = s->h_stage + size_t(slot) * s->frame_bytes;
  memcpy(stage, host_screen, s->frame_bytes);
  const size_t bytes = size_t(s->batch) * s->hist * s->frame_bytes;
  uint8_t* d_fresh = s->d_buf + bytes + size_t(slot) * s->frame_bytes;  // device landing slot
  B2_CHECK_CUDA(cudaMemcpyAsync(d_fresh, stage, s->frame_bytes, cudaMemcpyHostToDevice, st));
  B2_CHECK_CUDA(cudaEventRecord(s->slot_done[slot], st));
  if (s->frame_bytes % 16 == 0) {
    const int64_t n = s->frame_bytes / 16;
    k_statebuf_shift<uint4><<<unsigned((n + 127) / 128), 128, 0, st>>>(
        reinterpret_cast<uint4*>(s->d_buf), reinterpret_cast<const uint4*>(d_fresh), s->hist, n);
  } else {
    const int64_t n = s->frame_bytes;
    k_statebuf_shift<uint8_t><<<unsigned((n + 255) / 256), 256, 0, st>>>(s->d_buf, d_fresh, s->hist, n);
  }
  B2_LAUNCH_CHECK();
  return B200DQN_OK;
}

extern "C" int b200dqn_statebuf_reset(b200dqn_statebuf* s, void* stream) {
  B2_REQUIRE(s, B200DQN_EINVAL, "null statebuf");
  DeviceGuard g(s->device);
  B2_CHECK_CUDA(cudaMemsetAsync(s->d_buf, 0, size_t(s->batch) * s->hist * s->frame_bytes, as_stream(stream)));
  return B200DQN_OK;
}

extern "C" int b200dqn_statebuf_read(b200dqn_statebuf* s, uint8_t* host_out, int whole, void* stream) {
  B2_REQUIRE(s && host_out, B200DQN_EINVAL, "statebuf_read: null argument");
  DeviceGuard g(s->device);
  cudaStream_t st = as_stream(stream);
  const size_t bytes = size_t(whole ? s->batch : 1) * s->hist * s->frame_bytes;
  B2_CHECK_CUDA(cudaMemcpyAsync(host_out, s->d_buf, bytes, cudaMemcpyDeviceToHost, st));
  B2_CHECK_CUDA(cudaStreamSynchronize(st));
  return B200DQN_OK;
}

extern "C" int b200dqn_statebuf_device_ptr(b200dqn_statebuf* s, void** dev_ptr, size_t* bytes) {
  B2_REQUIRE(s && dev_ptr, B200DQN_EINVAL, "statebuf_device_ptr: null argument");
  *dev_ptr = s->d_buf;
  if (bytes) *bytes = size_t(s->batch) * s->hist * s->frame_bytes;
  return B200DQN_OK;
}
