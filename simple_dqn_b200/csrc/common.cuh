// common.cuh — error plumbing and small PTX helpers shared by every translation unit of
// libb200dqn.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/b200dqn.h"

namespace b200 {

void set_error(const char* fmt, ...);

#define B2_CHECK_CUDA(expr)                                                               \
  do {                                                                                    \
    cudaError_t e__ = (expr);                                                             \
    if (e__ != cudaSuccess) {                                                             \
      ::b200::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(e__)); \
      return B200DQN_ECUDA;                                                               \
    }                                                                                     \
  } while (0)

#define B2_REQUIRE(cond, code, ...)      \
  do {                                   \
    if (!(cond)) {                       \
      ::b200::set_error(__VA_ARGS__);    \
      return (code);                     \
    }                                    \
  } while (0)

#define B2_LAUNCH_CHECK() B2_CHECK_CUDA(cudaGetLastError())

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
    else prev = -1;
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

static inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// Results the host waits for (cost of a train step, MT words a sampling consumed) are written by the producing
// kernel straight into host-mapped pinned memory: [0] = a sequence number published last (after a system fence).
// The host polls that word — no memcpy, no cudaStreamSynchronize — and checks the stream every ~1k spins so that a
// failed launch turns into an error instead of a spin forever.
int poll_mapped_seq(const volatile uint32_t* seq, uint32_t want, cudaStream_t st, const char* what);

// Per-launch CUDA-event profiler (b200dqn_profile_begin/_end): when armed, every launch site
// drops an event on its stream right after the kernel, labelled with the kernel's role.
void prof_mark(const char* label, cudaStream_t st);
extern bool g_prof_on;
#define B2_PROF(label, st)                         \
  do {                                             \
    if (::b200::g_prof_on) ::b200::prof_mark(label, st); \
  } while (0)

// In-graph kernel timeline (b200dqn_ktrace_begin/_end): when armed, every instrumented launch gets a
// slot; each CTA's thread 0 folds its %globaltimer into [min start, max end] of that slot.  Unlike the
// event profiler this works inside the replayed CUDA graph with all branches and PDL overlap live.
struct KTrace {
  unsigned long long* buf;   // [slot][2] = {start_ns, end_ns}; nullptr = off
  int slot;
};
KTrace ktrace_slot(const char* label);   // host: slot for this launch (registers the label), {nullptr,0} when off
extern int g_ktrace_gen;                 // bumped whenever tracing is switched, invalidates captured graphs
bool ktrace_tick(cudaStream_t st);       // host: count one fused step (first node of the step); true when gated

// ---------------------------------------------------------------- device-side PTX helpers
#ifdef __CUDACC__
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// Gate words behind the slots: [kKtGate] counts fused steps since arming (k_kt_tick), [kKtGate + 1] is the
// one step to record (0 = record everything) — lets a trace pick a steady-state step out of a batch.
constexpr int kKtCap = 128, kKtGate = 2 * kKtCap;
__device__ __forceinline__ bool kt_armed(const KTrace& kt) {
  if (!kt.buf || threadIdx.x != 0) return false;
  const unsigned long long want = kt.buf[kKtGate + 1];
  return want == 0 || *reinterpret_cast<volatile unsigned long long*>(kt.buf + kKtGate) == want;
}
__device__ __forceinline__ void kt_begin(const KTrace& kt) {
  if (kt_armed(kt)) atomicMin(kt.buf + 2 * kt.slot, globaltimer_ns());
}
__device__ __forceinline__ void kt_end(const KTrace& kt) {
  if (kt_armed(kt)) atomicMax(kt.buf + 2 * kt.slot + 1, globaltimer_ns());
}
extern bool g_use_pdl;   // B200DQN_NO_PDL unset
extern long long g_launch_count;   // every kernel launch of the library (bench.py's gpu_launches)

// Launch `kernel` with the programmatic-dependent-launch attribute (every kernel launched this way
// calls pdl_wait() before it touches data produced by earlier kernels).
// Side-branch launches (wgrad / optimizer / pack off the critical path) run inside this scope: they
// must NOT start early — an early-launched 200-CTA wgrad parks on every SM at its pdl_wait() and
// starves the critical-path kernels of shared memory — so they get ordinary full dependencies.
extern thread_local bool g_pdl_suppressed;
struct NoPdlScope {
  bool prev;
  NoPdlScope() : prev(g_pdl_suppressed) { g_pdl_suppressed = true; }
  ~NoPdlScope() { g_pdl_suppressed = prev; }
};

template <class... KArgs, class... Args>
static inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                     Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  int na = 0;
  if (g_use_pdl && !g_pdl_suppressed) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  ++g_launch_count;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// TMA 1-D bulk copy global -> shared (SASS: UBLKCP), completion on an mbarrier.
// dst/src 16-byte aligned, bytes a multiple of 16.
__device__ __forceinline__ void tma_bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// TMA 1-D bulk copy shared -> global, tracked by the bulk async-group.
__device__ __forceinline__ void tma_bulk_s2g(void* gmem_dst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst),
               "r"(smem_u32(smem_src)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void tma_bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void tma_bulk_wait_read_all() {
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
// until at most N of the most recently committed bulk groups still read their shared-memory source
template <int N>
__device__ __forceinline__ void tma_bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
// Programmatic dependent launch: a kernel launched with the programmatic-stream-serialization
// attribute may begin while its predecessor is still running; pdl_wait() blocks until every
// prerequisite grid has completed and flushed (no-op without the attribute), pdl_launch_dependents()
// lets the successor start its own prologue (barrier init, index setup) early.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
// generic-proxy writes -> visible to the async proxy (TMA / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
#endif  // __CUDACC__

}  // namespace b200
