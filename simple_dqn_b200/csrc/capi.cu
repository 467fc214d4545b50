// capi.cu — library-wide entry points: error text, version, device probe.
#include <stdarg.h>
#include <stdlib.h>

#include "common.cuh"

namespace b200 {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int poll_mapped_seq(const volatile uint32_t* seq, uint32_t want, cudaStream_t st, const char* what) {
  for (uint32_t spins = 1;; ++spins) {
    if (int32_t(*seq - want) >= 0) return B200DQN_OK;
    if ((spins & 0x3ffu) == 0) {
      const cudaError_t e = cudaStreamQuery(st);
      if (e == cudaSuccess) {              // the stream has drained: the value is there now or will never be
        if (int32_t(*seq - want) >= 0) return B200DQN_OK;
        B2_REQUIRE(false, B200DQN_ESTATE, "%s: the stream finished without publishing result %u (have %u)", what, want, *seq);
      }
      if (e != cudaErrorNotReady) {
        set_error("%s: %s", what, cudaGetErrorString(e));
        return B200DQN_ECUDA;
      }
    }
#if defined(__x86_64__)
    __builtin_ia32_pause();
#endif
  }
}

bool g_prof_on = false;
bool g_use_pdl = getenv("B200DQN_NO_PDL") == nullptr;
thread_local bool g_pdl_suppressed = false;
long long g_launch_count = 0;
namespace {
constexpr int kProfCap = 8192;
struct Prof {
  cudaEvent_t ev[kProfCap + 1];
  const char* label[kProfCap + 1];
  int n = 0;
  int created = 0;
  int device = 0;
} g_prof;
}  // namespace

int g_ktrace_gen = 0;
namespace {
struct KtState {
  unsigned long long* d_buf = nullptr;
  bool on = false, gated = false;
  int n = 0;
  char names[kKtCap][32];
} g_kt;
}  // namespace

KTrace ktrace_slot(const char* label) {
  if (!g_kt.on) return KTrace{nullptr, 0};
  // a gated trace records one step only, so launches of later steps (eager replay re-launches every kernel)
  // share the slot of their label instead of exhausting the table
  if (g_kt.gated)
    for (int i = 0; i < g_kt.n; ++i)
      if (strncmp(g_kt.names[i], label, 31) == 0) return KTrace{g_kt.d_buf, i};
  if (g_kt.n >= kKtCap) return KTrace{nullptr, 0};
  const int slot = g_kt.n++;
  strncpy(g_kt.names[slot], label, 31);
  g_kt.names[slot][31] = 0;
  return KTrace{g_kt.d_buf, slot};
}

__global__ void k_kt_tick(unsigned long long* buf) { buf[kKtGate] += 1; }
bool ktrace_tick(cudaStream_t st) {
  if (!g_kt.on || !g_kt.gated) return false;
  k_kt_tick<<<1, 1, 0, st>>>(g_kt.d_buf);
  return true;
}

void prof_mark(const char* label, cudaStream_t st) {
  if (g_prof.n >= kProfCap) return;
  const int i = ++g_prof.n;
  if (i >= g_prof.created) {
    cudaEventCreate(&g_prof.ev[i]);
    g_prof.created = i + 1;
  }
  g_prof.label[i] = label;
  cudaEventRecord(g_prof.ev[i], st);
}
}  // namespace b200

extern "C" int b200dqn_profile_begin(int device, void* stream) {
  using namespace b200;
  DeviceGuard g(device);
  if (g_prof.created == 0) {
    B2_CHECK_CUDA(cudaEventCreate(&g_prof.ev[0]));
    g_prof.created = 1;
  }
  g_prof.n = 0;
  g_prof.device = device;
  B2_CHECK_CUDA(cudaEventRecord(g_prof.ev[0], as_stream(stream)));
  g_prof_on = true;
  return B200DQN_OK;
}

extern "C" int b200dqn_profile_end(int max_entries, char* names32, float* ms, int* count) {
  using namespace b200;
  B2_REQUIRE(names32 && ms && count && max_entries > 0, B200DQN_EINVAL, "profile_end: bad argument");
  g_prof_on = false;
  DeviceGuard g(g_prof.device);
  B2_CHECK_CUDA(cudaDeviceSynchronize());
  const int n = g_prof.n < max_entries ? g_prof.n : max_entries;
  for (int i = 1; i <= n; ++i) {
    float t = 0.f;
    B2_CHECK_CUDA(cudaEventElapsedTime(&t, g_prof.ev[i - 1], g_prof.ev[i]));
    ms[i - 1] = t;
    strncpy(names32 + (i - 1) * 32, g_prof.label[i], 31);
    names32[(i - 1) * 32 + 31] = 0;
  }
  *count = n;
  return B200DQN_OK;
}

extern "C" const char* b200dqn_last_error(void) { return b200::g_err; }
extern "C" int b200dqn_version(void) { return B200DQN_VERSION; }

extern "C" int b200dqn_device_info(int device, int* sm_count, int* cc_major, int* cc_minor, size_t* free_bytes,
                                   size_t* total_bytes) {
  cudaDeviceProp prop;
  B2_CHECK_CUDA(cudaGetDeviceProperties(&prop, device));
  if (sm_count) *sm_count = prop.multiProcessorCount;
  if (cc_major) *cc_major = prop.major;
  if (cc_minor) *cc_minor = prop.minor;
  b200::DeviceGuard g(device);
  size_t f = 0, t = 0;
  B2_CHECK_CUDA(cudaMemGetInfo(&f, &t));
  if (free_bytes) *free_bytes = f;
  if (total_bytes) *total_bytes = t;
  B2_REQUIRE(prop.major == 9 && prop.minor == 0, B200DQN_ECUDA,
             "device %d is sm_%d%d; libb200dqn.so is built for sm_90a (H100) only", device, prop.major, prop.minor);
  return B200DQN_OK;
}

extern "C" int b200dqn_copy_to_host(int device, void* host_dst, const void* dev_src, size_t bytes, void* stream) {
  B2_REQUIRE(host_dst && dev_src, B200DQN_EINVAL, "copy_to_host: null argument");
  b200::DeviceGuard g(device);
  cudaStream_t st = b200::as_stream(stream);
  B2_CHECK_CUDA(cudaMemcpyAsync(host_dst, dev_src, bytes, cudaMemcpyDeviceToHost, st));
  B2_CHECK_CUDA(cudaStreamSynchronize(st));
  return B200DQN_OK;
}

extern "C" int b200dqn_copy_to_device(int device, void* dev_dst, const void* host_src, size_t bytes, void* stream) {
  B2_REQUIRE(dev_dst && host_src, B200DQN_EINVAL, "copy_to_device: null argument");
  b200::DeviceGuard g(device);
  cudaStream_t st = b200::as_stream(stream);
  B2_CHECK_CUDA(cudaMemcpyAsync(dev_dst, host_src, bytes, cudaMemcpyHostToDevice, st));
  B2_CHECK_CUDA(cudaStreamSynchronize(st));
  return B200DQN_OK;
}

extern "C" int b200dqn_stream_create(int device, void** out_stream) {
  B2_REQUIRE(out_stream, B200DQN_EINVAL, "stream_create: null argument");
  b200::DeviceGuard g(device);
  cudaStream_t st;
  B2_CHECK_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  *out_stream = st;
  return B200DQN_OK;
}

extern "C" int b200dqn_stream_destroy(int device, void* stream) {
  b200::DeviceGuard g(device);
  if (stream) B2_CHECK_CUDA(cudaStreamDestroy(b200::as_stream(stream)));
  return B200DQN_OK;
}

extern "C" int b200dqn_stream_synchronize(int device, void* stream) {
  b200::DeviceGuard g(device);
  B2_CHECK_CUDA(cudaStreamSynchronize(b200::as_stream(stream)));
  return B200DQN_OK;
}

extern "C" int b200dqn_ktrace_begin_at(int device, int step) {
  using namespace b200;
  B2_REQUIRE(step >= 0, B200DQN_EINVAL, "ktrace_begin_at: step must be >= 0");
  DeviceGuard g(device);
  if (!g_kt.d_buf) B2_CHECK_CUDA(cudaMalloc(&g_kt.d_buf, (kKtCap * 2 + 2) * sizeof(unsigned long long)));
  unsigned long long init[kKtCap * 2 + 2];
  for (int i = 0; i < kKtCap; ++i) { init[2 * i] = ~0ull; init[2 * i + 1] = 0ull; }
  init[kKtGate] = 0;
  init[kKtGate + 1] = (unsigned long long)step;
  B2_CHECK_CUDA(cudaMemcpy(g_kt.d_buf, init, sizeof(init), cudaMemcpyHostToDevice));
  g_kt.n = 0;
  g_kt.on = true;
  g_kt.gated = step > 0;
  ++g_ktrace_gen;
  return B200DQN_OK;
}
extern "C" int b200dqn_ktrace_begin(int device) { return b200dqn_ktrace_begin_at(device, 0); }

extern "C" int b200dqn_ktrace_end(int max_entries, char* names32, unsigned long long* start_ns,
                                  unsigned long long* end_ns, int* count) {
  using namespace b200;
  B2_REQUIRE(names32 && start_ns && end_ns && count, B200DQN_EINVAL, "ktrace_end: null argument");
  B2_CHECK_CUDA(cudaDeviceSynchronize());
  g_kt.on = false;
  ++g_ktrace_gen;
  unsigned long long host[kKtCap * 2];
  B2_CHECK_CUDA(cudaMemcpy(host, g_kt.d_buf, sizeof(host), cudaMemcpyDeviceToHost));
  const int n = g_kt.n < max_entries ? g_kt.n : max_entries;
  for (int i = 0; i < n; ++i) {
    memcpy(names32 + i * 32, g_kt.names[i], 32);
    start_ns[i] = host[2 * i];
    end_ns[i] = host[2 * i + 1];
  }
  *count = n;
  return B200DQN_OK;
}
