// comm.cu — data-parallel learners over NVLink 5 / NVSwitch: communicator set-up, the peer-memory exchange
// (kernels in comm_p2p.cuh: plane push + LL all-reduce of the default "gather" schedule, two-shot in-place
// all-reduce of the "layer"/"tail" schedules) and the NCCL path (bootstrap, votes, fallback).
// libnccl.so.2 is dlopen()ed (the process normally already holds torch's bundled copy), so the
// library has no link-time NCCL dependency and single-GPU use never touches it.
#include <dlfcn.h>
#include <unistd.h>

#include <algorithm>
#include <cstring>
#include <vector>

#define B200_COMM_P2P_KERNELS
#include "net.cuh"
#include "net_umma.cuh"

namespace b200 {

// Minimal NCCL ABI (nccl.h 2.x): opaque comm, 128-byte unique id, enums by value.
struct NcclUniqueId { char internal[128]; };
typedef void* ncclComm_t;
typedef int (*fn_GetUniqueId)(NcclUniqueId*);
typedef int (*fn_CommInitRank)(ncclComm_t*, int, NcclUniqueId, int);
typedef int (*fn_AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t);
typedef int (*fn_AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t);
typedef int (*fn_CommDestroy)(ncclComm_t);
typedef const char* (*fn_GetErrorString)(int);
constexpr int kNcclInt8 = 0;     // ncclInt8
constexpr int kNcclInt32 = 2;    // ncclInt32
constexpr int kNcclFloat32 = 7;  // ncclFloat32
constexpr int kNcclSum = 0;      // ncclSum

static struct {
  void* handle = nullptr;
  fn_GetUniqueId GetUniqueId = nullptr;
  fn_CommInitRank CommInitRank = nullptr;
  fn_AllReduce AllReduce = nullptr;
  fn_AllGather AllGather = nullptr;
  fn_CommDestroy CommDestroy = nullptr;
  fn_GetErrorString GetErrorString = nullptr;
} g_nccl;

static int nccl_load() {
  if (g_nccl.handle) return B200DQN_OK;
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  B2_REQUIRE(h, B200DQN_ENCCL, "cannot dlopen libnccl.so.2: %s", dlerror());
  g_nccl.GetUniqueId = (fn_GetUniqueId)dlsym(h, "ncclGetUniqueId");
  g_nccl.CommInitRank = (fn_CommInitRank)dlsym(h, "ncclCommInitRank");
  g_nccl.AllReduce = (fn_AllReduce)dlsym(h, "ncclAllReduce");
  g_nccl.AllGather = (fn_AllGather)dlsym(h, "ncclAllGather");
  g_nccl.CommDestroy = (fn_CommDestroy)dlsym(h, "ncclCommDestroy");
  g_nccl.GetErrorString = (fn_GetErrorString)dlsym(h, "ncclGetErrorString");
  B2_REQUIRE(g_nccl.GetUniqueId && g_nccl.CommInitRank && g_nccl.AllReduce && g_nccl.CommDestroy, B200DQN_ENCCL,
             "libnccl.so.2 lacks an expected symbol");
  g_nccl.handle = h;
  return B200DQN_OK;
}

#define B2_CHECK_NCCL(expr)                                                                      \
  do {                                                                                           \
    int r__ = (expr);                                                                            \
    if (r__ != 0) {                                                                              \
      set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr,                                     \
                g_nccl.GetErrorString ? g_nccl.GetErrorString(r__) : "nccl error");              \
      return B200DQN_ENCCL;                                                                      \
    }                                                                                            \
  } while (0)

// In-place all-reduce of layers [l0, l1] through peer memory (comm_p2p.cuh); `chan` names the call site.
int comm_xchg_range(b200dqn_net* n, int l0, int l1, int chan, cudaStream_t st, const char* label) {
  B2_REQUIRE(n->xchg_ok && chan >= 0 && chan < kXChannels, B200DQN_ESTATE, "peer exchange not initialised");
  XPeers pp{};
  for (int p = 0; p < n->world; ++p) {
    pp.g[p] = reinterpret_cast<float4*>(n->xg[p]);
    pp.flags[p] = n->xflags[p];
  }
  const int64_t off4 = n->lt.off[l0] / 4, n4 = (n->lt.off[l1 + 1] - n->lt.off[l0]) / 4;
  const int64_t chunk = (n4 + n->world - 1) / n->world, per_blk = kXThreads * kXUnroll;
  const int cap = n->xchg_blocks > 0 ? std::min(n->xchg_blocks, kXMaxBlocks) : kXMaxBlocks;
  const int nblk = int(std::min<int64_t>(cap, std::max<int64_t>(1, (chunk + per_blk - 1) / per_blk)));
  NoPdlScope plain;
  B2_CHECK_CUDA(launch_pdl(k_xchg, dim3(nblk), dim3(kXThreads), 0, st, pp, n->rank, n->world, chan, off4, n4,
                           n->d_xepoch, n->d_xerr, n->xchg_flags, ktrace_slot(label)));
  B2_PROF(label, st);
  return B200DQN_OK;
}

constexpr int kXCounterWords = kXChannels * kXMaxBlocks + 1 + 2 * kXChannels + 2 * kXPushChannels + 1;

// B200DQN_HEAD_PUSH=1: the head kernel pushes its dZ4 rows itself (counted arrivals).  OFF by default: parity-clean
// (tests/test_gpu_multi.py) but measured slower on two GPUs of an earlier generation (not re-measured on H100): the
// system-scope fence in front of the arrival counter keeps every head CTA on the critical chain.
bool comm_head_push(const b200dqn_net* n, cudaStream_t st, HeadPush* out) {
  static const bool enabled = getenv("B200DQN_HEAD_PUSH") && atoi(getenv("B200DQN_HEAD_PUSH")) != 0;
  if (!enabled || !comm_gather_active(n, st)) return false;
  if (out) {
    HeadPush h{};
    h.world = n->world; h.rank = n->rank; h.rows = n->nb;
    const int64_t mine = int64_t(n->nb) * kHidden * 2;     // bytes of this rank's rows in one plane
    for (int p = 0; p < n->world; ++p) {
      h.gat[p] = reinterpret_cast<uint4*>(n->xbuf[p] + n->x_dz_off);
      h.cnt[p] = reinterpret_cast<uint32_t*>(n->xbuf[p]) + kXCountWord;
    }
    h.parity16 = n->x_dz_parity / 16;
    h.lo16 = mine * n->world / 16;
    h.epoch = n->d_xpush_epoch + 1;
    *out = h;
  }
  return true;
}

// true when this train step uses the gather schedule (net.cu::backward_and_update_gather)
bool comm_gather_active(const b200dqn_net* n, cudaStream_t st) {
  return n->world > 1 && n->xchg_ok && n->xchg_sched == 2 && n->d_xbuf && !g_prof_on && n->use_branches &&
         st != nullptr && n->cfg.math_mode == B200DQN_MATH_TCGEN05;
}

// One-shot LL all-reduce of one layer's gradient (fc1 excluded: its operands are gathered instead), in place
// in d_g.  The layer IS the channel: a line's flag words only ever carry that layer's epoch sequence.
int comm_xll_args(b200dqn_net* n, int l, XllArgs* out) {
  B2_REQUIRE(n->xchg_ok && n->d_xbuf, B200DQN_ESTATE, "LL exchange not initialised");
  B2_REQUIRE(l >= 0 && l < kLayers && l != 3 && l < kXChannels, B200DQN_EINVAL, "LL exchange: layer must be 0, 1, 2 or 4");
  const int64_t fc1_4 = (n->lt.off[4] - n->lt.off[3]) / 4;
  XllArgs a{};
  for (int p = 0; p < n->world; ++p) a.recv[p] = reinterpret_cast<uint4*>(n->xbuf[p] + n->x_ll_off);
  a.g = reinterpret_cast<float4*>(n->d_g);
  a.rank = n->rank; a.world = n->world; a.chan = l;
  a.off4 = n->lt.off[l] / 4;
  a.ll4 = l > 3 ? a.off4 - fc1_4 : a.off4;
  a.n4 = (n->lt.off[l + 1] - n->lt.off[l]) / 4;
  a.lines_per_src = n->x_ll_lines;
  a.epoch = n->d_xll_epoch; a.ticket = n->d_xll_epoch + kXChannels; a.err = n->d_xerr;
  *out = a;
  return B200DQN_OK;
}

int comm_xll_layer(b200dqn_net* n, int l, cudaStream_t st, const char* label) {
  XllArgs a{};
  int rc_args = comm_xll_args(n, l, &a);
  if (rc_args) return rc_args;
  const int cap = n->xchg_blocks > 0 ? std::min(n->xchg_blocks, kXMaxBlocks) : 64;
  const int nblk = int(std::min<int64_t>(cap, std::max<int64_t>(1, (a.n4 + kXThreads - 1) / kXThreads)));
  NoPdlScope plain;
  B2_CHECK_CUDA(launch_pdl(k_xll, dim3(nblk), dim3(kXThreads), 0, st, a, ktrace_slot(label)));
  B2_PROF(label, st);
  return B200DQN_OK;
}

// Push this rank's rows of a hi/lo plane pair (chan 0: H3, 1: dZ4) into every rank's gather area.
int comm_push_planes(b200dqn_net* n, int chan, const void* hi, int64_t lo_off_elems, cudaStream_t st) {
  B2_REQUIRE(n->xchg_ok && n->d_xbuf && (chan == 0 || chan == 1), B200DQN_ESTATE, "plane push not initialised");
  const int64_t row_elems = chan == 0 ? kFlat : kHidden;
  const int64_t mine = int64_t(n->nb) * row_elems * 2;            // bytes of this rank's rows in one plane
  const int64_t plane = mine * n->world;                          // bytes of one gathered plane
  XPushArgs a{};
  a.src[0] = static_cast<const uint4*>(hi);
  a.src[1] = reinterpret_cast<const uint4*>(static_cast<const __half*>(hi) + lo_off_elems);
  a.n16 = mine / 16;
  a.dst16[0] = (int64_t(n->rank) * mine) / 16;
  a.dst16[1] = (plane + int64_t(n->rank) * mine) / 16;
  a.parity16 = (chan == 0 ? n->x_h3_parity : n->x_dz_parity) / 16;
  for (int p = 0; p < n->world; ++p) {
    a.gat[p] = reinterpret_cast<uint4*>(n->xbuf[p] + (chan == 0 ? n->x_h3_off : n->x_dz_off));
    a.pflags[p] = reinterpret_cast<uint32_t*>(n->xbuf[p]);
  }
  a.rank = n->rank; a.world = n->world; a.chan = chan;
  a.epoch = n->d_xpush_epoch; a.ticket = n->d_xpush_epoch + kXPushChannels;
  const int nblk = int(std::min<int64_t>(64, std::max<int64_t>(1, (2 * a.n16 + kXThreads - 1) / kXThreads)));
  NoPdlScope plain;
  const char* label = chan == 0 ? "push_h3" : "push_dz4";
  B2_CHECK_CUDA(launch_pdl(k_xpush, dim3(nblk), dim3(kXThreads), 0, st, a, ktrace_slot(label)));
  B2_PROF(label, st);
  return B200DQN_OK;
}

// dZ4 rows of every rank into the local gather area in the LL protocol (one kernel on every rank: push + collect);
// off with B200DQN_DZ_LL=0 (then: plain push + flag wait)
bool comm_dz4_ll_enabled() {
  static const bool enabled = !(getenv("B200DQN_DZ_LL") && atoi(getenv("B200DQN_DZ_LL")) == 0);
  return enabled;
}
int comm_gather_dz4_ll(b200dqn_net* n, const void* hi, int64_t lo_off_elems, cudaStream_t st, bool wait_h3) {
  B2_REQUIRE(n->xchg_ok && n->d_xbuf && n->x_dzll_lines > 0, B200DQN_ESTATE, "LL gather not initialised");
  XGatherLL a{};
  a.src[0] = static_cast<const uint4*>(hi);
  a.src[1] = reinterpret_cast<const uint4*>(static_cast<const __half*>(hi) + lo_off_elems);
  a.n16 = int64_t(n->nb) * kHidden * 2 / 16;
  for (int p = 0; p < n->world; ++p) a.recv[p] = reinterpret_cast<uint4*>(n->xbuf[p] + n->x_dzll_off);
  a.gather = reinterpret_cast<uint4*>(n->d_xbuf + n->x_dz_off);
  a.parity16 = n->x_dz_parity / 16;
  a.lo16 = a.n16 * n->world;
  a.lines_per_src = n->x_dzll_lines;
  a.rank = n->rank; a.world = n->world;
  a.epoch = n->d_xpush_epoch + 1; a.ticket = n->d_xpush_epoch + kXPushChannels + 1; a.err = n->d_xerr;
  a.h3_flags = wait_h3 ? reinterpret_cast<const uint32_t*>(n->d_xbuf) : nullptr;
  a.h3_epoch = n->d_xpush_epoch;
  const int nblk = int(std::min<int64_t>(64, std::max<int64_t>(1, (2 * a.n16 + kXThreads - 1) / kXThreads)));
  NoPdlScope plain;
  B2_CHECK_CUDA(launch_pdl(k_xgather_ll, dim3(nblk), dim3(kXThreads), 0, st, a, ktrace_slot("gather_dz4")));
  B2_PROF("gather_dz4", st);
  return B200DQN_OK;
}

// Block the stream until every rank's H3 and dZ4 rows of this step have landed in the local gather area.
int comm_wait_pushes(b200dqn_net* n, cudaStream_t st, int dz_rows) {
  B2_REQUIRE(n->xchg_ok && n->d_xbuf, B200DQN_ESTATE, "plane push not initialised");
  NoPdlScope plain;
  B2_CHECK_CUDA(launch_pdl(k_xwait, dim3(1), dim3(32), 0, st, reinterpret_cast<uint32_t*>(n->d_xbuf), n->d_xpush_epoch,
                           n->world, n->d_xerr, dz_rows, n->d_xpush_epoch + 2 * kXPushChannels,
                           ktrace_slot("wait_push")));
  B2_PROF("wait_push", st);
  return B200DQN_OK;
}

int comm_allreduce_grads(b200dqn_net* n, cudaStream_t st) {
  if (n->xchg_ok) return comm_xchg_range(n, 0, kLayers - 1, 4, st, "xchg_all");
  B2_REQUIRE(n->nccl_comm, B200DQN_ESTATE, "communicator not initialised");
  B2_CHECK_NCCL(g_nccl.AllReduce(n->d_g, n->d_g, size_t(n->n_params), kNcclFloat32, kNcclSum,
                                 (ncclComm_t)n->nccl_comm, st));
  return B200DQN_OK;
}

// all-reduce the summed gradients of layers [l0, l1] (contiguous in d_g) on stream st
int comm_allreduce_range(b200dqn_net* n, int l0, int l1, cudaStream_t st) {
  if (n->xchg_ok) return comm_xchg_range(n, l0, l1, l0, st, l0 >= 3 ? "xchg_fc" : "xchg_conv");
  B2_REQUIRE(n->nccl_comm, B200DQN_ESTATE, "communicator not initialised");
  float* p = n->d_g + n->lt.off[l0];
  const size_t cnt = size_t(n->lt.off[l1 + 1] - n->lt.off[l0]);
  B2_CHECK_NCCL(g_nccl.AllReduce(p, p, cnt, kNcclFloat32, kNcclSum, (ncclComm_t)n->nccl_comm, st));
  return B200DQN_OK;
}

static void xchg_close(b200dqn_net* n) {
  for (int p = 0; p < kXMaxWorld; ++p) {
    if (n->xopened[p]) cudaIpcCloseMemHandle(n->xopened[p]);
    n->xopened[p] = nullptr;
    n->xg[p] = nullptr;
    n->xflags[p] = nullptr;
    if (n->xbuf_opened[p]) cudaIpcCloseMemHandle(n->xbuf_opened[p]);
    n->xbuf_opened[p] = nullptr;
    n->xbuf[p] = nullptr;
  }
  if (n->d_xbuf) cudaFree(n->d_xbuf);
  n->d_xbuf = nullptr;
  n->xchg_ok = false;
}

// What each rank publishes about its gradient buffer.
struct XRecord {
  cudaIpcMemHandle_t handle;    // d_g (+ flag words), 64 bytes
  cudaIpcMemHandle_t handle2;   // d_xbuf
  uint64_t pid, ptr, ptr2;
  int32_t device, want;
};

// Map every peer's gradient buffer, agree on the outcome, prove the path with a known-answer exchange.
// Leaves n->xchg_ok false (NCCL keeps doing the reductions) when any rank cannot take part.
static int xchg_setup(b200dqn_net* n, cudaStream_t ws) {
  const int W = n->world;
  ncclComm_t comm = (ncclComm_t)n->nccl_comm;
  const char* mode = getenv("B200DQN_COMM");
  const char* sched = getenv("B200DQN_P2P_SCHED");
  n->xchg_sched = !sched ? 2 : !strcmp(sched, "tail") ? 0 : !strcmp(sched, "layer") ? 1 : 2;
  if (const char* f = getenv("B200DQN_XCHG_FLAGS")) n->xchg_flags = atoi(f) & (kXStrongLoads | kXStrongStores);
  if (const char* f = getenv("B200DQN_XCHG_BLOCKS")) n->xchg_blocks = atoi(f);
  XRecord mine{};
  bool want = W >= 2 && W <= kXMaxWorld && g_nccl.AllGather && !(mode && !strcmp(mode, "nccl"));
  if (want && cudaIpcGetMemHandle(&mine.handle, n->d_g) != cudaSuccess) {
    cudaGetLastError();
    want = false;
  }
  // second shared allocation: push flags, LL lines, gather areas (layout identical on every rank)
  auto up = [](int64_t v) { return (v + 255) / 256 * 256; };
  const int64_t fc1_4 = (n->lt.off[4] - n->lt.off[3]) / 4;
  n->x_ll_lines = 2 * (n->n_params / 4 - fc1_4);
  n->x_ll_off = 4096;
  n->x_h3_lo = int64_t(W) * n->nb * kFlat;
  n->x_h3_parity = 2 * n->x_h3_lo * 2;
  n->x_h3_off = up(n->x_ll_off + 2 * int64_t(W) * n->x_ll_lines * 16);
  n->x_dz_lo = int64_t(W) * n->nb * kHidden;
  n->x_dz_parity = 2 * n->x_dz_lo * 2;
  n->x_dz_off = up(n->x_h3_off + 2 * n->x_h3_parity);
  n->x_dzll_off = up(n->x_dz_off + 2 * n->x_dz_parity);
  n->x_dzll_lines = 4 * (int64_t(n->nb) * kHidden * 2 / 16);
  const int64_t xbytes = up(n->x_dzll_off + 2 * int64_t(W) * n->x_dzll_lines * 16);
  if (want) {
    if (cudaMalloc(&n->d_xbuf, xbytes) != cudaSuccess || cudaMemsetAsync(n->d_xbuf, 0, xbytes, ws) != cudaSuccess ||
        cudaIpcGetMemHandle(&mine.handle2, n->d_xbuf) != cudaSuccess) {
      cudaGetLastError();
      want = false;
    }
  }
  mine.pid = uint64_t(getpid());
  mine.ptr = uint64_t(reinterpret_cast<uintptr_t>(n->d_g));
  mine.ptr2 = uint64_t(reinterpret_cast<uintptr_t>(n->d_xbuf));
  mine.device = n->device;
  mine.want = want ? 1 : 0;
  if (!g_nccl.AllGather) return B200DQN_OK;   // every rank loads the same library: nobody exchanges records

  // fresh flag words and epochs for this communicator, ordered before our record leaves
  B2_CHECK_CUDA(cudaMemsetAsync(n->d_xflags, 0, kXFlagWords * sizeof(uint32_t), ws));
  B2_CHECK_CUDA(cudaMemsetAsync(n->d_xepoch, 0, kXCounterWords * sizeof(uint32_t), ws));
  char* d_rec = nullptr;
  B2_CHECK_CUDA(cudaMalloc(&d_rec, size_t(W) * sizeof(XRecord) + sizeof(int32_t)));
  struct Free { char* p; ~Free() { cudaFree(p); } } free_rec{d_rec};
  B2_CHECK_CUDA(cudaMemcpyAsync(d_rec + size_t(n->rank) * sizeof(XRecord), &mine, sizeof(XRecord), cudaMemcpyHostToDevice, ws));
  B2_CHECK_NCCL(g_nccl.AllGather(d_rec + size_t(n->rank) * sizeof(XRecord), d_rec, sizeof(XRecord), kNcclInt8, comm, ws));
  std::vector<XRecord> rec(W);
  B2_CHECK_CUDA(cudaMemcpyAsync(rec.data(), d_rec, size_t(W) * sizeof(XRecord), cudaMemcpyDeviceToHost, ws));
  B2_CHECK_CUDA(cudaStreamSynchronize(ws));

  int32_t ok = 1;
  for (int p = 0; p < W; ++p) ok &= rec[p].want;
  for (int p = 0; p < W && ok; ++p) {
    float* base = nullptr;
    uint8_t* base2 = nullptr;
    if (p == n->rank) {
      base = n->d_g;
      base2 = n->d_xbuf;
    } else if (rec[p].pid == mine.pid) {   // learners sharing one process: plain peer access
      int can = 0;
      if (cudaDeviceCanAccessPeer(&can, n->device, rec[p].device) != cudaSuccess || !can) ok = 0;
      else {
        cudaError_t e = cudaDeviceEnablePeerAccess(rec[p].device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) ok = 0;
        cudaGetLastError();
        base = reinterpret_cast<float*>(uintptr_t(rec[p].ptr));
        base2 = reinterpret_cast<uint8_t*>(uintptr_t(rec[p].ptr2));
      }
    } else {
      void* mapped = nullptr, *mapped2 = nullptr;
      if (cudaIpcOpenMemHandle(&mapped, rec[p].handle, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
        cudaGetLastError();
        ok = 0;
      } else {
        n->xopened[p] = mapped;
        base = static_cast<float*>(mapped);
        if (cudaIpcOpenMemHandle(&mapped2, rec[p].handle2, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
          cudaGetLastError();
          ok = 0;
        } else {
          n->xbuf_opened[p] = mapped2;
          base2 = static_cast<uint8_t*>(mapped2);
        }
      }
    }
    if (ok) {
      n->xg[p] = base;
      n->xflags[p] = reinterpret_cast<uint32_t*>(base + n->n_params);
      n->xbuf[p] = base2;
    }
  }
  // every rank must take the same path
  int32_t* d_ok = reinterpret_cast<int32_t*>(d_rec + size_t(W) * sizeof(XRecord));
  B2_CHECK_CUDA(cudaMemcpyAsync(d_ok, &ok, sizeof(ok), cudaMemcpyHostToDevice, ws));
  B2_CHECK_NCCL(g_nccl.AllReduce(d_ok, d_ok, 1, kNcclInt32, kNcclSum, comm, ws));
  int32_t n_ok = 0;
  B2_CHECK_CUDA(cudaMemcpyAsync(&n_ok, d_ok, sizeof(n_ok), cudaMemcpyDeviceToHost, ws));
  B2_CHECK_CUDA(cudaStreamSynchronize(ws));
  if (n_ok != W) {
    xchg_close(n);
    return B200DQN_OK;
  }
  n->xchg_ok = true;

  // known-answer exchange outside any capture: element i of every rank's buffer = rank + 1 + i
  const int64_t kat = std::min<int64_t>(n->n_params, 1 << 16);
  std::vector<float> h(kat);
  for (int64_t i = 0; i < kat; ++i) h[i] = float(n->rank + 1) + float(i & 1023);
  B2_CHECK_CUDA(cudaMemcpyAsync(n->d_g, h.data(), kat * sizeof(float), cudaMemcpyHostToDevice, ws));
  int rc = comm_xchg_range(n, 0, kLayers - 1, 5, ws, "xchg_kat");
  if (rc) return rc;
  B2_CHECK_CUDA(cudaMemcpyAsync(h.data(), n->d_g, kat * sizeof(float), cudaMemcpyDeviceToHost, ws));
  uint32_t err = 0;
  B2_CHECK_CUDA(cudaMemcpyAsync(&err, n->d_xerr, sizeof(err), cudaMemcpyDeviceToHost, ws));
  B2_CHECK_CUDA(cudaStreamSynchronize(ws));
  bool good = err == 0;
  for (int64_t i = 0; i < kat && good; ++i) good = h[i] == float(W * (W + 1) / 2) + float(W) * float(i & 1023);
  B2_CHECK_CUDA(cudaMemsetAsync(n->d_g, 0, n->n_params * sizeof(float), ws));
  B2_CHECK_CUDA(cudaStreamSynchronize(ws));
  // A failed known-answer test must not leave the ranks on different paths: agree, then all fall back to NCCL.
  auto agree = [&](bool mine_ok, const char* what) -> int {
    int32_t v = mine_ok ? 1 : 0, sum = 0;
    B2_CHECK_CUDA(cudaMemcpyAsync(d_ok, &v, sizeof(v), cudaMemcpyHostToDevice, ws));
    B2_CHECK_NCCL(g_nccl.AllReduce(d_ok, d_ok, 1, kNcclInt32, kNcclSum, comm, ws));
    B2_CHECK_CUDA(cudaMemcpyAsync(&sum, d_ok, sizeof(sum), cudaMemcpyDeviceToHost, ws));
    B2_CHECK_CUDA(cudaStreamSynchronize(ws));
    if (sum == W) return B200DQN_OK;
    fprintf(stderr, "b200dqn: rank %d: %s failed its known-answer test on %d of %d ranks (local: %s, err word %u); "
                    "gradients will go through NCCL\n", n->rank, what, W - sum, W, mine_ok ? "ok" : "FAILED", err);
    B2_CHECK_CUDA(cudaMemsetAsync(n->d_xerr, 0, sizeof(uint32_t), ws));
    B2_CHECK_CUDA(cudaStreamSynchronize(ws));
    xchg_close(n);
    return 1;
  };
  if ((rc = agree(good, "the two-shot peer-memory exchange"))) return rc < 0 ? rc : B200DQN_OK;

  // known-answer tests of the LL all-reduce (conv1..3, fc2) and of the plane push, same pattern
  {
    std::vector<float> hp(n->n_params);
    for (int64_t i = 0; i < n->n_params; ++i) hp[i] = float(n->rank + 1) + float(i & 1023);
    B2_CHECK_CUDA(cudaMemcpyAsync(n->d_g, hp.data(), n->n_params * sizeof(float), cudaMemcpyHostToDevice, ws));
    for (int l = 0; l < kLayers; ++l)
      if (l != 3 && (rc = comm_xll_layer(n, l, ws, "xll_kat"))) return rc;
    B2_CHECK_CUDA(cudaMemcpyAsync(hp.data(), n->d_g, n->n_params * sizeof(float), cudaMemcpyDeviceToHost, ws));
    const int64_t mine_h3 = int64_t(n->nb) * kFlat * 2, mine_dz = int64_t(n->nb) * kHidden * 2;
    uint8_t* tmp = nullptr;
    B2_CHECK_CUDA(cudaMalloc(&tmp, 2 * mine_h3));
    struct FreeT { uint8_t* p; ~FreeT() { cudaFree(p); } } free_tmp{tmp};
    B2_CHECK_CUDA(cudaMemsetAsync(tmp, n->rank + 1, 2 * mine_h3, ws));
    if ((rc = comm_push_planes(n, 0, tmp, mine_h3 / 2, ws))) return rc;
    if ((rc = comm_push_planes(n, 1, tmp, mine_dz / 2, ws))) return rc;
    if ((rc = comm_wait_pushes(n, ws))) return rc;
    std::vector<uint8_t> hh(n->x_h3_parity), hd(n->x_dz_parity);   // epoch 1 -> parity 1
    B2_CHECK_CUDA(cudaMemcpyAsync(hh.data(), n->d_xbuf + n->x_h3_off + n->x_h3_parity, hh.size(), cudaMemcpyDeviceToHost, ws));
    B2_CHECK_CUDA(cudaMemcpyAsync(hd.data(), n->d_xbuf + n->x_dz_off + n->x_dz_parity, hd.size(), cudaMemcpyDeviceToHost, ws));
    B2_CHECK_CUDA(cudaMemcpyAsync(&err, n->d_xerr, sizeof(err), cudaMemcpyDeviceToHost, ws));
    B2_CHECK_CUDA(cudaStreamSynchronize(ws));
    bool ll_ok = err == 0, push_ok = err == 0;
    for (int64_t i = 0; i < n->n_params && ll_ok; ++i) {
      const bool fc1 = i >= n->lt.off[3] && i < n->lt.off[4];
      const float expect = fc1 ? float(n->rank + 1) + float(i & 1023) : float(W * (W + 1) / 2) + float(W) * float(i & 1023);
      ll_ok = hp[i] == expect;
    }
    for (int pl = 0; pl < 2 && push_ok; ++pl)
      for (int p = 0; p < W && push_ok; ++p) {
        for (int64_t i = 0; i < mine_h3 && push_ok; ++i) push_ok = hh[(int64_t(pl) * W + p) * mine_h3 + i] == uint8_t(p + 1);
        for (int64_t i = 0; i < mine_dz && push_ok; ++i) push_ok = hd[(int64_t(pl) * W + p) * mine_dz + i] == uint8_t(p + 1);
      }
    // the LL gather of dZ4 (second dZ4 epoch -> parity 0 of the plain area)
    bool gat_ok = true;
    if (comm_dz4_ll_enabled()) {
      if ((rc = comm_gather_dz4_ll(n, tmp, mine_dz / 2, ws, true))) return rc;
      std::vector<uint8_t> hg(n->x_dz_parity);
      B2_CHECK_CUDA(cudaMemcpyAsync(hg.data(), n->d_xbuf + n->x_dz_off, hg.size(), cudaMemcpyDeviceToHost, ws));
      B2_CHECK_CUDA(cudaMemcpyAsync(&err, n->d_xerr, sizeof(err), cudaMemcpyDeviceToHost, ws));
      B2_CHECK_CUDA(cudaStreamSynchronize(ws));
      gat_ok = err == 0;
      for (int pl = 0; pl < 2 && gat_ok; ++pl)
        for (int p = 0; p < W && gat_ok; ++p)
          for (int64_t i = 0; i < mine_dz && gat_ok; ++i) gat_ok = hg[(int64_t(pl) * W + p) * mine_dz + i] == uint8_t(p + 1);
    }
    B2_CHECK_CUDA(cudaMemsetAsync(n->d_g, 0, n->n_params * sizeof(float), ws));
    B2_CHECK_CUDA(cudaStreamSynchronize(ws));
    if ((rc = agree(ll_ok && push_ok && gat_ok, !ll_ok ? "the LL all-reduce" : !push_ok ? "the plane push" : "the LL gather")))
      return rc < 0 ? rc : B200DQN_OK;
  }
  return B200DQN_OK;
}

void comm_destroy(b200dqn_net* n) {
  xchg_close(n);
  if (n->nccl_comm && g_nccl.CommDestroy) g_nccl.CommDestroy((ncclComm_t)n->nccl_comm);
  n->nccl_comm = nullptr;
  n->world = 1;
  n->rank = 0;
}

}  // namespace b200

using namespace b200;

extern "C" int b200dqn_comm_unique_id(void* out_id128) {
  B2_REQUIRE(out_id128, B200DQN_EINVAL, "null id buffer");
  int rc = nccl_load();
  if (rc) return rc;
  NcclUniqueId id;
  B2_CHECK_NCCL(g_nccl.GetUniqueId(&id));
  memcpy(out_id128, &id, sizeof(id));
  return B200DQN_OK;
}

extern "C" int b200dqn_net_comm_init(b200dqn_net* n, const void* id128, int rank, int world_size) {
  B2_REQUIRE(n && id128 && world_size >= 1 && rank >= 0 && rank < world_size, B200DQN_EINVAL,
             "net_comm_init: bad argument");
  B2_REQUIRE(!n->nccl_comm, B200DQN_ESTATE, "net_comm_init: communicator already initialised");
  // conv1's exchange (k_opt_conv<..., XCHG>, the LL line counts) has only been validated for 4-frame windows
  B2_REQUIRE(n->cfg.history_length == kHist, B200DQN_ENOTIMPL,
             "net_comm_init: data-parallel learners are implemented for history_length %d only (got %d)", kHist,
             n->cfg.history_length);
  // the data-parallel schedules exchange and gather the two-slot forward's tensors only
  B2_REQUIRE(!n->double_q, B200DQN_ENOTIMPL,
             "net_comm_init: the Double DQN target is implemented for a single learner only (switch double Q off first)");
  B2_REQUIRE(!n->d_td_err, B200DQN_ENOTIMPL,
             "net_comm_init: prioritized replay is implemented for a single learner only (this net has trained from a "
             "prioritized ring)");
  B2_REQUIRE(!n->atoms, B200DQN_ENOTIMPL,
             "net_comm_init: the distributional head is implemented for a single learner only");
  B2_REQUIRE(!n->dueling, B200DQN_ENOTIMPL, "net_comm_init: the dueling network is implemented for a single learner only");
  B2_REQUIRE(!n->quantiles, B200DQN_ENOTIMPL,
             "net_comm_init: the quantile-regression head is implemented for a single learner only");
  B2_REQUIRE(!n->munchausen, B200DQN_ENOTIMPL,
             "net_comm_init: the Munchausen target is implemented for a single learner only");
  B2_REQUIRE(!n->fqf_n, B200DQN_ENOTIMPL, "net_comm_init: the FQF head is implemented for a single learner only");
  B2_REQUIRE(!n->iqn_n, B200DQN_ENOTIMPL, "net_comm_init: the IQN head is implemented for a single learner only");
  B2_REQUIRE(!n->boot, B200DQN_ENOTIMPL,
             "net_comm_init: bootstrapped heads are implemented for a single learner only");
  B2_REQUIRE(!n->rem_k, B200DQN_ENOTIMPL, "net_comm_init: the REM head is implemented for a single learner only");
  B2_REQUIRE(!n->clip, B200DQN_ENOTIMPL,
             "net_comm_init: gradient-norm clipping is implemented for a single learner only");
  B2_REQUIRE(!n->soft, B200DQN_ENOTIMPL,
             "net_comm_init: the soft target update is implemented for a single learner only");
  B2_REQUIRE(!n->crop_pad, B200DQN_ENOTIMPL,
             "net_comm_init: random-shift augmentation is implemented for a single learner only");
  B2_REQUIRE(n->ring_nstep == 1, B200DQN_ENOTIMPL,
             "net_comm_init: n-step returns are implemented for a single learner only (this net last trained from a "
             "ring with n_step %d)", n->ring_nstep);
  int rc = nccl_load();
  if (rc) return rc;
  DeviceGuard g(n->device);
  NcclUniqueId id;
  memcpy(&id, id128, sizeof(id));
  ncclComm_t comm = nullptr;
  B2_CHECK_NCCL(g_nccl.CommInitRank(&comm, world_size, id, rank));
  n->nccl_comm = comm;
  n->rank = rank;
  n->world = world_size;
  // Warm-up collective outside any capture: NCCL sets up its channels/proxies lazily on the first call,
  // which must not happen inside the CUDA-graph capture of the train step.
  cudaStream_t ws;
  B2_CHECK_CUDA(cudaStreamCreateWithFlags(&ws, cudaStreamNonBlocking));
  B2_CHECK_CUDA(cudaMemsetAsync(n->d_g, 0, n->n_params * sizeof(float), ws));
  B2_CHECK_NCCL(g_nccl.AllReduce(n->d_g, n->d_g, size_t(n->n_params), kNcclFloat32, kNcclSum, comm, ws));
  B2_CHECK_CUDA(cudaStreamSynchronize(ws));
  rc = xchg_setup(n, ws);
  cudaStreamDestroy(ws);
  return rc;
}

// Developer aid: time `iters` back-to-back exchanges of layers [l0, l1] with the given k_xchg switches and
// CTA cap on a private stream (every rank must make the same call); *us_out = mean microseconds per exchange,
// *ok_out = the exchange reproduced the known answer (meaningless with the diagnosis-only switches).
extern "C" int b200dqn_debug_xchg(b200dqn_net* n, int l0, int l1, int flags, int blocks, int iters, float* us_out,
                                  int* ok_out) {
  B2_REQUIRE(n && us_out && ok_out && l0 >= 0 && l1 < kLayers && l0 <= l1 && iters >= 1, B200DQN_EINVAL,
             "debug_xchg: bad argument");
  B2_REQUIRE(n->xchg_ok, B200DQN_ESTATE, "debug_xchg: peer exchange not initialised");
  DeviceGuard g(n->device);
  const int keep_flags = n->xchg_flags, keep_blocks = n->xchg_blocks;
  const bool ll = (flags & 16) != 0;   // time the one-shot LL all-reduce instead of the two-shot exchange
  B2_REQUIRE(!ll || (n->d_xbuf && l0 == l1 && l0 != 3), B200DQN_EINVAL, "debug_xchg: LL takes one of layers 0, 1, 2, 4");
  auto exchange = [&](cudaStream_t s) {
    return ll ? comm_xll_layer(n, l0, s, "xll_dbg") : comm_xchg_range(n, l0, l1, 5, s, "xchg_dbg");
  };
  n->xchg_flags = flags & 15;
  n->xchg_blocks = blocks;
  cudaStream_t ws;
  cudaEvent_t e0, e1;
  B2_CHECK_CUDA(cudaStreamCreateWithFlags(&ws, cudaStreamNonBlocking));
  B2_CHECK_CUDA(cudaEventCreate(&e0));
  B2_CHECK_CUDA(cudaEventCreate(&e1));
  const int64_t off = n->lt.off[l0], cnt = n->lt.off[l1 + 1] - off;
  const int W = n->world;
  std::vector<float> h(cnt);
  for (int64_t i = 0; i < cnt; ++i) h[i] = float(n->rank + 1) + float(i & 1023);
  B2_CHECK_CUDA(cudaMemcpyAsync(n->d_g + off, h.data(), cnt * sizeof(float), cudaMemcpyHostToDevice, ws));
  int rc = exchange(ws);
  if (!rc) {
    cudaMemcpyAsync(h.data(), n->d_g + off, cnt * sizeof(float), cudaMemcpyDeviceToHost, ws);
    cudaStreamSynchronize(ws);
    bool good = true;
    for (int64_t i = 0; i < cnt && good; ++i) good = h[i] == float(W * (W + 1) / 2) + float(W) * float(i & 1023);
    *ok_out = good ? 1 : 0;
    cudaMemsetAsync(n->d_g + off, 0, cnt * sizeof(float), ws);
    for (int i = 0; i < 10 && !rc; ++i) rc = exchange(ws);
    cudaEventRecord(e0, ws);
    for (int i = 0; i < iters && !rc; ++i) rc = exchange(ws);
    cudaEventRecord(e1, ws);
    cudaStreamSynchronize(ws);
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e0, e1);
    *us_out = ms * 1000.f / float(iters);
  }
  n->xchg_flags = keep_flags;
  n->xchg_blocks = keep_blocks;
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  cudaStreamDestroy(ws);
  B2_CHECK_CUDA(cudaGetLastError());
  return rc;
}

extern "C" int b200dqn_net_comm_status(b200dqn_net* n, int* mode, int* error) {
  B2_REQUIRE(n, B200DQN_EINVAL, "null net");
  DeviceGuard g(n->device);
  B2_CHECK_CUDA(cudaDeviceSynchronize());
  if (mode) *mode = n->world <= 1 ? 0 : (n->xchg_ok ? 2 : 1);
  uint32_t err = 0;
  B2_CHECK_CUDA(cudaMemcpy(&err, n->d_xerr, sizeof(err), cudaMemcpyDeviceToHost));
  if (error) *error = int(err);
  return B200DQN_OK;
}

extern "C" int b200dqn_net_comm_destroy(b200dqn_net* n) {
  B2_REQUIRE(n, B200DQN_EINVAL, "null net");
  DeviceGuard g(n->device);
  cudaDeviceSynchronize();
  // captured steps hold nodes of this communicator
  n->graph_step.drop();
  n->graph_train.drop();
  comm_destroy(n);
  return B200DQN_OK;
}
