// umma2.cuh — wgmma implicit-GEMM kernel (sm_90a), engine v2: operands arrive PRE-SPLIT (fp16 hi / scaled
// fp16 lo planes written once by their producer), so the mainloop is pure data movement:
//
//   kAsync : activations / gradients live in HBM as NHWC fp16 hi+lo planes; every 16-byte chunk of
//            the canonical K-major SWIZZLE_128B tile is one cp.async (LDGSTS) straight from global to
//            its swizzled shared-memory slot — the im2col gather costs no registers and no math.
//   kBulk  : weights live in HBM as ready-made tile images (the exact shared-memory byte image of a
//            [rows x 64] hi tile followed by the lo tile); one elected thread fetches a whole tile
//            with ONE TMA bulk copy (cp.async.bulk, SASS UBLKCP) that completes on an mbarrier.
//   kReg   : the u8 frame window of conv1 is converted in registers (u8 -> fp16 is exact, no lo part).
//
// 4-stage ring: loads for k-block i+3 are in flight while the tensor cores work on k-block i.
// Accumulation scheme (2 wgmma per k-step, fp32 accumulators in registers) as in umma.cuh.
#pragma once
#include <stdlib.h>
#include <type_traits>
#include <utility>

#include "umma.cuh"

namespace b200 {
namespace umma2 {

using umma::kBK;
using umma::kBM;
using umma::kThreads;

enum OperandMode { kReg = 0, kAsync = 1, kBulk = 2 };

struct RowCtx {      // per-row part of a gather address, computed once outside the k loop
  int64_t base;      // element offset
  int y, x;          // problem-specific (e.g. pixel coordinates for boundary tests)
  bool ok;           // row inside the problem
};
struct Planes {
  const __half* hi;
  int64_t lo_off;    // lo plane = hi + lo_off
};

__device__ __forceinline__ void cp_async16(uint32_t smem_dst, const void* gsrc, uint32_t src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 16, %2;" ::"r"(smem_dst), "l"(gsrc), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// fp32 -> fp16 hi + scaled fp16 lo (Rectlin masks are taken from the fp32 tensors, never from hi)
__device__ __forceinline__ void split1(float x, __half& hi, __half& lo) {
  const __half h = __float2half_rn(x);
  hi = h;
  lo = __float2half_rn((x - __half2float(h)) * umma::kLoScale);
}
__device__ __forceinline__ void split8_planes(const float v[8], __half* hi_dst, __half* lo_dst) {
  uint4 hi, lo;
  umma::split8(v, hi, lo);
  *reinterpret_cast<uint4*>(hi_dst) = hi;
  *reinterpret_cast<uint4*>(lo_dst) = lo;
}

// Problem P (see net_umma.cu):
//   static constexpr int kBN; static constexpr bool kAExact;
//   static constexpr int kAMode, kBMode;                         (OperandMode)
//   static constexpr bool kARowMajorThreads, kBRowMajorThreads;  (thread -> chunk mapping, as in umma.cuh)
//   int M(z), N(z); void krange(z, kb0, kb1);
//   kReg  : const uint8_t* a_row_ptr(z, m)  (once per row; nullptr = row outside the problem; a problem may return
//           any other per-row type instead, e.g. with the row's crop offsets)
//           uint2 a_raw8(row_ptr, k0)  8 raw bytes;  static void cvt8(uint2, float v[8])      (A only)
//   kAsync: RowCtx a_row(z, m)  — once per (thread, tile row): everything that depends on the row only
//           bool   a_chunk(z, row, kk, int64_t& off) — per k-block: element offset of the 8-wide chunk
//                  starting at k index kk; false -> zero fill.   PlanePair-like a_planes(z) -> (hi, lo_off)
//           same with b_row / b_chunk / b_planes for B
//   kBulk : const uint8_t* a_tile(z, mtile, kb) / b_tile(z, ntile, kb)      -> [hi image | lo image]
//           optional  static constexpr bool kAMnMajor = true  (bulk A only): the A tile is M-contiguous; it is fetched
//           as two [64 k-rows x 128 B] sub-tiles per half,  a_sub(z, mtile, kb, chunk) -> hi sub-tile, the lo
//           sub-tile kAMnLoOffset bytes behind it
//   void store8(z, m, n0, const float v[8])
//   static constexpr bool kDumpA: after k-block kb is staged, bulk-store the A_hi tile to a_dump(z, mtile, kb); one
//        bulk group per k-block, and a stage is refilled only once its dump has finished reading it
//   static constexpr bool kStagedEpilogue: store8 writes 8 CONTIGUOUS outputs of row m (NHWC tensors) ->
//        the tile is transposed through smem so that a warp's stores are whole cache lines
template <class P, class = void>
struct AMnMajor { static constexpr bool value = false; };
template <class P>
struct AMnMajor<P, std::void_t<decltype(P::kAMnMajor)>> { static constexpr bool value = P::kAMnMajor; };

// The bulk copies of one k-block's operand images into stage memory `st_gen` (one thread).
template <class P, class C>
__device__ __forceinline__ void issue_bulk_stage(const P& p, int z, int mtile, int ntile, int kb, uint8_t* st_gen,
                                                 uint64_t* bar) {
  if constexpr (P::kAMode == kBulk) {
    if constexpr (AMnMajor<P>::value) {
      constexpr uint32_t kSub = 64 * 128;   // [64 k-rows x 128 B]
      static_assert(2 * kSub == C::kABytes, "M = 128 is two 64-wide chunks");
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const uint8_t* src = p.a_sub(z, mtile, kb, c);
        tma_bulk_g2s(st_gen + c * kSub, src, kSub, bar);
        tma_bulk_g2s(st_gen + C::kABytes + c * kSub, src + P::kAMnLoOffset, kSub, bar);
      }
    } else {
      tma_bulk_g2s(st_gen, p.a_tile(z, mtile, kb), 2 * C::kABytes, bar);
    }
  }
  if constexpr (P::kBMode == kBulk)
    tma_bulk_g2s(st_gen + C::kAStage, p.b_tile(z, ntile, kb), 2 * C::kBBytes, bar);
}

template <class P, class = void>   // what a kReg problem's a_row_ptr returns
struct ARegRow { using type = const uint8_t*; };
template <class P>
struct ARegRow<P, std::void_t<decltype(std::declval<const P&>().a_row_ptr(0, 0))>> {
  using type = decltype(std::declval<const P&>().a_row_ptr(0, 0));
};

template <class P, class = void>
struct StagesOf { static constexpr int value = 0; };
template <class P>
struct StagesOf<P, std::void_t<decltype(P::kStagesOverride)>> { static constexpr int value = P::kStagesOverride; };

template <class P>
struct Cfg2 {
  static constexpr int BN = P::kBN;
  static constexpr uint32_t kABytes = kBM * 128;
  static constexpr uint32_t kBBytes = BN * 128;
  static constexpr uint32_t kAStage = (P::kAExact ? 1 : 2) * kABytes;
  static constexpr uint32_t kStageBytes = kAStage + 2 * kBBytes;
  // default: as deep a ring as one CTA per SM allows; a problem may ask for a shallower ring (kStagesOverride) so
  // that two CTAs — of this or of another kernel of the step — share an SM
  static constexpr int kStages = StagesOf<P>::value ? StagesOf<P>::value : (4 * kStageBytes <= 200 * 1024) ? 4 : 3;
  static constexpr uint32_t kSmemBytes = kStages * kStageBytes + 1024;
  static_assert(BN == 32 || BN == 64, "wgmma N = 2*BN (and BN) of the instantiated shapes");
  static_assert(kSmemBytes <= 227 * 1024, "H100: at most 227 KB of shared memory per block");
  static_assert(!(P::kAMode == kBulk && P::kAExact), "bulk A images always carry hi+lo");
};

// Debug timeline (B200DQN_TRACE_LABEL=<kernel label>): thread 0 of CTA (0,0,0) of the selected kernel stamps
// clock64() at pipeline events; read with b200dqn_debug_trace().
constexpr int kTraceSlots = 96;
__device__ unsigned long long g_trace[kTraceSlots];
#define B2_TRACE(cond, slot)                                                      \
  do {                                                                            \
    if (trace && (cond) && (slot) < kTraceSlots) g_trace[(slot)] = clock64();     \
  } while (0)

__device__ __forceinline__ void cp_async_arrive_noinc(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

constexpr int kLoadThreads = 256;            // 2 warpgroups: operand staging, MMAs of their 64 rows, epilogue
constexpr int kThreads2 = kLoadThreads;

// Pipeline, every thread in every role (the accumulators of wgmma live in the registers of the issuing warpgroup):
//   stage j % S is filled S k-blocks ahead (cp.async / TMA bulk / st.shared; cp.async.mbarrier.arrive.noinc fires
//   when this thread's copies have landed) and completes on full[j % S];
//   k-block it: wait full[it % S]; fence.proxy.async (generic-proxy smem writes -> async proxy); each warpgroup
//   issues, on its 64 rows of A, per k-step  [acc0 | acc1] += A_hi x [B_hi ; B_lo]  (one N = 2*BN wgmma: the hi and
//   lo weight tiles are adjacent in shared memory) and  acc2 += A_lo x B_hi;  then wgmma.wait_group 1 (k-block it-1
//   has completed in this warpgroup), one named barrier over both warpgroups, and stage (it-1) % S is refilled with
//   k-block it-1+S while the tensor cores work on k-block it.
//   release_early: the successor may pre-launch as soon as this kernel has passed its dependency wait (links of the
//   single-GPU critical chain), instead of once this CTA's mainloop has issued all its loads.
template <class P>
__global__ void __launch_bounds__(kThreads2, 1) k_umma2(const P p, const int trace_in, const bool release_early,
                                                        const KTrace kt) {
  using C = Cfg2<P>;
  constexpr int BN = C::BN;
  constexpr int S = C::kStages;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t s_full[S];    // operands of the stage have landed

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const int z = blockIdx.z;
  const bool trace = trace_in && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0;
  kt_begin(kt);
  B2_TRACE(tid == 0, 0);
  const int M = p.M(z), N = p.N(z);
  const int mtile = blockIdx.x;
  const int m0 = mtile * kBM, n0 = blockIdx.y * BN;
  if (m0 >= M || n0 >= N) return;
  int kb0, kb1;
  p.krange(z, kb0, kb1);
  const int nkb = kb1 - kb0;

  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  constexpr bool kAnyBulk = (P::kAMode == kBulk) || (P::kBMode == kBulk);
  constexpr uint32_t kBulkBytes = (P::kAMode == kBulk ? 2 * C::kABytes : 0) + (P::kBMode == kBulk ? 2 * C::kBBytes : 0);

  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < S; ++s) mbar_init(&s_full[s], kLoadThreads + (kAnyBulk ? 1 : 0));
    mbar_fence_init();
  }
  __syncthreads();
  B2_TRACE(tid == 0, 1);

  constexpr int kACh = kBM * 8 / kLoadThreads;
  constexpr int kBCh = (BN * 8 + kLoadThreads - 1) / kLoadThreads;
  RowCtx arow[kACh];
  RowCtx brow[kBCh];
  Planes apl{nullptr, 0}, bpl{nullptr, 0};
  if constexpr (P::kAMode == kAsync) {
    apl = p.a_planes(z);
#pragma unroll
    for (int i = 0; i < kACh; ++i) {
      const int id = tid + i * kLoadThreads;
      arow[i] = p.a_row(z, m0 + (P::kARowMajorThreads ? (id >> 3) : (id % kBM)));
    }
  }
  if constexpr (P::kBMode == kAsync) {
    bpl = p.b_planes(z);
#pragma unroll
    for (int i = 0; i < kBCh; ++i) {
      const int id = tid + i * kLoadThreads;
      brow[i] = p.b_row(z, n0 + (P::kBRowMajorThreads ? (id >> 3) : (id % BN)));
    }
  }
  // Weight tile images do not depend on the predecessor kernel (they were refreshed by the PREVIOUS step's
  // optimizer, long finished): the TMA bulk copies of the first S k-blocks are issued ahead of the dependency
  // wait, so that for the weight-heavy kernels (fc1 forward / dgrad: 32 KB of image per k-block) the first
  // stages are already full when the activations may be touched.
  if constexpr (kAnyBulk) {
    if (tid == 0) {
#pragma unroll
      for (int j = 0; j < S; ++j) {
        if (j < nkb) {
          uint8_t* st_gen = smem_gen + j * C::kStageBytes;
          mbar_arrive_expect_tx(&s_full[j], kBulkBytes);
          issue_bulk_stage<P, C>(p, z, mtile, blockIdx.y, kb0 + j, st_gen, &s_full[j]);
        }
      }
    }
  }
  // Everything above (barrier init, the gather index tables, the first weight tiles) overlapped the previous kernel
  // of the chain; only from here on do we touch its outputs.
  pdl_wait();
  if (release_early) pdl_launch_dependents();
  // kReg operands: per-row source pointers, once per kernel (they may depend on upstream data — the
  // sampled indexes — so they are built after the wait, but not again for every k-block)
  typename ARegRow<P>::type areg[kACh];
  if constexpr (P::kAMode == kReg) {
#pragma unroll
    for (int i = 0; i < kACh; ++i) {
      const int id = tid + i * kLoadThreads;
      areg[i] = p.a_row_ptr(z, m0 + (P::kARowMajorThreads ? (id >> 3) : (id % kBM)));
    }
  }
  // ... and the raw bytes of the first S k-blocks are requested up front: one exposed global-memory
  // latency for the whole tile instead of one per k-block (the conversion path is synchronous).
  uint2 araw[S][kACh];
  if constexpr (P::kAMode == kReg) {
#pragma unroll
    for (int j = 0; j < S; ++j)
#pragma unroll
      for (int i = 0; i < kACh; ++i) {
        const int id = tid + i * kLoadThreads;
        const int c = P::kARowMajorThreads ? (id & 7) : (id / kBM);
        araw[j][i] = (j < nkb) ? p.a_raw8(areg[i], (kb0 + j) * kBK + c * 8) : make_uint2(0u, 0u);
      }
  }
  // operands of k-block j into stage j % S (the stage is free: its previous k-block has been consumed)
  auto stage = [&](int j) {
    const int s = j % S, kb = kb0 + j, k0 = kb * kBK;
    B2_TRACE(tid == 0, 8 + j * 4 + 2);
    const uint32_t st_addr = smem_base + s * C::kStageBytes;
    uint8_t* st_gen = smem_gen + s * C::kStageBytes;
    const uint32_t a_hi = st_addr, a_lo = st_addr + C::kABytes, b_hi = st_addr + C::kAStage, b_lo = b_hi + C::kBBytes;
    if (kAnyBulk && tid == 0 && j >= S) {   // the first S k-blocks' images were requested before the dependency wait
      mbar_arrive_expect_tx(&s_full[s], kBulkBytes);
      issue_bulk_stage<P, C>(p, z, mtile, blockIdx.y, kb, st_gen, &s_full[s]);
    }
    if constexpr (P::kAMode == kAsync) {
#pragma unroll
      for (int i = 0; i < kACh; ++i) {
        const int id = tid + i * kLoadThreads;
        const int r = P::kARowMajorThreads ? (id >> 3) : (id % kBM);
        const int c = P::kARowMajorThreads ? (id & 7) : (id / kBM);
        int64_t eoff = 0;
        const bool ok = arow[i].ok && p.a_chunk(z, arow[i], k0 + c * 8, eoff);
        const uint32_t bytes = ok ? 16u : 0u;
        const __half* hi = apl.hi + (ok ? eoff : 0);
        const uint32_t off = umma::sw128_off(r, c);
        cp_async16(a_hi + off, hi, bytes);
        if (!P::kAExact) cp_async16(a_lo + off, hi + apl.lo_off, bytes);
      }
    } else if constexpr (P::kAMode == kReg) {
      float av[kACh][8];
#pragma unroll
      for (int i = 0; i < kACh; ++i) {
        const int id = tid + i * kLoadThreads;
        const int c = P::kARowMajorThreads ? (id & 7) : (id / kBM);
        uint2 raw = make_uint2(0u, 0u);
        if (j < S) {
#pragma unroll
          for (int jj = 0; jj < S; ++jj) if (jj == j) raw = araw[jj][i];   // static indexing keeps araw in registers
        } else {
          raw = p.a_raw8(areg[i], k0 + c * 8);
        }
        P::cvt8(raw, av[i]);
      }
#pragma unroll
      for (int i = 0; i < kACh; ++i) {
        const int id = tid + i * kLoadThreads;
        const int r = P::kARowMajorThreads ? (id >> 3) : (id % kBM);
        const int c = P::kARowMajorThreads ? (id & 7) : (id / kBM);
        uint4 hi, lo;
        umma::split8(av[i], hi, lo);
        *reinterpret_cast<uint4*>(st_gen + umma::sw128_off(r, c)) = hi;
        if (!P::kAExact) *reinterpret_cast<uint4*>(st_gen + C::kABytes + umma::sw128_off(r, c)) = lo;
      }
      fence_proxy_async_smem();   // st.shared (generic proxy) -> async proxy, writer side
    }
    if constexpr (P::kBMode == kAsync) {
#pragma unroll
      for (int i = 0; i < kBCh; ++i) {
        const int id = tid + i * kLoadThreads;
        if (id < BN * 8) {
          const int r = P::kBRowMajorThreads ? (id >> 3) : (id % BN);
          const int c = P::kBRowMajorThreads ? (id & 7) : (id / BN);
          int64_t eoff = 0;
          const bool ok = brow[i].ok && p.b_chunk(z, brow[i], k0 + c * 8, eoff);
          const uint32_t bytes = ok ? 16u : 0u;
          const __half* hi = bpl.hi + (ok ? eoff : 0);
          const uint32_t off = umma::sw128_off(r, c);
          cp_async16(b_hi + off, hi, bytes);
          cp_async16(b_lo + off, hi + bpl.lo_off, bytes);
        }
      }
    }
    if constexpr (P::kAMode == kAsync || P::kBMode == kAsync)
      cp_async_arrive_noinc(&s_full[s]);   // fires when this thread's copies for the stage have landed
    else
      mbar_arrive(&s_full[s]);
    B2_TRACE(tid == 0, 8 + j * 4 + 3);
  };

  for (int j = 0; j < S && j < nkb; ++j) stage(j);

  // ================================================================ mainloop
  constexpr bool kAMn = AMnMajor<P>::value;
  constexpr uint32_t kAStep = kAMn ? 128 : 2;        // descriptor address units (16 B) per 16 k: 16 k-rows x 128 B or 32 B
  constexpr uint32_t kAWg = umma::kWgM * 128;        // this warpgroup's A: 64 rows further (K-major) / the 2nd m chunk (MN)
  float acc[BN];                                     // N = 2*BN fragment: [acc0 | acc1]
  float acc2[P::kAExact ? 1 : BN / 2];               // N = BN fragment: A_lo x B_hi
#pragma unroll
  for (int i = 0; i < BN; ++i) acc[i] = 0.f;
#pragma unroll
  for (int i = 0; i < (P::kAExact ? 1 : BN / 2); ++i) acc2[i] = 0.f;
  for (int it = 0; it < nkb; ++it) {
    const int s = it % S;
    mbar_wait(&s_full[s], (it / S) & 1);
    fence_proxy_async_smem();
    B2_TRACE(tid == 0, 8 + it * 4 + 0);
    const uint32_t sa = smem_base + s * C::kStageBytes;
    if constexpr (P::kDumpA) {
      // The staged [128 x 64] A_hi tile IS the MN-major operand the wgrad of this layer needs
      // (row = pixel, 64 contiguous taps): ship it out with one TMA bulk store per k-block.
      if (tid == 0) {
        uint8_t* dump = p.a_dump(z, mtile, kb0 + it);
        if (dump) tma_bulk_s2g(dump, smem_gen + s * C::kStageBytes, C::kABytes);
        tma_bulk_commit();
      }
    }
    const uint32_t a_hi = sa + wg * kAWg, a_lo = a_hi + C::kABytes;
    const uint64_t da_hi = kAMn ? umma::make_desc_mn(a_hi, 64 * 128) : umma::make_desc_sw128(a_hi);
    const uint64_t da_lo = kAMn ? umma::make_desc_mn(a_lo, 64 * 128) : umma::make_desc_sw128(a_lo);
    const uint64_t db = umma::make_desc_sw128(sa + C::kAStage);   // [B_hi ; B_lo], 2*BN rows
    umma::wgmma_fence();
#pragma unroll
    for (int k = 0; k < kBK / 16; ++k) {
      umma::wgmma_f16<2 * BN, kAMn ? 1 : 0, 0>(acc, da_hi + kAStep * k, db + 2 * k);
      if constexpr (!P::kAExact) umma::wgmma_f16<BN, kAMn ? 1 : 0, 0>(acc2, da_lo + kAStep * k, db + 2 * k);
    }
    umma::wgmma_commit();
    umma::wgmma_wait<1>();
    B2_TRACE(tid == 0, 8 + it * 4 + 1);
    if (it >= 1 && it - 1 + S < nkb) {
      // more k-blocks than stages (conv1 with H > S frames): k-block it-1's dump must have read its stage
      if (P::kDumpA && tid == 0) tma_bulk_wait_read<1>();
      named_bar_sync(1, kThreads2);   // both warpgroups are done with k-block it-1: its stage takes k-block it-1+S
      stage(it - 1 + S);
    }
  }
  B2_TRACE(tid == 0, 3);
  // All of this CTA's loads are issued: let the successor kernel pre-launch NOW (it sets up its barriers and index
  // tables, then parks at its pdl_wait) — late enough that its parked CTAs do not hog shared memory for long, early
  // enough to hide its prologue behind our epilogue.  (A no-op when release_early already did it.)
  pdl_launch_dependents();

  // ================================================================ epilogue
  // The combined tile goes through (now idle) stage memory: a thread then owns (row, 8 consecutive columns) items —
  // row-major items (kStagedEpilogue: 8 CONTIGUOUS outputs of row m, a warp's stores cover whole lines) or lanes along
  // m (strided outputs).  Row pitch BN*4 + 16 B keeps both phases nearly bank-conflict free.
  constexpr int kPitch = BN * 4 + 16;
  constexpr int kChunksPerRow = BN / 8;
  constexpr int kIt = kBM * kChunksPerRow / kLoadThreads;
  static_assert(kBM * kPitch <= C::kStages * C::kStageBytes, "staging tile must fit the stage ring");
  auto item = [&](int i, int& r, int& cc) {
    const int id = tid + i * kLoadThreads;
    if constexpr (P::kStagedEpilogue) { r = id / kChunksPerRow; cc = id % kChunksPerRow; }
    else { r = id % kBM; cc = id / kBM; }
  };
  // Operands of the epilogue that do not depend on the accumulators (Rectlin masks of the dgrads) are
  // fetched now, while the tensor cores are still draining the last k-blocks.
  float pf[P::kPrefetch ? kIt : 1][8];
  if constexpr (P::kPrefetch) {
#pragma unroll
    for (int i = 0; i < kIt; ++i) {
      int r, cc;
      item(i, r, cc);
      if (m0 + r < M && n0 + cc * 8 < N) p.prefetch8(z, m0 + r, n0 + cc * 8, pf[i]);
    }
  }
  umma::wgmma_wait<0>();
  if constexpr (P::kDumpA) {
    if (tid == 0) tma_bulk_wait_read_all();   // smem may now be reused by the staging tile
  }
  named_bar_sync(1, kThreads2);   // every warpgroup's MMAs (and the A dump) have finished reading the stages
  B2_TRACE(tid == 0, 4);
  umma::stage_acc<BN>(acc, P::kAExact ? nullptr : acc2, smem_gen, kPitch, wg, warp, lane);
  named_bar_sync(1, kThreads2);
#pragma unroll
  for (int i = 0; i < kIt; ++i) {
    int r, cc;
    item(i, r, cc);
    uint8_t* src = smem_gen + r * kPitch + cc * 32;
    const float4 v0 = *reinterpret_cast<const float4*>(src), v1 = *reinterpret_cast<const float4*>(src + 16);
    float v[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
    if (m0 + r < M && n0 + cc * 8 < N) {
      if constexpr (P::kPrefetch) p.store8p(z, m0 + r, n0 + cc * 8, v, pf[i]);
      else p.store8(z, m0 + r, n0 + cc * 8, v);
    }
  }
  B2_TRACE(tid == 0, 5);
  kt_end(kt);
  B2_TRACE(tid == 0, 6);
}

static inline int read_trace(unsigned long long* out, int n) {
  if (n > kTraceSlots) n = kTraceSlots;
  return cudaMemcpyFromSymbol(out, g_trace, n * sizeof(unsigned long long)) == cudaSuccess ? n : -1;
}

template <class P>
static int launch_umma2(const char* label, const P& p, int M, int N, int Z, cudaStream_t st, bool release_early) {
  using C = Cfg2<P>;
  static bool configured = false;
  if (!configured) {
    B2_CHECK_CUDA(cudaFuncSetAttribute(k_umma2<P>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::kSmemBytes));
    configured = true;
  }
  dim3 grid((M + kBM - 1) / kBM, (N + C::BN - 1) / C::BN, Z);
  static const char* trace_label = getenv("B200DQN_TRACE_LABEL");
  const int trace = (trace_label && strcmp(trace_label, label) == 0) ? 1 : 0;
  B2_CHECK_CUDA(launch_pdl(k_umma2<P>, grid, dim3(kThreads2), C::kSmemBytes, st, p, trace, release_early,
                           ktrace_slot(label)));
  B2_PROF(label, st);
  return B200DQN_OK;
}

// ------------------------------------------------------------------------------------------
// Tile-image packer: one thread per 16-byte chunk of the image.
// Source S: int tiles(), rows(), kblocks(); void src8(tile, row, k0, float v[8]) (zeros when out of range)
// image layout: [tile][kb][hi rows*128 B | lo rows*128 B], chunk (r, c) at sw128_off(r, c).
// ------------------------------------------------------------------------------------------
template <class S>
__global__ void __launch_bounds__(256) k_pack_image(const S src, uint8_t* __restrict__ image, const KTrace kt) {
  kt_begin(kt);
  const int rows = src.rows(), nkb = src.kblocks();
  const int64_t chunks_per_tile_kb = int64_t(rows) * 8;
  const int64_t total = int64_t(src.tiles()) * nkb * chunks_per_tile_kb;
  pdl_wait();
  pdl_launch_dependents();
  for (int64_t id = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; id < total; id += int64_t(gridDim.x) * blockDim.x) {
  const int64_t tk = id / chunks_per_tile_kb;
  const int within = int(id % chunks_per_tile_kb);
  const int tile = int(tk / nkb), kb = int(tk % nkb);
  const int r = S::kRowMajorThreads ? (within >> 3) : (within % rows);
  const int c = S::kRowMajorThreads ? (within & 7) : (within / rows);
  float v[8];
  src.src8(tile, r, kb * kBK + c * 8, v);
  uint4 hi, lo;
  umma::split8(v, hi, lo);
  uint8_t* base = image + tk * (int64_t(rows) * 256);
  *reinterpret_cast<uint4*>(base + umma::sw128_off(r, c)) = hi;
  *reinterpret_cast<uint4*>(base + int64_t(rows) * 128 + umma::sw128_off(r, c)) = lo;
  }
  kt_end(kt);
}

// max_ctas > 0 caps the grid (grid-stride loop) for launches that must not crowd the SMs
template <class S>
static int launch_pack(const char* label, const S& src, uint8_t* image, cudaStream_t st, int max_ctas = 0) {
  const int64_t total = int64_t(src.tiles()) * src.kblocks() * src.rows() * 8;
  unsigned grid = unsigned((total + 255) / 256);
  if (max_ctas > 0 && grid > unsigned(max_ctas)) grid = unsigned(max_ctas);
  B2_CHECK_CUDA(launch_pdl(k_pack_image<S>, dim3(grid), dim3(256), 0, st, src, image, ktrace_slot(label)));
  B2_PROF(label, st);
  return B200DQN_OK;
}

}  // namespace umma2
}  // namespace b200
