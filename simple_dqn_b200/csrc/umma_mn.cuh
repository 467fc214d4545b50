// umma_mn.cuh — wgmma kernel (sm_90a) for the weight-gradient family: D[M x N] = sum_k A[m][k] * B[n][k]
// where the reduction index k runs over (sample, pixel) and BOTH operands are stored with their
// M / N index contiguous (NHWC activations: one pixel = one contiguous run of channels).  Those are
// "MN-major" wgmma operands: the 128-byte shared-memory row is a run of 64 consecutive m (or n) for
// ONE k, eight consecutive k rows form the 1024-byte swizzle atom (cute canonical layout
// Swizzle<3,4,3> o ((8,8,m),(8,k)) : ((1,8,LBO),(64,SBO)) in fp16 elements).  So the gather is again
// pure cp.async of 16-byte pieces (or TMA bulk copies of ready-made sub-tiles), no transposition anywhere.
//
// Per 64-pixel k-block the stage holds   A_hi [2 chunks x 64 rows x 128 B] (+ A_lo)   and
//   BN = 64:  B_hi [64 x 128 B] followed by B_lo [64 x 128 B]   -> one N = 128 wgmma gives [acc0 | acc1]
//   BN = 32:  one tile whose rows are [32 hi | 32 lo]            -> one N = 64  wgmma gives [acc0 | acc1]
// and, when A is not exact,  acc2 += A_lo x B_hi  (N = BN, own accumulator, see umma.cuh); each of the two warpgroups multiplies one 64-wide
// m chunk of A (wgmma M = 64).  Split-K over blockIdx.z.
#pragma once
#include "umma2.cuh"

namespace b200 {
namespace umma_mn {

using umma::kBM;
using umma2::kLoadThreads;
using umma2::kThreads2;
using umma2::Planes;

constexpr int kKB = 64;  // reduction rows (pixels) per k-block

using umma::make_desc_mn;   // MN-major SWIZZLE_128B descriptor (umma.cuh)
// byte offset of 16-byte piece j of k-row kr inside one [64 k-rows x 128 B] sub-tile
__device__ __forceinline__ uint32_t mn_off(int kr, int j) {
  return uint32_t((kr >> 3) * 1024 + (kr & 7) * 128 + ((j ^ (kr & 7)) << 4));
}

struct PixCtx {   // decoded reduction index (one per thread per k-block)
  int n, p, q;
  bool ok;
};

// Problem P:
//   static constexpr int kBN (32 or 64); static constexpr bool kAExact, kABulk;
//   int M(z), N(z); void krange(z, kb0, kb1);  PixCtx pix(z, kpix);
//   !kABulk: Planes a_planes(z); bool a_run(z, pix, mchunk, int64_t& off)     64 contiguous fp16 of A for this pixel
//    kABulk: const uint8_t* a_sub(z, mchunk, kb)   ready-made [64 k-rows x 128 B] sub-tile image (exact A only);
//            nullptr for the second m chunk of a tile whose rows 64..127 lie beyond M (not fetched: those
//            accumulator rows are never stored)
//   Planes b_planes(z); int64_t b_off(z, pix)                                  BN contiguous fp16 of B for this pixel
//   void store8(z, m, n0, const float v[8])
template <class P>
struct CfgMN {
  static constexpr int BN = P::kBN;
  static_assert(BN == 32 || BN == 64, "B rows are packed as [hi | lo] (BN = 32) or hi tile + lo tile (BN = 64)");
  static constexpr uint32_t kSub = kKB * 128;                      // one [64 x 128 B] sub-tile
  static constexpr uint32_t kAHalf = 2 * kSub;                     // A_hi (two m chunks)
  static constexpr uint32_t kAStage = (P::kAExact ? 1 : 2) * kAHalf;
  static constexpr uint32_t kBStage = (BN == 64 ? 2 : 1) * kSub;
  static constexpr uint32_t kStageBytes = kAStage + kBStage;
  static constexpr int kStages = P::kStages;   // 4 for the split-K conv wgrads; 2 for the single-k-block fc1 wgrad
  static constexpr uint32_t kSmemBytes = kStages * kStageBytes + 1024;
  static_assert(kBM * (BN * 4 + 16) <= kStages * kStageBytes, "epilogue staging tile must fit the stage ring");
  static_assert(kSmemBytes <= 227 * 1024, "H100: at most 227 KB of shared memory per block");
};

// release_early: as in umma2.cuh's k_umma2
template <class P>
__global__ void __launch_bounds__(kThreads2, 1) k_umma_mn(const P p, const bool release_early, const KTrace kt) {
  using C = CfgMN<P>;
  constexpr int BN = C::BN;
  constexpr int S = C::kStages;
  static_assert(P::kAExact || BN == 64, "acc2 += A_lo x B_hi reads B_hi as one whole 64-wide MN chunk");
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t s_full[S];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const int z = blockIdx.z;
  kt_begin(kt);
  const int M = p.M(z), N = p.N(z);
  const int m0 = blockIdx.x * kBM, n0 = blockIdx.y * BN;
  if (m0 >= M || n0 >= N) return;
  int kb0, kb1;
  p.krange(z, kb0, kb1);
  const int nkb = kb1 - kb0;

  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));

  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < S; ++s) mbar_init(&s_full[s], kLoadThreads + (P::kABulk ? 1 : 0));
    mbar_fence_init();
  }
  __syncthreads();

  if (nkb <= 0) {
    // nothing to reduce in this split: the partial is all zeros
    pdl_wait();
    const float zero[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int id = tid; id < kBM * (BN / 8); id += kLoadThreads) {
      const int r = id / (BN / 8), cc = id % (BN / 8);
      if (m0 + r < M && n0 + cc * 8 < N) p.store8(z, m0 + r, n0 + cc * 8, zero);
    }
    kt_end(kt);
    return;
  }

  // ================================================================ loaders
  // thread -> k row (tid >> 2) and a quarter (tid & 3) of that row's 16-byte pieces
  const int kr = tid >> 2, sub = tid & 3;
  const Planes bpl = p.b_planes(z);
  Planes apl{nullptr, 0};
  if constexpr (!P::kABulk) apl = p.a_planes(z);
  pdl_wait();   // the prologue above overlapped the predecessor
  if (release_early) pdl_launch_dependents();
  auto stage = [&](int j) {
    const int s = j % S;
    const uint32_t st_addr = smem_base + s * C::kStageBytes;
    uint8_t* st_gen = smem_gen + s * C::kStageBytes;
    const PixCtx px = p.pix(z, (kb0 + j) * kKB + kr);
    // ---- A: 2 m-chunks x 8 pieces per row; this thread: chunk (sub >> 1), pieces (sub & 1) * 4 .. + 3
    if constexpr (P::kABulk) {
      static_assert(P::kAExact, "bulk A sub-tiles carry no lo part");
      if (tid == 0) {
        const uint8_t* a1 = p.a_sub(z, blockIdx.x * 2 + 1, kb0 + j);
        mbar_arrive_expect_tx(&s_full[s], (a1 ? 2 : 1) * C::kSub);
        tma_bulk_g2s(st_gen, p.a_sub(z, blockIdx.x * 2, kb0 + j), C::kSub, &s_full[s]);
        if (a1) tma_bulk_g2s(st_gen + C::kSub, a1, C::kSub, &s_full[s]);
      }
    } else {
      const int mc = sub >> 1, j0 = (sub & 1) * 4;
      const int mchunk = blockIdx.x * 2 + mc;
      int64_t eoff = 0;
      const bool ok = px.ok && p.a_run(z, px, mchunk, eoff);
      const __half* src = apl.hi + (ok ? eoff : 0);
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const uint32_t dst = st_addr + mc * C::kSub + mn_off(kr, j0 + t);
        umma2::cp_async16(dst, src + (j0 + t) * 8, ok ? 16u : 0u);
        if (!P::kAExact) umma2::cp_async16(dst + C::kAHalf, src + apl.lo_off + (j0 + t) * 8, ok ? 16u : 0u);
      }
    }
    // ---- B
    {
      const __half* src = bpl.hi + (px.ok ? p.b_off(z, px) + n0 : 0);
      const uint32_t bytes = px.ok ? 16u : 0u;
      if constexpr (BN == 64) {   // pieces 0..7 of the hi tile and of the lo tile; this thread: 2 + 2
#pragma unroll
        for (int t = 0; t < 2; ++t) {
          const int jj = sub * 2 + t;
          const uint32_t dst = st_addr + C::kAStage + mn_off(kr, jj);
          umma2::cp_async16(dst, src + jj * 8, bytes);
          umma2::cp_async16(dst + C::kSub, src + bpl.lo_off + jj * 8, bytes);
        }
      } else {                    // row = [32 hi | 32 lo]: pieces 0..3 hi, 4..7 lo; this thread: 1 + 1
        const uint32_t dst = st_addr + C::kAStage;
        umma2::cp_async16(dst + mn_off(kr, sub), src + sub * 8, bytes);
        umma2::cp_async16(dst + mn_off(kr, 4 + sub), src + bpl.lo_off + sub * 8, bytes);
      }
    }
    umma2::cp_async_arrive_noinc(&s_full[s]);
  };
  for (int j = 0; j < S && j < nkb; ++j) stage(j);

  // ================================================================ mainloop (pipeline as in umma2.cuh)
  // warpgroup wg multiplies m chunk wg of A (64 m x 64 k-rows); B = [B_hi | B_lo] as 2 chunks (BN = 64, LBO = one
  // sub-tile) or one chunk of [32 hi | 32 lo] rows (BN = 32)
  float acc[BN];                           // N = 2*BN fragment: [acc0 | acc1]
  float acc2[P::kAExact ? 1 : BN / 2];     // N = BN fragment: A_lo x B_hi
#pragma unroll
  for (int i = 0; i < BN; ++i) acc[i] = 0.f;
#pragma unroll
  for (int i = 0; i < (P::kAExact ? 1 : BN / 2); ++i) acc2[i] = 0.f;
  for (int it = 0; it < nkb; ++it) {
    const int s = it % S;
    mbar_wait(&s_full[s], (it / S) & 1);
    fence_proxy_async_smem();
    const uint32_t sa = smem_base + s * C::kStageBytes;
    const uint64_t da_hi = make_desc_mn(sa + wg * C::kSub, C::kSub);
    const uint64_t da_lo = make_desc_mn(sa + C::kAHalf + wg * C::kSub, C::kSub);
    const uint64_t db = make_desc_mn(sa + C::kAStage, C::kSub);
    umma::wgmma_fence();
#pragma unroll
    for (int k = 0; k < kKB / 16; ++k) {   // 16 k rows = 2048 bytes = +128 in the address field
      umma::wgmma_f16<2 * BN, 1, 1>(acc, da_hi + 128 * k, db + 128 * k);
      if constexpr (!P::kAExact) umma::wgmma_f16<BN, 1, 1>(acc2, da_lo + 128 * k, db + 128 * k);
    }
    umma::wgmma_commit();
    umma::wgmma_wait<1>();
    if (it >= 1 && it - 1 + S < nkb) {
      umma2::named_bar_sync(1, kThreads2);   // both warpgroups are done with k-block it-1
      stage(it - 1 + S);
    }
  }
  pdl_launch_dependents();   // see umma2.cuh: successor pre-launch is deferred to the end of our mainloop

  // ================================================================ epilogue (smem-transposed, see umma2.cuh)
  umma::wgmma_wait<0>();
  umma2::named_bar_sync(1, kThreads2);   // every warpgroup's MMAs have finished reading the stages
  {
    constexpr int kPitch = BN * 4 + 16;
    umma::stage_acc<BN>(acc, P::kAExact ? nullptr : acc2, smem_gen, kPitch, wg, warp, lane);
    umma2::named_bar_sync(1, kLoadThreads);
    constexpr int kChunksPerRow = BN / 8;
#pragma unroll
    for (int i = 0; i < kBM * kChunksPerRow / kLoadThreads; ++i) {
      const int id = tid + i * kLoadThreads;
      const int r = id / kChunksPerRow, cc = id % kChunksPerRow;
      const float* src = reinterpret_cast<const float*>(smem_gen + r * kPitch + cc * 32);
      const float4 v0 = *reinterpret_cast<const float4*>(src), v1 = *reinterpret_cast<const float4*>(src + 4);
      const float v[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
      if (m0 + r < M && n0 + cc * 8 < N) p.store8(z, m0 + r, n0 + cc * 8, v);
    }
  }
  kt_end(kt);
}

template <class P>
static int launch_umma_mn(const char* label, const P& p, int M, int N, int Z, cudaStream_t st, bool release_early) {
  using C = CfgMN<P>;
  static bool configured = false;
  if (!configured) {
    B2_CHECK_CUDA(cudaFuncSetAttribute(k_umma_mn<P>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::kSmemBytes));
    configured = true;
  }
  dim3 grid((M + kBM - 1) / kBM, (N + C::BN - 1) / C::BN, Z);
  B2_CHECK_CUDA(launch_pdl(k_umma_mn<P>, grid, dim3(kThreads2), C::kSmemBytes, st, p, release_early,
                           ktrace_slot(label)));
  B2_PROF(label, st);
  return B200DQN_OK;
}

}  // namespace umma_mn
}  // namespace b200
