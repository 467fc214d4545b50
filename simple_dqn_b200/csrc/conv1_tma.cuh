// conv1_tma.cuh — first conv layer (8x8x32, stride 4, src/deepqnetwork.py:83) with the replay gather of
// ReplayMemory.getMinibatch (src/replay_memory.py:71-72) fused in and done by tensor-map TMA:
//
//   * the frame window of a tile — 28 image rows of every frame of the sample's state, both networks' states at
//     once when they come out of the ring (prestates = frames idx-4..idx-1, poststates = idx-3..idx share 3 of 4) —
//     is ONE cp.async.bulk.tensor.3d (SASS UTMALDG) from the u8 ring straight into shared memory: the ring
//     [size][84][84] u8 is described to TMA as [size][21][84 x u32] (21 groups of 4 rows = 336 bytes, every
//     stride a multiple of 16 bytes), box = {84, 7, 5}: 11,760 bytes, each ring byte leaves HBM once per CTA;
//   * 8 warps turn the window into the canonical K-major SWIZZLE_128B fp16 tiles of the implicit GEMM (u8 -> fp16
//     is exact: no lo plane), one [128 pixels x 64 taps] tile per FRAME; a frame shared by both networks is
//     converted once and multiplied by both networks' weights (online k-block f, target k-block f-1);
//   * the same two warpgroups issue wgmma (M = 64 per warpgroup, N = 64 = [W_hi ; W_lo] in one instruction) as tiles
//     become ready; accumulators of both networks live in registers; the epilogue applies 1/255 (the _setInput divide,
//     src/deepqnetwork.py:100) and Rectlin and writes fp32 + fp16 hi/lo planes;
//   * the online network's tiles are also shipped to the im2col image conv1_wgrad reads (TMA bulk store).
//
// Tiling: one CTA = 5 output rows x 20 columns = 100 pixels of one sample (a 128-row tile, 100 live rows);
// grid = 4 x samples.  Shared memory: the window(s) (12 KB each) + a 3-stage ring of [A tile 16 KB | weight tiles
// 2 x 8 KB] = 109 KB, so two CTAs share an SM and the next kernels of the PDL chain can still pre-launch.
#pragma once
#include <cuda.h>

#include "umma2.cuh"

namespace b200 {
namespace conv1tma {

constexpr int kTileRows = 100;                  // live rows of a 128-row tile: 5 output rows x 20
constexpr int kTilesPerSample = 4;
constexpr int kBoxGroups = 7;                   // 7 groups of 4 image rows = the 28 rows under 5 output rows
constexpr int kGroupBytes = 4 * kFrameW;        // 336
constexpr int kFrameBoxBytes = kBoxGroups * kGroupBytes;   // 2352 per frame
constexpr uint32_t kATile = 128 * 128;          // [128 rows x 64 fp16]
constexpr uint32_t kWTile = 64 * 128;           // [32 hi rows ; 32 lo rows] x 64 fp16
constexpr int kRing = 3;                        // stages: one frame's A tile + the (<= 2) weight tiles that multiply it
constexpr uint32_t kStage = kATile + 2 * kWTile;   // 32 KB
constexpr uint32_t kBoxStride = 12288;          // one window (<= 5 frames x 2352 B), 128-byte aligned
// 109 KB with one window (ring train / predict): two CTAs per SM, and successor kernels of the PDL chain still find
// room to pre-launch; 121 KB with two windows (staged states)
static inline uint32_t smem_bytes(int windows) { return kRing * kStage + uint32_t(windows) * kBoxStride + 1024; }

struct Params {
  // frame sources: src 0 feeds the online network, src 1 the target network.  shared5: both read ONE 5-frame
  // window of src 0 (ring case: frame0[1] == frame0[0] + 1).
  const int32_t* idx[2];     // per-sample frame index table
  int shift[2];              // first frame of the state = idx[n] + shift
  int shared5;
  int nets;                  // 1 (predict) or 2 (train)
  int rows;                  // samples
  const uint8_t* wimg[2];    // [4 kb][hi 32x128 | lo 32x128]
  float* out[2];             // H1 [rows][20][20][32] fp32 (may be nullptr for the target network)
  __half* out16[2];          // hi planes
  int64_t lo_off;            // lo plane = hi + lo_off (elements)
  uint8_t* im2col;           // online network's A tiles [rows * 4][4][16 KB] (nullptr = off)
};

__device__ __forceinline__ void tma_load_3d(uint32_t smem_dst, const CUtensorMap* map, int c0, int c1, int c2,
                                            uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

// which k-block of network z multiplies the tile of slot j (frame f of window b); -1: none
__device__ __forceinline__ int kb_for(const Params& p, int nets, int b, int f, int z) {
  int kb;
  if (p.shared5) kb = f - z;                     // online: frame f is k-block f; target: k-block f - 1
  else if (nets == 2 && b != z) return -1;       // staged: window b belongs to network b
  else kb = f;
  return (kb >= 0 && kb < kHist) ? kb : -1;
}

__global__ void __launch_bounds__(umma2::kThreads2, 2)
k_conv1_tma(const __grid_constant__ CUtensorMap map0, const __grid_constant__ CUtensorMap map1, const Params p,
            const KTrace kt) {
  using umma2::kLoadThreads;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t s_box[2];          // windows have landed
  __shared__ __align__(8) uint64_t s_full[kRing];     // A tile converted + weight tiles landed

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const int n = blockIdx.x / kTilesPerSample, t = blockIdx.x % kTilesPerSample;
  kt_begin(kt);
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  const uint32_t box_base = smem_base + kRing * kStage;
  const int nets = p.nets;
  const int nboxes = (nets == 2 && !p.shared5) ? 2 : 1;
  const int box_frames = (nets == 2 && p.shared5) ? kHist + 1 : kHist;
  const int nslots = nboxes * box_frames;          // 4 (predict), 5 (ring train), 8 (staged train)

  if (tid == 0) {
    mbar_init(&s_box[0], 1);
    mbar_init(&s_box[1], 1);
#pragma unroll
    for (int s = 0; s < kRing; ++s) mbar_init(&s_full[s], kLoadThreads + 1);
    mbar_fence_init();
  }
  __syncthreads();

  // weight tiles of slot j into its stage (thread 0): they do not depend on the predecessor kernel
  auto fetch_weights = [&](int j) {
    const int s = j % kRing, b = j / box_frames, f = j % box_frames;
    uint32_t bytes = 0;
    for (int z = 0; z < nets; ++z) bytes += kb_for(p, nets, b, f, z) >= 0 ? kWTile : 0u;
    mbar_arrive_expect_tx(&s_full[s], bytes);
    for (int z = 0; z < nets; ++z) {
      const int kb = kb_for(p, nets, b, f, z);
      if (kb >= 0) tma_bulk_g2s(smem_gen + s * kStage + kATile + z * kWTile, p.wimg[z] + kb * kWTile, kWTile, &s_full[s]);
    }
  };
  if (tid == 0) {
    tma_prefetch_desc(&map0);
    if (nboxes == 2) tma_prefetch_desc(&map1);
    for (int j = 0; j < kRing && j < nslots; ++j) fetch_weights(j);
  }
  pdl_wait();   // the sampled indexes come from the predecessor
  if (tid == 0) {
    for (int b = 0; b < nboxes; ++b) {
      const int frame = p.idx[b][n] + p.shift[b];
      mbar_arrive_expect_tx(&s_box[b], uint32_t(box_frames) * kFrameBoxBytes);
      tma_load_3d(box_base + b * kBoxStride, b ? &map1 : &map0, 0, t * 5, frame, &s_box[b]);
    }
  }

  // chunk (row, r): the 8 taps of filter row r for output pixel `row` = 8 consecutive bytes of window row 4*pl + r
  int src_off[4];
  uint32_t dst_off[4];
  bool live[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int id = tid + i * kLoadThreads;
    const int row = id >> 3, r = id & 7;
    const int pl = row / 20, q = row % 20;
    live[i] = row < kTileRows;
    src_off[i] = (4 * pl + r) * kFrameW + 4 * q;
    dst_off[i] = umma::sw128_off(row, r);
  }
  float acc[2][32];   // per network: the N = 64 fragment [acc_hi (32 channels) | acc_lo (32 channels)]
#pragma unroll
  for (int z = 0; z < 2; ++z)
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[z][i] = 0.f;
  for (int j = 0; j < nslots; ++j) {
    const int s = j % kRing, b = j / box_frames, f = j % box_frames;
    if (f == 0) mbar_wait(&s_box[b], 0);
    if (j >= kRing) {
      // both warpgroups are past the wgmma.wait_group that completed slot j - kRing's MMAs (and thread 0 waited for
      // its im2col store to read the stage): the stage takes slot j
      umma2::named_bar_sync(1, kLoadThreads);
      if (tid == 0) fetch_weights(j);
    }
    // ---- window -> fp16 tile (all 8 warps)
    const uint8_t* win = smem_gen + (box_base - smem_base) + b * kBoxStride + f * kFrameBoxBytes;
    uint8_t* tile = smem_gen + s * kStage;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      uint4 hi = make_uint4(0u, 0u, 0u, 0u);
      if (live[i]) {
        const uint32_t x = *reinterpret_cast<const uint32_t*>(win + src_off[i]);
        const uint32_t y = *reinterpret_cast<const uint32_t*>(win + src_off[i] + 4);
        // u8 -> fp16 is exact: 0x6400 | v is the half 1024 + v; subtract 1024
        const __half2 k1024 = __half2half2(__ushort_as_half(0x6400));
        const uint32_t a0 = 0x64006400u | (x & 0xffu) | ((x & 0xff00u) << 8);
        const uint32_t a1 = 0x64006400u | ((x >> 16) & 0xffu) | ((x >> 8) & 0xff0000u);
        const uint32_t a2 = 0x64006400u | (y & 0xffu) | ((y & 0xff00u) << 8);
        const uint32_t a3 = 0x64006400u | ((y >> 16) & 0xffu) | ((y >> 8) & 0xff0000u);
        __half2 h0 = __hsub2(*reinterpret_cast<const __half2*>(&a0), k1024);
        __half2 h1 = __hsub2(*reinterpret_cast<const __half2*>(&a1), k1024);
        __half2 h2 = __hsub2(*reinterpret_cast<const __half2*>(&a2), k1024);
        __half2 h3 = __hsub2(*reinterpret_cast<const __half2*>(&a3), k1024);
        hi = make_uint4(*reinterpret_cast<uint32_t*>(&h0), *reinterpret_cast<uint32_t*>(&h1),
                        *reinterpret_cast<uint32_t*>(&h2), *reinterpret_cast<uint32_t*>(&h3));
      }
      *reinterpret_cast<uint4*>(tile + dst_off[i]) = hi;
    }
    fence_proxy_async_smem();   // st.shared (generic proxy) -> async proxy, writer side
    mbar_arrive(&s_full[s]);
    // ---- MMAs of the slot: each warpgroup multiplies its 64 pixel rows by the weights of every network that uses
    // this frame (M = 64, N = 64 = [W_hi ; W_lo] in one instruction)
    mbar_wait(&s_full[s], (j / kRing) & 1);
    fence_proxy_async_smem();
    const uint32_t stage = smem_base + s * kStage;
    const uint64_t da = umma::make_desc_sw128(stage + wg * (umma::kWgM * 128));
    umma::wgmma_fence();
#pragma unroll
    for (int z = 0; z < 2; ++z) {
      const int kb = z < nets ? kb_for(p, nets, b, f, z) : -1;
      if (kb < 0) continue;
      const uint64_t db = umma::make_desc_sw128(stage + kATile + z * kWTile);
#pragma unroll
      for (int k = 0; k < 4; ++k) umma::wgmma_f16<64>(acc[z], da + 2 * k, db + 2 * k);
    }
    umma::wgmma_commit();
    if (tid == 0 && p.im2col) {
      const int kb = kb_for(p, nets, b, f, 0);
      if (kb >= 0) {   // the online network's tile IS conv1_wgrad's MN-major A operand
        tma_bulk_s2g(p.im2col + (int64_t(blockIdx.x) * 4 + kb) * kATile, smem_gen + s * kStage, kATile);
        tma_bulk_commit();
        if (j + kRing < nslots) tma_bulk_wait_read_all();   // the stage is about to be overwritten
      }
    }
    umma::wgmma_wait<1>();
  }
  pdl_launch_dependents();
  if (tid == 0 && p.im2col) tma_bulk_wait_read_all();   // shared memory must outlive the im2col stores' reads

  // ---- epilogue straight from the accumulator fragments: x 1/255, Rectlin, fp32 + hi/lo planes
  umma::wgmma_wait<0>();
#pragma unroll
  for (int z = 0; z < 2; ++z) {
    if (z >= nets) break;
#pragma unroll
    for (int i = 0; i < 16; i += 2) {   // registers [0, 16) = channels 0..31 of acc_hi; acc_lo 16 registers further
      const int row = wg * umma::kWgM + umma::frag_row(i, lane, warp), c = umma::frag_col(i, lane);
      if (row < kTileRows) {
        const float o0 = fmaxf(fmaf(acc[z][16 + i], umma::kLoInv, acc[z][i]) * (1.0f / 255.0f), 0.f);
        const float o1 = fmaxf(fmaf(acc[z][17 + i], umma::kLoInv, acc[z][i + 1]) * (1.0f / 255.0f), 0.f);
        const int64_t e = (int64_t(n) * (kP1 * kP1) + t * kTileRows + row) * kC1 + c;
        if (p.out[z]) *reinterpret_cast<float2*>(p.out[z] + e) = make_float2(o0, o1);
        const __half2 hh = __floats2half2_rn(o0, o1);
        const float2 back = __half22float2(hh);
        *reinterpret_cast<__half2*>(p.out16[z] + e) = hh;
        *reinterpret_cast<__half2*>(p.out16[z] + p.lo_off + e) =
            __floats2half2_rn((o0 - back.x) * umma::kLoScale, (o1 - back.y) * umma::kLoScale);
      }
    }
  }
  kt_end(kt);
}

// ---- host: tensor map over a frame array [frames][84][84] u8 as [frames][21][84 x u32]
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static inline EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* sym = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(sym);
  }
  return fn;
}

static inline int make_frame_map(CUtensorMap* map, const uint8_t* frames, int64_t nframes, int box_frames) {
  EncodeTiledFn fn = encode_fn();
  B2_REQUIRE(fn, B200DQN_ECUDA, "cuTensorMapEncodeTiled is not available from this driver");
  B2_REQUIRE((reinterpret_cast<uintptr_t>(frames) & 15) == 0, B200DQN_EINVAL, "frame array must be 16-byte aligned for TMA");
  const cuuint64_t dims[3] = {cuuint64_t(kGroupBytes / 4), cuuint64_t(kFrameH / 4), cuuint64_t(nframes)};   // 84 u32, 21 groups
  const cuuint64_t strides[2] = {cuuint64_t(kGroupBytes), cuuint64_t(kFrameBytes)};
  const cuuint32_t box[3] = {cuuint32_t(kGroupBytes / 4), cuuint32_t(kBoxGroups), cuuint32_t(box_frames)};
  const cuuint32_t estr[3] = {1, 1, 1};
  const CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, const_cast<uint8_t*>(frames), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  B2_REQUIRE(r == CUDA_SUCCESS, B200DQN_ECUDA, "cuTensorMapEncodeTiled failed (%d)", int(r));
  return B200DQN_OK;
}

}  // namespace conv1tma
}  // namespace b200
