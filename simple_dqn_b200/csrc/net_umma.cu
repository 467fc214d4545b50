// net_umma.cu — math_mode TCGEN05 (the name is historical): the GEMM-shaped ops of the Nature-DQN step on the
// Hopper tensor cores (wgmma.mma_async, register accumulators): forward + dgrad through the K-major kernel of
// umma2.cuh, wgrad through the MN-major kernel of umma_mn.cuh, plus the fused optimizer / tile-image
// kernels.  Same fp32 HBM tensors as the SIMT engine (net_simt.cuh), so every kernel here is checked
// against its SIMT twin and against the CPU oracle.
#include "net.cuh"
#include "net_umma.cuh"
#include "umma.cuh"
#include "umma2.cuh"
#include "umma_mn.cuh"

namespace b200 {

__device__ __forceinline__ void ld8(const float* p, float v[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p);
  const float4 b = *reinterpret_cast<const float4*>(p + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void st8(float* p, const float v[8]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
}
__device__ __forceinline__ void zero8(float v[8]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) v[i] = 0.f;
}

// ==========================================================================================
// Engine v2 (umma2.cuh): pre-split fp16 hi/lo operand planes + weight tile images.
// ==========================================================================================
struct UmmaState {
  // activation planes per net: [hi plane | lo plane], NHWC fp16
  __half* h16[3][3] = {};     // H1, H2, H3  x  network slot (online, target, online on the poststates: Double DQN only)
  int64_t h_elems[3] = {};
  __half* dz16[4] = {};       // dZ4, dZ3, dZ2, dZ1 (online)
  int64_t dz_elems[4] = {};
  // weight tile images ([hi | lo] per (tile, k-block))
  uint8_t* img_fwd[2][4] = {};  // conv1, conv2, conv3, fc1  x  (online, target)
  int64_t img_fwd_bytes[4] = {};
  uint8_t* im2col1 = nullptr;   // conv1_fwd's A_hi tiles of the online net: [ceil(nb*400/128)][H][16 KB]
  uint8_t* img_dgr[3] = {};     // fc1_dgrad (A operand), conv3_dgrad (B), conv2_dgrad (B, 4 parity classes)
};
static inline UmmaState* ust(b200dqn_net* n) { return static_cast<UmmaState*>(n->umma_state); }

// f(std::integral_constant<int, H>{}) for H = hist in 1..kMaxHist: conv1's kernels take the history length as a template
// argument, so its k-block count, M extent and parameter count are compile-time constants.  One source path for every H;
// a run-time H made conv1_fwd's refill path live for every H (72 -> 110 registers) and the batch-32 step 0.6 us slower
// at H = 4 (H100 80GB HBM3, 400 W).
template <int H = 1, class F>
static auto with_hist(int hist, F&& f) -> decltype(f(std::integral_constant<int, 1>{})) {
  if constexpr (H == kMaxHist) {
    return f(std::integral_constant<int, H>{});   // net_create admits 1..kMaxHist only
  } else {
    if (hist == H) return f(std::integral_constant<int, H>{});
    return with_hist<H + 1>(hist, f);
  }
}

struct PlanePair {
  __half* hi;
  int64_t lo_off;   // lo plane = hi + lo_off
};

// Network slots of a train-step forward (blockIdx z of k_umma2, y of k_conv23_fwd; slot3 / wslot in net_simt.cuh): slot
// 2 reads slot 1's frames, the online network's weight images and has its own fp16 planes.
__device__ __forceinline__ void store_f32_and_planes(float* f32, const PlanePair& pl, int64_t i, const float v[8]) {
  if (f32) st8(f32 + i, v);
  umma2::split8_planes(v, pl.hi + i, pl.hi + pl.lo_off + i);
}

// ---- forward -----------------------------------------------------------------------------
// H = history_length, a template argument (see with_hist): H k-blocks of 64 taps (8x8 pixels), one per frame.  Up to
// kStages frames every k-block has its own ring stage, and the loads of later k-blocks compile away.
template <int H>
struct V2Conv1Fwd {
  static constexpr int kBN = 32;
  static constexpr bool kAExact = true, kARowMajorThreads = true, kBRowMajorThreads = false;
  static constexpr int kAMode = umma2::kReg, kBMode = umma2::kBulk;
  static constexpr bool kStagedEpilogue = true, kDumpA = true, kPrefetch = false;
  uint8_t* im2col;          // online net only: [mtile][H kb][128 x 128 B] A_hi tiles for conv1_wgrad (nullptr = off)
  const uint8_t* src[2];    // frame sources of slots 0 and 1; slot 2 reads slot 1's
  const int32_t* idx[2];
  int shift[2];
  const uint8_t* wimg[2];   // [H kb][hi 32x128 | lo 32x128]
  float* out[3];
  PlanePair out16[3];
  int rows;
  __device__ int M(int) const { return rows * kP1 * kP1; }
  __device__ int N(int) const { return kC1; }
  __device__ void krange(int, int& kb, int& ke) const { kb = 0; ke = H; }
  // first byte of output pixel m's receptive field in frame 0 of its sample (nullptr = padding row)
  __device__ const uint8_t* a_row_ptr(int z, int m) const {
    if (m >= rows * kP1 * kP1) return nullptr;
    const int n = m / (kP1 * kP1), pq = m % (kP1 * kP1), p = pq / kP1, q = pq % kP1;
    const int64_t f = static_cast<int64_t>((z ? idx[1] : idx[0])[n]) + (z ? shift[1] : shift[0]);
    return (z ? src[1] : src[0]) + f * kFrameBytes + (p * 4) * kFrameW + q * 4;
  }
  __device__ uint2 a_raw8(const uint8_t* row, int k0) const {   // k0 = (c, r, 0): 8 pixels of filter row r, frame c
    if (!row) return make_uint2(0u, 0u);
    const int c = k0 >> 6, r = (k0 >> 3) & 7;
    const uint8_t* ptr = row + c * kFrameBytes + r * kFrameW;
    return make_uint2(*reinterpret_cast<const uint32_t*>(ptr), *reinterpret_cast<const uint32_t*>(ptr + 4));
  }
  __device__ static void cvt8(uint2 raw, float v[8]) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      v[j] = float((raw.x >> (8 * j)) & 0xffu);
      v[4 + j] = float((raw.y >> (8 * j)) & 0xffu);
    }
  }
  __device__ const uint8_t* b_tile(int z, int, int kb) const { return wslot(wimg, z) + kb * (kC1 * 256); }
  __device__ uint8_t* a_dump(int z, int mtile, int kb) const {
    return (z == 0 && im2col) ? im2col + (int64_t(mtile) * H + kb) * (128 * 128) : nullptr;
  }
  __device__ void store8(int z, int m, int n0, const float v[8]) const {
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = fmaxf(v[j] * (1.0f / 255.0f), 0.f);
    store_f32_and_planes(slot3(out, z), slot3(out16, z), int64_t(m) * kC1 + n0, o);
  }
};

// conv1 forward on shifted states (random_shift > 0; b200dqn.h has the rule): the same kernel with the crop offsets
// applied in the gather, so the im2col tiles it dumps for conv1_wgrad hold the shifted pixels and the wgrad needs no
// change.  crop[z] = [nb][2] (dy, dx) of frame source z; slot 2 reads slot 1's frames and offsets.
struct CropRow {
  const uint8_t* frame;   // frame 0 of the row's sample (nullptr = padding row)
  int y0;                 // top filter row before the clamp: p * 4 + dy
  int wa;                 // first 32-bit word of the clamped columns
  uint32_t sel;           // byte selectors of the 8 columns (see a_raw8)
};
template <int H>
struct V2Conv1FwdCrop : V2Conv1Fwd<H> {
  const int32_t* crop[2];
  // Columns x0 + j (j < 8), x0 = q * 4 + dx, clamp to [0, 83]; relative to word wa they are rel_j in [0, 11], rising
  // with j.  rel_0..3 lie in words wa, wa + 1 (rel <= 6); rel_4..7 lie either there (rel_4 < 4) or in words wa + 1,
  // wa + 2.  sel packs the four 4-bit selectors of each output word for __byte_perm.
  __device__ CropRow a_row_ptr(int z, int m) const {
    if (m >= this->rows * kP1 * kP1) return CropRow{nullptr, 0, 0, 0u};
    const int n = m / (kP1 * kP1), pq = m % (kP1 * kP1), p = pq / kP1, q = pq % kP1;
    const int32_t* c = z ? crop[1] : crop[0];
    const int64_t f = static_cast<int64_t>((z ? this->idx[1] : this->idx[0])[n]) + (z ? this->shift[1] : this->shift[0]);
    const int x0 = q * 4 + c[2 * n + 1];
    const int wa = min(max(x0, 0), kFrameW - 1) >> 2;
    uint32_t sel = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) sel |= uint32_t(min(max(x0 + j, 0), kFrameW - 1) - 4 * wa) << (4 * j);
    return CropRow{(z ? this->src[1] : this->src[0]) + f * kFrameBytes, p * 4 + c[2 * n], wa, sel};
  }
  // Only aligned 32-bit words of the clamped row, and of words 0..20 of it, are read: no byte outside the frame.
  __device__ uint2 a_raw8(const CropRow& row, int k0) const {
    if (!row.frame) return make_uint2(0u, 0u);
    const int c = k0 >> 6, r = (k0 >> 3) & 7;
    const int y = min(max(row.y0 + r, 0), kFrameH - 1);
    const uint32_t* line = reinterpret_cast<const uint32_t*>(row.frame + c * kFrameBytes + y * kFrameW);
    constexpr int kLastWord = kFrameW / 4 - 1;
    const uint32_t w0 = line[row.wa], w1 = line[min(row.wa + 1, kLastWord)], w2 = line[min(row.wa + 2, kLastWord)];
    const uint32_t shi = row.sel >> 16;
    const uint32_t hi = (shi & 0xfu) >= 4u ? __byte_perm(w1, w2, shi - 0x4444u) : __byte_perm(w0, w1, shi);
    return make_uint2(__byte_perm(w0, w1, row.sel & 0xffffu), hi);
  }
};

template <int H, int C, int R, int ST, int KO>
struct V2ConvFwd {
  static constexpr int P = (H - R) / ST + 1, K = R * R * C;
  static_assert(K % 64 == 0 && C % 8 == 0, "k-blocks of 64, chunks of 8 channels");
  static constexpr int kBN = KO;
  static constexpr bool kAExact = false, kARowMajorThreads = true, kBRowMajorThreads = false;
  static constexpr int kAMode = umma2::kAsync, kBMode = umma2::kBulk;
  static constexpr bool kStagedEpilogue = true, kDumpA = false, kPrefetch = false;
  PlanePair in16[3];
  const uint8_t* wimg[2];   // [K/64][hi KOx128 | lo KOx128]
  float* out[3];
  PlanePair out16[3];
  int rows;
  __device__ int M(int) const { return rows * P * P; }
  __device__ int N(int) const { return KO; }
  __device__ void krange(int, int& kb, int& ke) const { kb = 0; ke = K / 64; }
  __device__ umma2::Planes a_planes(int z) const { return {slot3(in16, z).hi, in16[0].lo_off}; }
  __device__ umma2::RowCtx a_row(int, int m) const {
    const int n = m / (P * P), pq = m % (P * P), p = pq / P, q = pq % P;
    return {(int64_t(n * H + p * ST) * H + q * ST) * C, 0, 0, m < rows * P * P};
  }
  __device__ bool a_chunk(int, const umma2::RowCtx& rc, int kk, int64_t& off) const {
    const int r = kk / (R * C), sc = kk % (R * C);
    off = rc.base + r * (H * C) + sc;
    return true;
  }
  __device__ const uint8_t* b_tile(int z, int, int kb) const { return wslot(wimg, z) + kb * (KO * 256); }
  __device__ void store8(int z, int m, int n0, const float v[8]) const {
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = fmaxf(v[j], 0.f);
    store_f32_and_planes(slot3(out, z), slot3(out16, z), int64_t(m) * KO + n0, o);
  }
};

// ---- conv2 + conv3 forward, one CTA per (sample, network slot) --------------------------------------
// conv3's receptive field never leaves a sample, so one CTA runs conv2 on its sample (81 live rows of a 128-row tile,
// the k_umma2 pipeline), keeps H2 in shared memory as fp16 hi/lo rows and runs conv3 on it (49 live rows of one
// 64-row wgmma tile, one k-block per filter tap): no CTA waits on another, and the conv2 -> conv3 link of the chain
// (grid drain, dependency release, first loads) is gone.  Operand bits, k-block order and the MMAs each output
// element sees are those of the two V2ConvFwd launches, so the results are the same bits.
struct Conv23Fwd {
  using C2 = V2ConvFwd<kP1, kC1, 4, 2, kC2>;   // conv2: gather addressing of H1; out / out16 = H2 of the online net
  using C3 = V2ConvFwd<kP2, kC2, 3, 1, kC3>;   // conv3: wimg, out / out16 = H3 (in16 unused: H2 stays on chip)
  C2 c2;
  C3 c3;
};

namespace conv23 {
constexpr int kStages = 4;                               // conv2 ring
constexpr int kM2 = kP2 * kP2, kM3 = kP3 * kP3;          // live rows: 81 of 128, 49 of 64
constexpr int kKb2 = kK2 / 64, kKb3 = kK3 / 64;          // 8, 9
constexpr uint32_t kA2 = umma::kBM * 128;                // conv2 A_hi tile (A_lo follows)
constexpr uint32_t kB2 = kC2 * 128;                      // conv2 B_hi tile (B_lo follows)
constexpr uint32_t kStage2 = 2 * kA2 + 2 * kB2;          // 48 KB
constexpr uint32_t kB3 = kC3 * 256;                      // conv3 weight image of one tap: [hi 64 rows | lo 64 rows]
constexpr uint32_t kA3 = umma::kWgM * 128;               // conv3 A_hi tile (A_lo follows)
// Shared memory, from the 1024-aligned base: the conv2 ring; once a conv2 stage is retired it takes the weight images
// of three conv3 taps (stages 0-2 hold all nine), while stage 3 takes conv2's epilogue tile and then conv3's 3-deep
// A ring; behind the ring the H2 rows of the sample, [hi 81 x 128 B | lo 81 x 128 B].
constexpr uint32_t kStaging = 3 * kStage2;
constexpr uint32_t kH2 = kStages * kStage2;
constexpr uint32_t kPitch2 = kC2 * 4 + 16, kPitch3 = kC3 * 4 + 16;   // epilogue tile rows (bytes)
constexpr uint32_t kSmemBytes = kH2 + 2 * kM2 * 128 + 1024;
static_assert(kKb3 * kB3 == 3 * kStage2, "stages 0-2 of the conv2 ring hold the nine conv3 weight images");
static_assert(kStaging + umma::kBM * kPitch2 <= kH2 && kStaging + 3 * 2 * kA3 <= kH2, "stage 3: epilogue tile, A ring");
static_assert(umma::kWgM * kPitch3 <= kStaging, "conv3 epilogue tile over the retired weight images");
static_assert(kSmemBytes <= 227 * 1024, "H100: at most 227 KB of shared memory per block");
}  // namespace conv23

// Trace stamps (B200DQN_TRACE_LABEL=conv23_fwd): 0 start, 1 barriers ready, 3 conv2 MMAs issued, 4 conv2 accumulators
// ready, 2 H2 in shared memory, 7 conv3 accumulators ready, 5 H3 stored, 6 end; k-block rows 8 + 4 * it as in
// k_umma2, conv2's it = 0..7 and conv3's it = 8..16 (conv3 stamps [it][2] when it starts copying its A tile).
__global__ void __launch_bounds__(umma2::kThreads2, 1) k_conv23_fwd(const Conv23Fwd p, const int trace_in,
                                                                    const KTrace kt) {
  using namespace conv23;
  using umma2::g_trace;
  using umma2::kTraceSlots;
  constexpr int S = kStages;
  constexpr int kThreads = umma2::kThreads2;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t s_full[S];      // conv2: operands of the stage have landed
  __shared__ __align__(8) uint64_t s_w3[kKb3];     // conv3: weight image of tap kb has landed

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const int n = blockIdx.x, z = blockIdx.y;
  const bool trace = trace_in && n == 0 && z == 0;
  kt_begin(kt);
  B2_TRACE(tid == 0, 0);
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  uint8_t* h2 = smem_gen + kH2;
  const uint8_t* wimg2 = wslot(p.c2.wimg, z);
  const uint8_t* wimg3 = wslot(p.c3.wimg, z);

  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < S; ++s) mbar_init(&s_full[s], kThreads + 1);
#pragma unroll
    for (int kb = 0; kb < kKb3; ++kb) mbar_init(&s_w3[kb], 1);
    mbar_fence_init();
  }
  __syncthreads();
  B2_TRACE(tid == 0, 1);

  // conv2 gather rows of this thread (sample-local row m = id >> 3; rows 81..127 are zero-filled)
  constexpr int kACh = umma::kBM * 8 / kThreads;
  umma2::RowCtx arow[kACh];
  const umma2::Planes apl = p.c2.a_planes(z);
#pragma unroll
  for (int i = 0; i < kACh; ++i) {
    const int m = (tid + i * kThreads) >> 3;
    arow[i] = p.c2.a_row(z, n * kM2 + m);
    arow[i].ok = m < kM2;
  }
  // conv2's first S weight tiles do not depend on the predecessor kernel: in flight before the dependency wait
  if (tid == 0) {
#pragma unroll
    for (int j = 0; j < S; ++j) {
      mbar_arrive_expect_tx(&s_full[j], 2 * kB2);
      tma_bulk_g2s(smem_gen + j * kStage2 + 2 * kA2, wimg2 + j * (2 * kB2), 2 * kB2, &s_full[j]);
    }
  }
  pdl_wait();

  // conv2 operands of k-block j into stage j % S
  auto stage2 = [&](int j) {
    const int s = j % S, k0 = j * umma::kBK;
    B2_TRACE(tid == 0, 8 + j * 4 + 2);
    const uint32_t a_hi = smem_base + s * kStage2, a_lo = a_hi + kA2;
    if (tid == 0 && j >= S) {
      mbar_arrive_expect_tx(&s_full[s], 2 * kB2);
      tma_bulk_g2s(smem_gen + s * kStage2 + 2 * kA2, wimg2 + j * (2 * kB2), 2 * kB2, &s_full[s]);
    }
#pragma unroll
    for (int i = 0; i < kACh; ++i) {
      const int id = tid + i * kThreads, r = id >> 3, c = id & 7;
      int64_t eoff = 0;
      const bool ok = arow[i].ok && p.c2.a_chunk(z, arow[i], k0 + c * 8, eoff);
      const uint32_t bytes = ok ? 16u : 0u;
      const __half* hi = apl.hi + (ok ? eoff : 0);
      const uint32_t off = umma::sw128_off(r, c);
      umma2::cp_async16(a_hi + off, hi, bytes);
      umma2::cp_async16(a_lo + off, hi + apl.lo_off, bytes);
    }
    umma2::cp_async_arrive_noinc(&s_full[s]);
    B2_TRACE(tid == 0, 8 + j * 4 + 3);
  };
  for (int j = 0; j < S; ++j) stage2(j);

  // ================================================================ conv2 mainloop (as k_umma2, BN = 64)
  float acc[kC2];          // N = 128 fragment: [A_hi x B_hi | A_hi x B_lo]
  float acc2[kC2 / 2];     // N = 64 fragment: A_lo x B_hi
#pragma unroll
  for (int i = 0; i < kC2; ++i) acc[i] = 0.f;
#pragma unroll
  for (int i = 0; i < kC2 / 2; ++i) acc2[i] = 0.f;
  for (int it = 0; it < kKb2; ++it) {
    const int s = it % S;
    mbar_wait(&s_full[s], (it / S) & 1);
    fence_proxy_async_smem();
    B2_TRACE(tid == 0, 8 + it * 4 + 0);
    const uint32_t sa = smem_base + s * kStage2;
    const uint64_t da_hi = umma::make_desc_sw128(sa + wg * umma::kWgM * 128);
    const uint64_t da_lo = umma::make_desc_sw128(sa + kA2 + wg * umma::kWgM * 128);
    const uint64_t db = umma::make_desc_sw128(sa + 2 * kA2);
    umma::wgmma_fence();
#pragma unroll
    for (int k = 0; k < umma::kBK / 16; ++k) {
      umma::wgmma_f16<2 * kC2>(acc, da_hi + 2 * k, db + 2 * k);
      umma::wgmma_f16<kC2>(acc2, da_lo + 2 * k, db + 2 * k);
    }
    umma::wgmma_commit();
    umma::wgmma_wait<1>();
    B2_TRACE(tid == 0, 8 + it * 4 + 1);
    if (it >= 1) {
      umma2::named_bar_sync(1, kThreads);   // both warpgroups are done with k-block it-1: its stage is free
      const int freed = (it - 1) % S;
      if (it - 1 + S < kKb2) {
        stage2(it - 1 + S);
      } else if (tid == 0) {              // conv2 is done with stage `freed`: it takes the images of conv3 taps 3*freed..+2
#pragma unroll
        for (int t = 0; t < 3; ++t) {
          const int kb = 3 * freed + t;
          mbar_arrive_expect_tx(&s_w3[kb], kB3);
          tma_bulk_g2s(smem_gen + kb * kB3, wimg3 + kb * kB3, kB3, &s_w3[kb]);
        }
      }
    }
  }
  B2_TRACE(tid == 0, 3);
  // Every load of the kernel has been issued: fc1_fwd may pre-launch.  On an H100 80GB HBM3 (400 W) this was 0.5 us
  // faster at batch 32 than releasing right after the dependency wait.
  pdl_launch_dependents();

  // ================================================================ conv2 epilogue: H2 -> shared memory (+ HBM)
  umma::wgmma_wait<0>();
  umma2::named_bar_sync(1, kThreads);     // stage 3 (the epilogue tile) is no longer read by the MMAs
  B2_TRACE(tid == 0, 4);
  umma::stage_acc<kC2>(acc, acc2, smem_gen + kStaging, kPitch2, wg, warp, lane);
  umma2::named_bar_sync(1, kThreads);
  {
    float* out = p.c2.out[0];
    const PlanePair pl = p.c2.out16[0];
#pragma unroll
    for (int i = 0; i < umma::kBM * 8 / kThreads; ++i) {
      const int id = tid + i * kThreads, r = id >> 3, cc = id & 7;
      if (r < kM2) {
        const uint8_t* src = smem_gen + kStaging + r * kPitch2 + cc * 32;
        const float4 v0 = *reinterpret_cast<const float4*>(src), v1 = *reinterpret_cast<const float4*>(src + 16);
        const float v[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = fmaxf(v[j], 0.f);
        uint4 hi, lo;
        umma::split8(o, hi, lo);
        *reinterpret_cast<uint4*>(h2 + r * 128 + cc * 16) = hi;
        *reinterpret_cast<uint4*>(h2 + kM2 * 128 + r * 128 + cc * 16) = lo;
        if (z == 0) {   // conv2_dgrad reads the fp32 H2 (Rectlin mask), conv3_wgrad the planes; the target's H2 has no reader
          const int64_t e = int64_t(n * kM2 + r) * kC2 + cc * 8;
          if (out) st8(out + e, o);
          *reinterpret_cast<uint4*>(pl.hi + e) = hi;
          *reinterpret_cast<uint4*>(pl.hi + pl.lo_off + e) = lo;
        }
      }
    }
  }
  umma2::named_bar_sync(1, kThreads);     // H2 complete; the epilogue tile is free for the A ring
  B2_TRACE(tid == 0, 2);

  // ================================================================ conv3 mainloop
  // Tap kb = (r, s): A row m = (p, q) is H2 row (p + r, q + s), copied into a SW128 tile (rows 49..63 zero).  Each
  // warpgroup takes 32 output channels: per k-step three N = 32 wgmmas, A_hi x B_hi, A_hi x B_lo and A_lo x B_hi.
  float acc3[kC3 / 2];     // [A_hi x B_hi | A_hi x B_lo] laid out as one N = 64 fragment (stage_acc<32>)
  float acc3l[kC3 / 4];    // A_lo x B_hi
#pragma unroll
  for (int i = 0; i < kC3 / 2; ++i) acc3[i] = 0.f;
#pragma unroll
  for (int i = 0; i < kC3 / 4; ++i) acc3l[i] = 0.f;
  for (int it = 0; it < kKb3; ++it) {
    const int r = it / 3, s = it % 3;
    const uint32_t a_off = kStaging + (it % 3) * (2 * kA3);
    B2_TRACE(tid == 0, 8 + (kKb2 + it) * 4 + 2);
    // buffer it % 3 was last read by tap it-3, complete in both warpgroups (wgmma.wait_group 1 of tap it-2, then the
    // barrier of tap it-1)
#pragma unroll
    for (int i = 0; i < umma::kWgM * 8 / kThreads; ++i) {
      const int id = tid + i * kThreads, m = id >> 3, c = id & 7;
      uint4 hi = make_uint4(0u, 0u, 0u, 0u), lo = hi;
      if (m < kM3) {
        const int src = (m / kP3 + r) * kP2 + m % kP3 + s;
        hi = *reinterpret_cast<const uint4*>(h2 + src * 128 + c * 16);
        lo = *reinterpret_cast<const uint4*>(h2 + kM2 * 128 + src * 128 + c * 16);
      }
      *reinterpret_cast<uint4*>(smem_gen + a_off + umma::sw128_off(m, c)) = hi;
      *reinterpret_cast<uint4*>(smem_gen + a_off + kA3 + umma::sw128_off(m, c)) = lo;
    }
    fence_proxy_async_smem();               // st.shared (generic proxy) -> wgmma operand reads (async proxy)
    umma2::named_bar_sync(1, kThreads);     // both warpgroups read the whole A tile
    mbar_wait(&s_w3[it], 0);
    B2_TRACE(tid == 0, 8 + (kKb2 + it) * 4 + 0);
    const uint64_t da_hi = umma::make_desc_sw128(smem_base + a_off);
    const uint64_t da_lo = umma::make_desc_sw128(smem_base + a_off + kA3);
    const uint32_t b = smem_base + it * kB3 + wg * 32 * 128;   // this warpgroup's 32 rows: 1024-byte aligned
    const uint64_t db_hi = umma::make_desc_sw128(b), db_lo = umma::make_desc_sw128(b + kC3 * 128);
    umma::wgmma_fence();
#pragma unroll
    for (int k = 0; k < umma::kBK / 16; ++k) {
      umma::wgmma_f16<32>(acc3, da_hi + 2 * k, db_hi + 2 * k);
      umma::wgmma_f16<32>(acc3 + kC3 / 4, da_hi + 2 * k, db_lo + 2 * k);
      umma::wgmma_f16<32>(acc3l, da_lo + 2 * k, db_hi + 2 * k);
    }
    umma::wgmma_commit();
    umma::wgmma_wait<1>();
    B2_TRACE(tid == 0, 8 + (kKb2 + it) * 4 + 1);
  }

  // ================================================================ conv3 epilogue (V2ConvFwd::store8 of conv3_fwd)
  umma::wgmma_wait<0>();
  umma2::named_bar_sync(1, kThreads);     // the weight images are no longer read: the epilogue tile goes over them
  B2_TRACE(tid == 0, 7);
  umma::stage_acc<32>(acc3, acc3l, smem_gen + wg * 32 * 4, kPitch3, 0, warp, lane);
  umma2::named_bar_sync(1, kThreads);
#pragma unroll
  for (int i = 0; i < umma::kWgM * 8 / kThreads; ++i) {
    const int id = tid + i * kThreads, m = id >> 3, cc = id & 7;
    if (m < kM3) {
      const uint8_t* src = smem_gen + m * kPitch3 + cc * 32;
      const float4 v0 = *reinterpret_cast<const float4*>(src), v1 = *reinterpret_cast<const float4*>(src + 16);
      const float v[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
      p.c3.store8(z, n * kM3 + m, cc * 8, v);
    }
  }
  B2_TRACE(tid == 0, 5);
  kt_end(kt);
  B2_TRACE(tid == 0, 6);
}

// Up to this many samples the forward runs conv2 and conv3 as conv23_fwd, beyond it as the two V2ConvFwd launches.
// Small minibatches leave most SMs idle and pay for each link of the chain; large ones fill the GPU, and there the
// per-sample tiles (81 of 128 conv2 rows, 49 of 64 conv3 rows live) cost more than the link saves.  tools/period.py on
// an H100 80GB HBM3 at 400 W, median us per step, two-kernel against fused: 88.1 / 84.9 at batch 32,
// 120.4-120.5 / 119.7-122.5 at 64, 191.9-194.9 / 199.5-200.8 at 128, 262.5-262.7 / 274.3-275.3 at 192 and
// 343.6-344.3 / 353.3-354.2 at 256.
constexpr int kConv23MaxRows = 64;

static int launch_conv23(const Conv23Fwd& p, int rows, int nets, cudaStream_t st) {
  static bool configured = false;
  if (!configured) {
    B2_CHECK_CUDA(cudaFuncSetAttribute(k_conv23_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, conv23::kSmemBytes));
    configured = true;
  }
  static const char* trace_label = getenv("B200DQN_TRACE_LABEL");
  const int trace = (trace_label && strcmp(trace_label, "conv23_fwd") == 0) ? 1 : 0;
  B2_CHECK_CUDA(launch_pdl(k_conv23_fwd, dim3(rows, nets), dim3(umma2::kThreads2), conv23::kSmemBytes, st, p, trace,
                           ktrace_slot("conv23_fwd")));
  B2_PROF("conv23_fwd", st);
  return B200DQN_OK;
}

// W = fc1's width (kHidden, or kDuelHidden on a dueling net) in the fc1 problems, image and update below.
template <int W>
struct V2Fc1Fwd {
  static constexpr int kBN = 32;
  static constexpr bool kAExact = false, kARowMajorThreads = false, kBRowMajorThreads = true;
  static constexpr int kAMode = umma2::kBulk, kBMode = umma2::kAsync;
  static constexpr bool kStagedEpilogue = false, kDumpA = false, kPrefetch = false;   // strided outputs; lanes run along m
  // The weights come from the ROW-oriented fc1 image (the one fc1_dgrad reads K-major: rows = flat index, 64 hidden
  // units per 128-byte row): read with "row = k" it is an M-contiguous (MN-major) A operand, so the forward needs no
  // image of its own and nothing has to be re-packed after the optimizer.
  static constexpr bool kAMnMajor = true;
  static constexpr uint32_t kAMnLoOffset = 128 * 128;   // lo half of a [hi 128x128 B | lo 128x128 B] tile
  PlanePair in16[3];        // H3 planes [rows][3136]
  const uint8_t* wimg[2];   // [25 flat tiles][W / 64 hidden blocks][hi 128x128 | lo 128x128]
  float* part;              // [nets*splits][rows][W]
  int rows, splits;
  __device__ int M(int) const { return W; }
  __device__ int N(int) const { return rows; }
  __device__ void krange(int z, int& kb, int& ke) const {
    const int per = (kFlat / 64 + splits - 1) / splits;
    kb = (z % splits) * per;
    ke = min(kb + per, kFlat / 64);
  }
  // hi sub-tile [64 flat rows x 64 hidden] of hidden block 2*mtile + chunk, flat k-block kb
  __device__ const uint8_t* a_sub(int z, int mtile, int kb, int chunk) const {
    return wslot(wimg, z / splits) + (int64_t(kb >> 1) * (W / 64) + 2 * mtile + chunk) * (128 * 256) +
           (kb & 1) * (64 * 128);
  }
  __device__ umma2::Planes b_planes(int z) const { return {slot3(in16, z / splits).hi, in16[0].lo_off}; }
  __device__ umma2::RowCtx b_row(int, int n) const { return {int64_t(n) * kFlat, 0, 0, n < rows}; }
  __device__ bool b_chunk(int, const umma2::RowCtx& rc, int kk, int64_t& off) const {
    off = rc.base + kk;
    return true;
  }
  __device__ void store8(int z, int m, int n0, const float v[8]) const {
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (n0 + j < rows) part[(z * rows + n0 + j) * W + m] = v[j];
  }
};

// ---- dgrad -------------------------------------------------------------------------------
template <int W>
struct V2Fc1Dgrad {
  static constexpr int kBN = 32;
  static constexpr bool kAExact = false, kARowMajorThreads = true, kBRowMajorThreads = true;
  static constexpr int kAMode = umma2::kBulk, kBMode = umma2::kAsync;
  static constexpr bool kStagedEpilogue = false, kDumpA = false, kPrefetch = true;
  const uint8_t* wimg;   // [25 mtiles][W / 64 kb][hi | lo]   rows m = flat index (p,q,c), K = hidden unit
  PlanePair dz4;         // [rows][W]
  const float* h3;       // [rows][3136] (mask)
  float* dz3;
  PlanePair dz3_16;
  int rows;
  __device__ int M(int) const { return kFlat; }
  __device__ int N(int) const { return rows; }
  __device__ void krange(int, int& kb, int& ke) const { kb = 0; ke = W / 64; }
  __device__ const uint8_t* a_tile(int, int mtile, int kb) const {
    return wimg + (int64_t(mtile) * (W / 64) + kb) * (128 * 256);
  }
  __device__ umma2::Planes b_planes(int) const { return {dz4.hi, dz4.lo_off}; }
  __device__ umma2::RowCtx b_row(int, int n) const { return {int64_t(n) * W, 0, 0, n < rows}; }
  __device__ bool b_chunk(int, const umma2::RowCtx& rc, int kk, int64_t& off) const {
    off = rc.base + kk;
    return true;
  }
  __device__ void prefetch8(int, int m, int n0, float pf[8]) const {   // Rectlin mask of H3
#pragma unroll
    for (int j = 0; j < 8; ++j) pf[j] = (n0 + j < rows) ? h3[int64_t(n0 + j) * kFlat + m] : 0.f;
  }
  __device__ void store8p(int, int m, int n0, const float v[8], const float pf[8]) const {
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (n0 + j < rows) {
        const int64_t i = int64_t(n0 + j) * kFlat + m;
        const float o = pf[j] > 0.f ? v[j] : 0.f;
        if (dz3) dz3[i] = o;
        __half h, l;
        umma2::split1(o, h, l);
        dz3_16.hi[i] = h;
        dz3_16.hi[dz3_16.lo_off + i] = l;
      }
  }
};

template <int H, int C, int R, int ST, int KO, int STG = 0>
struct V2ConvDgrad {
  static constexpr int kStagesOverride = STG;   // 0 = the deepest ring that fits (umma2::Cfg2)
  static constexpr int P = (H - R) / ST + 1, RT = R / ST, HC = (H + ST - 1) / ST, K = RT * RT * KO;
  static_assert(K % 64 == 0 && KO % 8 == 0, "k-blocks of 64");
  static constexpr int kBN = C;
  static constexpr bool kAExact = false, kARowMajorThreads = true, kBRowMajorThreads = true;
  static constexpr int kAMode = umma2::kAsync, kBMode = umma2::kBulk;
  static constexpr bool kStagedEpilogue = true, kDumpA = false, kPrefetch = true;
  PlanePair dz;          // [rows][P][P][KO]
  const uint8_t* wimg;   // [ST*ST classes][K/64][hi Cx128 | lo Cx128]
  const float* x;        // forward activation (mask)
  float* dx;
  PlanePair dx16;        // hi == nullptr -> not needed
  int rows;
  __device__ int M(int) const { return rows * HC * HC; }
  __device__ int N(int) const { return C; }
  __device__ void krange(int, int& kb, int& ke) const { kb = 0; ke = K / 64; }
  __device__ umma2::Planes a_planes(int) const { return {dz.hi, dz.lo_off}; }
  __device__ umma2::RowCtx a_row(int z, int m) const {
    const int n = m / (HC * HC), yx = m % (HC * HC), yy = yx / HC, xx = yx % HC;
    const bool ok = m < rows * HC * HC && yy * ST + z / ST < H && xx * ST + z % ST < H;
    return {(int64_t(n * P + yy) * P + xx) * KO, yy, xx, ok};
  }
  __device__ bool a_chunk(int, const umma2::RowCtx& rc, int kk, int64_t& off) const {
    const int rp = kk / (RT * KO), sp = (kk / KO) % RT, ko = kk % KO;
    const int p = rc.y - rp, q = rc.x - sp;
    off = rc.base - (rp * P + sp) * KO + ko;
    return p >= 0 && p < P && q >= 0 && q < P;
  }
  __device__ const uint8_t* b_tile(int z, int, int kb) const { return wimg + (int64_t(z) * (K / 64) + kb) * (C * 256); }
  __device__ void prefetch8(int z, int m, int c0, float pf[8]) const {   // Rectlin mask: the forward activation
    const int n = m / (HC * HC), yx = m % (HC * HC), yy = yx / HC, xx = yx % HC;
    const int y = yy * ST + z / ST, xq = xx * ST + z % ST;
    if (y >= H || xq >= H) { zero8(pf); return; }
    ld8(x + (int64_t(n * H + y) * H + xq) * C + c0, pf);
  }
  __device__ void store8p(int z, int m, int c0, const float v[8], const float xv[8]) const {
    const int n = m / (HC * HC), yx = m % (HC * HC), yy = yx / HC, xx = yx % HC;
    const int y = yy * ST + z / ST, xq = xx * ST + z % ST;
    if (y >= H || xq >= H) return;
    const int64_t i = (int64_t(n * H + y) * H + xq) * C + c0;
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = xv[j] > 0.f ? v[j] : 0.f;
    if (dx) st8(dx + i, o);
    if (dx16.hi) umma2::split8_planes(o, dx16.hi + i, dx16.hi + dx16.lo_off + i);
  }
};

// ---- wgrad (MN-major operands, umma_mn.cuh) -----------------------------------------------------
// conv2 / conv3: dW[(r,s,c)][ko] = sum_{n,p,q} X[n, p*ST+r, q*ST+s, c] * dZ[n,p,q,ko]
// One 64-wide m chunk is a contiguous run of the NHWC input: (s, c) are adjacent dims and R*C % 64 == 0.
template <int H, int C, int R, int ST, int KO>
struct WConvWgrad {
  static constexpr int P = (H - R) / ST + 1, KW = R * R * C;
  static_assert((R * C) % 64 == 0 && KO == 64, "64-element runs must not straddle a filter row");
  static constexpr int kBN = 64, kStages = 4;   // 193 KB: one CTA per SM
  static constexpr bool kAExact = false, kABulk = false;
  PlanePair x16;    // [rows][H][H][C]
  PlanePair dz16;   // [rows][P][P][KO]
  float* part;      // [splits][KW][KO]
  int rows, kb_per_split;
  __device__ int M(int) const { return KW; }
  __device__ int N(int) const { return KO; }
  __device__ void krange(int z, int& kb, int& ke) const {
    const int total = (rows * P * P + 63) / 64;
    kb = min(z * kb_per_split, total);
    ke = min(kb + kb_per_split, total);
  }
  __device__ umma_mn::PixCtx pix(int, int kpix) const {
    const int n = kpix / (P * P), pq = kpix % (P * P);
    return {n, pq / P, pq % P, kpix < rows * P * P};
  }
  __device__ umma2::Planes a_planes(int) const { return {x16.hi, x16.lo_off}; }
  __device__ bool a_run(int, const umma_mn::PixCtx& px, int mchunk, int64_t& off) const {
    const int m = mchunk * 64, r = m / (R * C), sc = m % (R * C);
    off = (int64_t(px.n * H + px.p * ST + r) * H + px.q * ST) * C + sc;
    return m < KW;
  }
  __device__ umma2::Planes b_planes(int) const { return {dz16.hi, dz16.lo_off}; }
  __device__ int64_t b_off(int, const umma_mn::PixCtx& px) const { return (int64_t(px.n * P + px.p) * P + px.q) * KO; }
  __device__ void store8(int z, int m, int n0, const float v[8]) const { st8(part + (int64_t(z) * KW + m) * KO + n0, v); }
};

// conv1: the A operand (row = output pixel, 64 contiguous taps (r,s) of frame c, exact u8 values) is
// exactly the tile conv1_fwd staged for its own MMA, so conv1_fwd ships those tiles to an im2col image
// (V2Conv1Fwd::kDumpA) and this kernel fetches each [64 pixels x 64 taps] sub-tile with ONE TMA bulk copy.
// M = 64 H rows (c, r, s): each 64-row m chunk is one frame c, so for odd H the last 128-row M tile has one live chunk.
template <int H>
struct WConv1Wgrad {
  static constexpr int kBN = 32, kStages = 4;
  static constexpr bool kAExact = true, kABulk = true;
  const uint8_t* im2col;   // [pixel tile of 128][c = H][128 x 128 B]
  PlanePair dz16;          // dZ1 [rows][20][20][32]
  float* part;             // [splits][64 H][32]
  int rows, kb_per_split;
  __device__ int M(int) const { return 64 * H; }
  __device__ int N(int) const { return kC1; }
  __device__ void krange(int z, int& kb, int& ke) const {
    const int total = (rows * kP1 * kP1 + 63) / 64;
    kb = min(z * kb_per_split, total);
    ke = min(kb + kb_per_split, total);
  }
  // kpix = the im2col row = the output pixel (row of dZ1); the last 128-row tile is padded
  __device__ umma_mn::PixCtx pix(int, int kpix) const { return {kpix, 0, 0, kpix < rows * kP1 * kP1}; }
  __device__ const uint8_t* a_sub(int, int c, int kb) const {   // kb = global 64-pixel block; nullptr: c >= H
    if (c >= H) return nullptr;
    return im2col + (int64_t(kb >> 1) * H + c) * (128 * 128) + (kb & 1) * (64 * 128);
  }
  __device__ umma2::Planes b_planes(int) const { return {dz16.hi, dz16.lo_off}; }
  __device__ int64_t b_off(int, const umma_mn::PixCtx& px) const { return int64_t(px.n) * kC1; }
  __device__ void store8(int z, int m, int n0, const float v[8]) const {
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = v[j] * (1.0f / 255.0f);
    st8(part + (int64_t(z) * 64 * H + m) * kC1 + n0, o);
  }
};

// fc1: dW4[m][n] = sum_b H3[b][m] * dZ4[b][n]; the reduction rows are the batch samples.
template <int W>
struct WFc1Wgrad {
  static constexpr int kBN = 64, kStages = 2;
  static constexpr bool kAExact = false, kABulk = false;
  PlanePair h3_16;   // [rows][3136]
  PlanePair dz4_16;  // [rows][W]
  float* dw4;        // [3136][W]
  int rows;
  __device__ int M(int) const { return kFlat; }
  __device__ int N(int) const { return W; }
  __device__ void krange(int, int& kb, int& ke) const { kb = 0; ke = (rows + 63) / 64; }
  __device__ umma_mn::PixCtx pix(int, int b) const { return {b, 0, 0, b < rows}; }
  __device__ umma2::Planes a_planes(int) const { return {h3_16.hi, h3_16.lo_off}; }
  __device__ bool a_run(int, const umma_mn::PixCtx& px, int mchunk, int64_t& off) const {
    off = int64_t(px.n) * kFlat + mchunk * 64;
    return mchunk * 64 < kFlat;
  }
  __device__ umma2::Planes b_planes(int) const { return {dz4_16.hi, dz4_16.lo_off}; }
  __device__ int64_t b_off(int, const umma_mn::PixCtx& px) const { return int64_t(px.n) * W; }
  __device__ void store8(int, int m, int n0, const float v[8]) const { st8(dw4 + int64_t(m) * W + n0, v); }
};

// Data-parallel variant: the rows are ALL learners' samples, read from the gather areas that every rank's
// k_xpush fills (comm_p2p.cuh); the parity of the current push epoch selects the area.
struct WFc1WgradGather {
  static constexpr int kBN = 64, kStages = 2;
  static constexpr bool kAExact = false, kABulk = false;
  const __half* h3g;   // [parity][hi | lo][rows][3136]
  const __half* dzg;   // [parity][hi | lo][rows][512]
  int64_t h3_parity, h3_lo, dz_parity, dz_lo;   // elements
  const uint32_t* epoch;   // [0] H3 pushes, [1] dZ4 pushes completed by this rank
  float* dw4;
  int rows;            // world x per-rank minibatch
  __device__ int M(int) const { return kFlat; }
  __device__ int N(int) const { return kHidden; }
  __device__ void krange(int, int& kb, int& ke) const { kb = 0; ke = (rows + 63) / 64; }
  __device__ umma_mn::PixCtx pix(int, int b) const { return {b, 0, 0, b < rows}; }
  __device__ umma2::Planes a_planes(int) const { return {h3g + int64_t(epoch[0] & 1) * h3_parity, h3_lo}; }
  __device__ bool a_run(int, const umma_mn::PixCtx& px, int mchunk, int64_t& off) const {
    off = int64_t(px.n) * kFlat + mchunk * 64;
    return mchunk * 64 < kFlat;
  }
  __device__ umma2::Planes b_planes(int) const { return {dzg + int64_t(epoch[1] & 1) * dz_parity, dz_lo}; }
  __device__ int64_t b_off(int, const umma_mn::PixCtx& px) const { return int64_t(px.n) * kHidden; }
  __device__ void store8(int, int m, int n0, const float v[8]) const { st8(dw4 + int64_t(m) * kHidden + n0, v); }
};

// ---- weight tile-image sources (k_pack_image) --------------------------------------------------
// at(tile, row, k): the element of w behind image element (tile, row, k), -1 for padding; kContig8: the 8 elements of
// a chunk (k0 .. k0 + 7) are consecutive in w
template <int K, int N>
struct PackFwdConv {   // B operand of a forward conv: rows = output channel n, K = filter taps
  static constexpr bool kRowMajorThreads = false;
  static constexpr bool kContig8 = false;
  const float* w;      // [K][N]
  __host__ __device__ int tiles() const { return 1; }
  __host__ __device__ int rows() const { return N; }
  __host__ __device__ int kblocks() const { return K / 64; }
  __device__ int at(int, int r, int k) const { return k * N + r; }
  __device__ void src8(int, int r, int k0, float v[8]) const {
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = w[at(0, r, k0 + j)];
  }
};
template <int W>
struct PackFc1Dgrad {  // the fc1 image: rows = flat index m, 64 hidden units per row (dgrad: K-major A; forward: MN-major A)
  static constexpr bool kRowMajorThreads = true;
  static constexpr bool kContig8 = true;
  const float* w;
  __host__ __device__ int tiles() const { return (kFlat + 127) / 128; }
  __host__ __device__ int rows() const { return 128; }
  __host__ __device__ int kblocks() const { return W / 64; }
  __device__ int at(int tile, int r, int k) const {
    const int m = tile * 128 + r;
    return m < kFlat ? m * W + k : -1;
  }
  __device__ void src8(int tile, int r, int k0, float v[8]) const {
    const int m = tile * 128 + r;
    if (m >= kFlat) { zero8(v); return; }
    ld8(w + m * W + k0, v);
  }
};
// Soft target update fused into the pack of the target's forward image (b200dqn_net_config::soft_target_tau): the
// source blends each master weight of a chunk on load, tw <- fl(fl(c tw) + fl(t w)), stores it back and hands the new
// value to the packer.  P (a packer over the target layer) supplies the tiling, so every target weight is read and
// written once, by the thread that packs it.
template <class P>
struct SoftBlendSrc {
  static constexpr bool kRowMajorThreads = P::kRowMajorThreads;
  P tgt;               // the packer over the target layer (tgt.w == tw)
  float* tw;           // the target layer, updated in place
  const float* w;      // the online layer, after this step's optimizer update
  float c, t;
  __host__ __device__ int tiles() const { return tgt.tiles(); }
  __host__ __device__ int rows() const { return tgt.rows(); }
  __host__ __device__ int kblocks() const { return tgt.kblocks(); }
  __device__ void src8(int tile, int r, int k0, float v[8]) const {
    if constexpr (P::kContig8) {
      const int i = tgt.at(tile, r, k0);
      if (i < 0) { zero8(v); return; }
      float a[8], b[8];
      ld8(tw + i, a);
      ld8(w + i, b);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = soft_blend1(a[j], b[j], c, t);
      st8(tw + i, v);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int i = tgt.at(tile, r, k0 + j);
        v[j] = soft_blend1(tw[i], w[i], c, t);
        tw[i] = v[j];
      }
    }
  }
};
template <int H, int C, int R, int ST, int KO>
struct PackConvDgrad { // B operand of a conv dgrad, one tile per output-parity class
  static constexpr int RT = R / ST, K = RT * RT * KO;
  static constexpr bool kRowMajorThreads = true;
  const float* w;      // [(r,s,c)][KO]
  __host__ __device__ int tiles() const { return ST * ST; }
  __host__ __device__ int rows() const { return C; }
  __host__ __device__ int kblocks() const { return K / 64; }
  __device__ void src8(int z, int c, int k0, float v[8]) const {
    const int rp = k0 / (RT * KO), sp = (k0 / KO) % RT, ko = k0 % KO;
    const int r = rp * ST + z / ST, s = sp * ST + z % ST;
    ld8(w + ((r * R + s) * C + c) * KO + ko, v);
  }
};

// ------------------------------------------------------------------------------------------
// Conv-layer optimizer, fused: split-K partial reduction (8 lanes per element, fixed tree ->
// deterministic) + Neon RMSProp (same operation order as k_optimizer, bit-exact given equal gradients)
// + refresh of the layer's fp16 tile images (forward B operand; dgrad B operand for conv2/conv3).
// Replaces three launches (optimizer, pack fwd, pack dgrad) on the tail of the step.
// ------------------------------------------------------------------------------------------
// XCHG (data-parallel learners, experimental — see umma_opt_conv_xll): between the reduction and the update the
// 8 lanes of an element exchange it with the other ranks in the LL protocol of comm_p2p.cuh — lane p pushes this
// rank's float4 to rank p and polls rank p's line — and the W contributions are added in rank order.
template <int KR, int N, bool DGRAD, int C, int R, int ST, bool XCHG = false>
__global__ void __launch_bounds__(256)
k_opt_conv(const float* __restrict__ part, int splits, float* __restrict__ w, float* __restrict__ sst,
           uint8_t* __restrict__ img_fwd, uint8_t* __restrict__ img_dgr, const OptArgs opt, const XllArgs x,
           const KTrace kt) {
  constexpr int64_t kSize = int64_t(KR) * N;
  kt_begin(kt);
  pdl_wait();
  pdl_launch_dependents();
  const int tid = threadIdx.x, lane8 = tid & 7;
  uint32_t epoch = 0;
  if constexpr (XCHG) epoch = *reinterpret_cast<volatile uint32_t*>(x.epoch + x.chan) + 1;
  const int64_t e4 = blockIdx.x * 32 + (tid >> 3);
  const int64_t i = e4 * 4;
  const bool live = i < kSize;
  float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
  if (live) {
    const float* p = part + i;
    float4 v[8];
    int cnt = 0;
#pragma unroll
    for (int u = 0; u < 8; ++u) {          // up to 64 splits: 8 independent loads per lane
      const int sp = lane8 + 8 * u;
      if (sp < splits) { v[u] = *reinterpret_cast<const float4*>(p + sp * kSize); cnt = u + 1; }
    }
    for (int u = 0; u < cnt; ++u) { g.x += v[u].x; g.y += v[u].y; g.z += v[u].z; g.w += v[u].w; }
  }
#pragma unroll
  for (int o = 1; o < 8; o <<= 1) {
    g.x += __shfl_xor_sync(0xffffffffu, g.x, o);
    g.y += __shfl_xor_sync(0xffffffffu, g.y, o);
    g.z += __shfl_xor_sync(0xffffffffu, g.z, o);
    g.w += __shfl_xor_sync(0xffffffffu, g.w, o);
  }
  if constexpr (XCHG) {
    float4 v = lane8 == x.rank ? g : make_float4(0.f, 0.f, 0.f, 0.f);
    if (live && lane8 < x.world && lane8 != x.rank) {
      const int64_t par = int64_t(epoch & 1) * x.world * x.lines_per_src, el = (x.ll4 + e4) * 2;
      uint4* dst = x.recv[lane8] + par + int64_t(x.rank) * x.lines_per_src + el;
      st_ll(dst, __float_as_uint(g.x), __float_as_uint(g.y), epoch);
      st_ll(dst + 1, __float_as_uint(g.z), __float_as_uint(g.w), epoch);
      const uint4* src = x.recv[x.rank] + par + int64_t(lane8) * x.lines_per_src + el;
      ll_wait(src, epoch, x.err, v.x, v.y);
      ll_wait(src + 1, epoch, x.err, v.z, v.w);
    }
    __syncwarp();
    const int base = (tid & 31) & ~7;
    g = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int p = 0; p < x.world; ++p) {   // rank order, the same on every rank
      const float a = __shfl_sync(0xffffffffu, v.x, base + p), b = __shfl_sync(0xffffffffu, v.y, base + p);
      const float c = __shfl_sync(0xffffffffu, v.z, base + p), d = __shfl_sync(0xffffffffu, v.w, base + p);
      if (p == 0) g = make_float4(a, b, c, d);
      else { g.x += a; g.y += b; g.z += c; g.w += d; }
    }
  }
  if (live && lane8 == 0) {
    float wp[4];
    opt_update_vec<4>(opt, opt_step_scalar(opt), reinterpret_cast<const float*>(&g), wp, w + i, sst + i);
    __half hi[4], lo[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) umma2::split1(wp[j], hi[j], lo[j]);
    const int k = int(i / N), n0 = int(i % N);
    {  // forward image: rows = output channel n, 8-element chunks along k
      uint8_t* base = img_fwd + int64_t(k / 64) * (N * 256) + (k % 8) * 2;
      const int c8 = (k % 64) / 8;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t off = umma::sw128_off(n0 + j, c8);
        *reinterpret_cast<__half*>(base + off) = hi[j];
        *reinterpret_cast<__half*>(base + N * 128 + off) = lo[j];
      }
    }
    if constexpr (DGRAD) {  // dgrad image: one tile per output-parity class, rows = input channel c, K = (r', s', ko)
      constexpr int RT = R / ST, NKB = RT * RT * N / 64;
      const int r = k / (R * C), s = (k / C) % R, c = k % C;
      const int z = (r % ST) * ST + (s % ST);
      const int kd = ((r / ST) * RT + (s / ST)) * N + n0;
      uint8_t* base = img_dgr + (int64_t(z) * NKB + kd / 64) * (C * 256) + umma::sw128_off(c, (kd % 64) / 8) + (kd % 8) * 2;
      *reinterpret_cast<uint2*>(base) = *reinterpret_cast<const uint2*>(hi);
      *reinterpret_cast<uint2*>(base + C * 128) = *reinterpret_cast<const uint2*>(lo);
    }
  }
  if constexpr (XCHG) {   // the last block to finish publishes the layer's new epoch (as in k_xll)
    __syncthreads();
    if (tid == 0) {
      __threadfence();
      if (atomicAdd(x.ticket + x.chan, 1u) == gridDim.x - 1) {
        x.ticket[x.chan] = 0;
        __threadfence();
        *reinterpret_cast<volatile uint32_t*>(x.epoch + x.chan) = epoch;
      }
    }
  }
  kt_end(kt);
}

// fc1 optimizer: RMSProp on 8 consecutive hidden units of one flat index per thread — which is exactly
// one 16-byte chunk of the row-oriented (dgrad) tile image, refreshed in the same pass; the
// column-oriented (forward) image is rebuilt by k_pack_image right after.  Both kernels are smem-free,
// light on registers and launched on a CAPPED grid (2 CTAs per SM, grid-stride loop) so that they
// co-reside with the tensor-core kernels of the critical chain instead of locking them out of the SMs.
template <int W, bool CLIP>
__device__ __forceinline__ void opt_fc1_body(const float* __restrict__ dw, float* __restrict__ w,
                                             float* __restrict__ sst, uint8_t* __restrict__ img_dgr,
                                             const OptArgs& opt, const float* __restrict__ clip, const KTrace& kt) {
  kt_begin(kt);
  pdl_wait();
  pdl_launch_dependents();
  constexpr int kNB = W / 8;
  const float l_step = opt_step_scalar(opt);
  float c = 1.f;
  if constexpr (CLIP) c = __ldcg(clip);
  for (int id = blockIdx.x * blockDim.x + threadIdx.x; id < kFlat * kNB; id += gridDim.x * blockDim.x) {
    const int m = id / kNB, n0 = (id % kNB) * 8;
    const int64_t i = int64_t(m) * W + n0;
    float g[8], wv[8];
    ld8(dw + i, g);
    opt_update_vec<8, CLIP>(opt, l_step, g, wv, w + i, sst + i, c);   // the configured Neon optimizer (optim.cuh)
    uint4 hi, lo;
    umma::split8(wv, hi, lo);
    uint8_t* base = img_dgr + (int64_t(m / 128) * (W / 64) + n0 / 64) * (128 * 256) +
                    umma::sw128_off(m % 128, (n0 % 64) / 8);
    *reinterpret_cast<uint4*>(base) = hi;
    *reinterpret_cast<uint4*>(base + 128 * 128) = lo;
  }
  kt_end(kt);
}

template <int W>
__global__ void __launch_bounds__(256)
k_opt_fc1(const float* __restrict__ dw, float* __restrict__ w, float* __restrict__ sst, uint8_t* __restrict__ img_dgr,
          const OptArgs opt, const KTrace kt) {
  opt_fc1_body<W, false>(dw, w, sst, img_dgr, opt, nullptr, kt);
}

// the same under global gradient-norm clipping, with the coefficient c32 read from *clip
template <int W>
__global__ void __launch_bounds__(256)
k_opt_fc1_clip(const float* __restrict__ dw, float* __restrict__ w, float* __restrict__ sst,
               uint8_t* __restrict__ img_dgr, const OptArgs opt, const float* __restrict__ clip, const KTrace kt) {
  opt_fc1_body<W, true>(dw, w, sst, img_dgr, opt, clip, kt);
}

int umma_opt_fc1(b200dqn_net* n, int rows, cudaStream_t st, bool from_g, const float* clip) {
  UmmaState* u = ust(n);
  const LayerTable& lt = n->lt;
  const float* dw = from_g ? n->d_g + lt.off[3] : n->d_part + lt.part_off[3];
  // One kernel, one image: the update refreshes the row-oriented tile image in the same pass, and the forward reads
  // that image too (MN-major) — the column-oriented forward image and its re-pack kernel (round 1-2: 6.4 MB read +
  // 6.4 MB written per step, 5 us at the end of the fc1 branch) are gone.
  // capped grid (2 CTAs per SM, grid-stride): the kernel shares the SMs — and the L2 — with the dgrad chain
  const int ctas = 2 * n->sm_count;
  if (clip) {
    B2_CHECK_CUDA(launch_pdl(n->dueling ? k_opt_fc1_clip<kDuelHidden> : k_opt_fc1_clip<kHidden>, dim3(ctas), dim3(256),
                             0, st, dw, n->d_w + lt.off[3], n->d_s + lt.off[3], u->img_dgr[0], make_opt_args(n, rows),
                             clip, ktrace_slot("opt_fc1_clip")));
    B2_PROF("opt_fc1_clip", st);
    return B200DQN_OK;
  }
  B2_CHECK_CUDA(launch_pdl(n->dueling ? k_opt_fc1<kDuelHidden> : k_opt_fc1<kHidden>, dim3(ctas), dim3(256), 0, st, dw,
                           n->d_w + lt.off[3],
                           n->d_s + lt.off[3], u->img_dgr[0], make_opt_args(n, rows), ktrace_slot("opt_fc1")));
  B2_PROF("opt_fc1", st);
  return B200DQN_OK;
}

// RMSProp + image refresh of conv layer l (0..2), fused (single-GPU path of the tensor-core engine).
int umma_opt_conv(b200dqn_net* n, int l, int rows, cudaStream_t st, const char* label, bool from_g) {
  UmmaState* u = ust(n);
  const LayerTable& lt = n->lt;
  const OptArgs opt = make_opt_args(n, rows);
  const float* part = from_g ? n->d_g + lt.off[l] : n->d_part + lt.part_off[l];
  const int nsplits = from_g ? 1 : lt.splits[l];
  float* w = n->d_w + lt.off[l];
  float* s = n->d_s + lt.off[l];
  B2_REQUIRE(nsplits <= 64, B200DQN_EINVAL, "k_opt_conv handles at most 64 split-K partials");
  const int64_t size = lt.off[l + 1] - lt.off[l];
  const dim3 grid(unsigned((size / 4 + 31) / 32)), block(256);
  cudaError_t e;
  const XllArgs none{};
  if (l == 0)
    e = with_hist(n->cfg.history_length, [&](auto h) {
      constexpr int H = decltype(h)::value;
      return launch_pdl(k_opt_conv<64 * H, kC1, false, 4, 8, 4>, grid, block, 0, st, part, nsplits, w, s,
                        u->img_fwd[0][0], (uint8_t*)nullptr, opt, none, ktrace_slot(label));
    });
  else if (l == 1)
    e = launch_pdl(k_opt_conv<kK2, kC2, true, kC1, 4, 2>, grid, block, 0, st, part, nsplits, w, s, u->img_fwd[0][1],
                   u->img_dgr[2], opt, none, ktrace_slot(label));
  else
    e = launch_pdl(k_opt_conv<kK3, kC3, true, kC2, 3, 1>, grid, block, 0, st, part, nsplits, w, s, u->img_fwd[0][2],
                   u->img_dgr[1], opt, none, ktrace_slot(label));
  B2_CHECK_CUDA(e);
  B2_PROF(label, st);
  return B200DQN_OK;
}

// EXPERIMENTAL (B200DQN_FUSED_XLL=1; written after round 1's GPU budget was spent, not yet run on hardware):
// split-K reduction + LL all-reduce across the learners + RMSProp + image refresh of conv layer l in ONE launch
// instead of three (reduce, k_xll, k_opt_conv) on the tail of the data-parallel step.
int umma_opt_conv_xll(b200dqn_net* n, int l, int rows, cudaStream_t st, const char* label) {
  UmmaState* u = ust(n);
  const LayerTable& lt = n->lt;
  const OptArgs opt = make_opt_args(n, rows);
  B2_REQUIRE(l >= 0 && l < 3 && lt.splits[l] <= 64 && n->world <= 8, B200DQN_EINVAL, "opt_conv_xll: bad layer / world");
  XllArgs x{};
  int rc = comm_xll_args(n, l, &x);
  if (rc) return rc;
  const float* part = n->d_part + lt.part_off[l];
  float* w = n->d_w + lt.off[l];
  float* s = n->d_s + lt.off[l];
  const int64_t size = lt.off[l + 1] - lt.off[l];
  const dim3 grid(unsigned((size / 4 + 31) / 32)), block(256);
  cudaError_t e;
  // data-parallel learners run 4-frame windows only (b200dqn_net_comm_init)
  B2_REQUIRE(lt.rows[0] == 64 * kHist, B200DQN_ENOTIMPL, "opt_conv_xll: history_length %d", n->cfg.history_length);
  if (l == 0)
    e = launch_pdl(k_opt_conv<64 * kHist, kC1, false, 4, 8, 4, true>, grid, block, 0, st, part, lt.splits[l], w, s,
                   u->img_fwd[0][0], (uint8_t*)nullptr, opt, x, ktrace_slot(label));
  else if (l == 1)
    e = launch_pdl(k_opt_conv<kK2, kC2, true, kC1, 4, 2, true>, grid, block, 0, st, part, lt.splits[l], w, s,
                   u->img_fwd[0][1], u->img_dgr[2], opt, x, ktrace_slot(label));
  else
    e = launch_pdl(k_opt_conv<kK3, kC3, true, kC2, 3, 1, true>, grid, block, 0, st, part, lt.splits[l], w, s,
                   u->img_fwd[0][2], u->img_dgr[1], opt, x, ktrace_slot(label));
  B2_CHECK_CUDA(e);
  B2_PROF(label, st);
  return B200DQN_OK;
}

static int64_t fwd_image_bytes(int layer, int hist, int hidden) {
  switch (layer) {
    case 0: return int64_t(hist) * kC1 * 256;
    case 1: return int64_t(kK2 / 64) * kC2 * 256;
    case 2: return int64_t(kK3 / 64) * kC3 * 256;
    default: return int64_t((kFlat + 127) / 128) * (hidden / 64) * 128 * 256;   // fc1: the row-oriented image
  }
}

// (re)build the tile images of layers [l0, l1] of network `which` from its fp32 master weights
int umma_pack_layers(b200dqn_net* n, int which, int l0, int l1, cudaStream_t st) {
  if (n->cfg.math_mode != B200DQN_MATH_TCGEN05) return B200DQN_OK;
  UmmaState* u = ust(n);
  const LayerTable& lt = n->lt;
  const float* w = which ? n->d_tw : n->d_w;
  int rc = 0;
  for (int l = l0; l <= l1 && !rc; ++l) {
    switch (l) {
      case 0:
        rc = with_hist(n->cfg.history_length, [&](auto h) {
          constexpr int H = decltype(h)::value;
          return umma2::launch_pack("pack_c1", PackFwdConv<64 * H, kC1>{w + lt.off[0]}, u->img_fwd[which][0], st);
        });
        break;
      case 1:
        rc = umma2::launch_pack("pack_c2f", PackFwdConv<kK2, kC2>{w + lt.off[1]}, u->img_fwd[which][1], st);
        if (!rc && !which)
          rc = umma2::launch_pack("pack_c2d", PackConvDgrad<kP1, kC1, 4, 2, kC2>{w + lt.off[1]}, u->img_dgr[2], st);
        break;
      case 2:
        rc = umma2::launch_pack("pack_c3f", PackFwdConv<kK3, kC3>{w + lt.off[2]}, u->img_fwd[which][2], st);
        if (!rc && !which)
          rc = umma2::launch_pack("pack_c3d", PackConvDgrad<kP2, kC2, 3, 1, kC3>{w + lt.off[2]}, u->img_dgr[1], st);
        break;
      case 3:
        rc = n->dueling ? umma2::launch_pack("pack_fc1", PackFc1Dgrad<kDuelHidden>{w + lt.off[3]}, u->img_fwd[which][3], st)
                        : umma2::launch_pack("pack_fc1", PackFc1Dgrad<kHidden>{w + lt.off[3]}, u->img_fwd[which][3], st);
        break;
      default: break;  // fc2 runs on CUDA cores (N = A <= 18)
    }
  }
  return rc;
}

// soft target update of layer l (0..3) fused with the rebuild of the target's forward image: one pass over the layer
// reads the online and target weights, writes the target weights and the image.  The target has no dgrad images.
int umma_soft_pack(b200dqn_net* n, int l, float c, float t, cudaStream_t st) {
  UmmaState* u = ust(n);
  const LayerTable& lt = n->lt;
  float* tw = n->d_tw + lt.off[l];
  const float* w = n->d_w + lt.off[l];
  uint8_t* img = u->img_fwd[1][l];
  switch (l) {
    case 0:
      return with_hist(n->cfg.history_length, [&](auto h) {
        constexpr int H = decltype(h)::value;
        using P = PackFwdConv<64 * H, kC1>;
        return umma2::launch_pack("soft_c1", SoftBlendSrc<P>{P{tw}, tw, w, c, t}, img, st);
      });
    case 1: {
      using P = PackFwdConv<kK2, kC2>;
      return umma2::launch_pack("soft_c2", SoftBlendSrc<P>{P{tw}, tw, w, c, t}, img, st);
    }
    case 2: {
      using P = PackFwdConv<kK3, kC3>;
      return umma2::launch_pack("soft_c3", SoftBlendSrc<P>{P{tw}, tw, w, c, t}, img, st);
    }
    default:
      if (n->dueling) {
        using P = PackFc1Dgrad<kDuelHidden>;
        return umma2::launch_pack("soft_fc1", SoftBlendSrc<P>{P{tw}, tw, w, c, t}, img, st);
      } else {
        using P = PackFc1Dgrad<kHidden>;
        return umma2::launch_pack("soft_fc1", SoftBlendSrc<P>{P{tw}, tw, w, c, t}, img, st);
      }
  }
}

// fc1 forward split-K over blockIdx.z (the head kernel sums the partials): 49 k-blocks of 64 -> 7 per CTA,
// 4 M-tiles x 7 x 2 nets = 56 CTAs at batch 32; large minibatches bring their own tiles, so fewer splits keep the
// partial-sum traffic down.  (13 splits = 104 CTAs was measured: fc1_fwd 6.3 -> 12 us inside the step — see below.)
// B200DQN_FC1_SPLITS=n overrides: on an H100 80GB HBM3 at 700 W, 4 splits were 2 % faster at batch 256, the same at 32.
static inline int fc1_splits_for(int rows) {
  static const int forced = getenv("B200DQN_FC1_SPLITS") ? atoi(getenv("B200DQN_FC1_SPLITS")) : 0;
  if (forced >= 1 && forced <= kFc1Splits) return forced;
  return rows <= 256 ? 7 : 4;
}
constexpr int kUWgradKb = 4;      // minimum k-blocks (of 64 pixels) per wgrad split

// k-blocks (of 64 pixels) per wgrad split: at least kUWgradKb, and few enough splits (<= 48) for the
// one-pass reduction of k_opt_conv
int umma_wgrad_kb(int layer, int rows) {
  const int kred = layer == 0 ? rows * kP1 * kP1 : layer == 1 ? rows * kP2 * kP2 : rows * kP3 * kP3;
  const int kbs = (kred + 63) / 64;
  int per = (kbs + 47) / 48;
  // conv1: at least 8 k-blocks per split (25 splits at batch 32).  On an H100 80GB HBM3 (400 W) the batch-32 step took
  // 92.5 / 92.1 / 89.3 / 90.9 / 89.8 us with 5 / 6 / 8 / 10 / 13 k-blocks per split (40 / 34 / 25 / 20 / 16 splits,
  // each partial read back by opt_conv1).
  if (layer == 0 && per < 8) per = 8;
  return per > kUWgradKb ? per : kUWgradKb;
}
int umma_wgrad_splits(int layer, int rows) {
  const int kred = layer == 0 ? rows * kP1 * kP1 : layer == 1 ? rows * kP2 * kP2 : rows * kP3 * kP3;
  const int kbs = (kred + 63) / 64, per = umma_wgrad_kb(layer, rows);
  return (kbs + per - 1) / per;
}

int umma_net_init(b200dqn_net* n) {
  if (n->cfg.math_mode != B200DQN_MATH_TCGEN05) return B200DQN_OK;
  auto* u = new UmmaState();
  n->umma_state = u;
  const int nb = n->nb;
  u->h_elems[0] = int64_t(nb) * kP1 * kP1 * kC1;
  u->h_elems[1] = int64_t(nb) * kP2 * kP2 * kC2;
  u->h_elems[2] = int64_t(nb) * kFlat;
  u->dz_elems[0] = int64_t(n->iqn_n ? n->iqn_rows : nb) * n->hidden;   // IQN: dZ4 of every expanded row
  u->dz_elems[1] = int64_t(nb) * kFlat;
  u->dz_elems[2] = int64_t(nb) * kP2 * kP2 * kC2;
  u->dz_elems[3] = int64_t(nb) * kP1 * kP1 * kC1;
  for (int i = 0; i < 3; ++i) {
    for (int z = 0; z < 2; ++z) {
      B2_CHECK_CUDA(cudaMalloc(&u->h16[i][z], 2 * u->h_elems[i] * sizeof(__half)));
      B2_CHECK_CUDA(cudaMemset(u->h16[i][z], 0, 2 * u->h_elems[i] * sizeof(__half)));
    }
  }
  for (int i = 0; i < 4; ++i) {
    B2_CHECK_CUDA(cudaMalloc(&u->dz16[i], 2 * u->dz_elems[i] * sizeof(__half)));
    B2_CHECK_CUDA(cudaMemset(u->dz16[i], 0, 2 * u->dz_elems[i] * sizeof(__half)));
  }
  for (int l = 0; l < 4; ++l) {
    u->img_fwd_bytes[l] = fwd_image_bytes(l, n->cfg.history_length, n->hidden);
    for (int z = 0; z < 2; ++z) {
      if (z == 1 && n->d_tw == n->d_w) { u->img_fwd[1][l] = u->img_fwd[0][l]; continue; }
      B2_CHECK_CUDA(cudaMalloc(&u->img_fwd[z][l], u->img_fwd_bytes[l]));
      B2_CHECK_CUDA(cudaMemset(u->img_fwd[z][l], 0, u->img_fwd_bytes[l]));
    }
  }
  B2_CHECK_CUDA(cudaMalloc(&u->im2col1,
                           int64_t((nb * kP1 * kP1 + 127) / 128) * n->cfg.history_length * 128 * 128));
  u->img_dgr[0] = u->img_fwd[0][3];   // fc1: ONE row-oriented image serves the dgrad (K-major) and the forward (MN-major)
  const int64_t dgr_bytes[3] = {0, int64_t(kK3 / 64) * kC2 * 256, int64_t(4) * (256 / 64) * kC1 * 256};
  for (int i = 1; i < 3; ++i) {
    B2_CHECK_CUDA(cudaMalloc(&u->img_dgr[i], dgr_bytes[i]));
    B2_CHECK_CUDA(cudaMemset(u->img_dgr[i], 0, dgr_bytes[i]));
  }
  return B200DQN_OK;
}

// fp16 planes of network slot 2 (Double DQN), allocated the first time it is switched on
int umma_double_q_alloc(b200dqn_net* n) {
  UmmaState* u = ust(n);
  if (!u) return B200DQN_OK;
  for (int i = 0; i < 3; ++i) {
    if (u->h16[i][2]) continue;
    B2_CHECK_CUDA(cudaMalloc(&u->h16[i][2], 2 * u->h_elems[i] * sizeof(__half)));
    B2_CHECK_CUDA(cudaMemset(u->h16[i][2], 0, 2 * u->h_elems[i] * sizeof(__half)));
  }
  return B200DQN_OK;
}

void umma_net_destroy(b200dqn_net* n) {
  UmmaState* u = ust(n);
  if (!u) return;
  for (int i = 0; i < 3; ++i) {
    for (int z = 0; z < 3; ++z) cudaFree(u->h16[i][z]);
    if (i > 0) cudaFree(u->img_dgr[i]);   // [0] aliases img_fwd[0][3]
  }
  for (int i = 0; i < 4; ++i) cudaFree(u->dz16[i]);
  cudaFree(u->im2col1);
  for (int l = 0; l < 4; ++l) {
    if (u->img_fwd[1][l] != u->img_fwd[0][l]) cudaFree(u->img_fwd[1][l]);
    cudaFree(u->img_fwd[0][l]);
  }
  delete u;
  n->umma_state = nullptr;
}

int umma_weights_changed(b200dqn_net* n, cudaStream_t st) {
  if (n->cfg.math_mode != B200DQN_MATH_TCGEN05) return B200DQN_OK;
  int rc = umma_pack_layers(n, 0, 0, 3, st);
  if (!rc && n->d_tw != n->d_w) rc = umma_pack_layers(n, 1, 0, 3, st);
  return rc;
}

int umma_target_synced(b200dqn_net* n, cudaStream_t st) {
  if (n->cfg.math_mode != B200DQN_MATH_TCGEN05 || n->d_tw == n->d_w) return B200DQN_OK;
  UmmaState* u = ust(n);
  for (int l = 0; l < 4; ++l)
    B2_CHECK_CUDA(cudaMemcpyAsync(u->img_fwd[1][l], u->img_fwd[0][l], u->img_fwd_bytes[l], cudaMemcpyDeviceToDevice, st));
  return B200DQN_OK;
}

void umma_dz4_planes(b200dqn_net* n, __half** hi, int64_t* lo_off) {
  UmmaState* u = ust(n);
  *hi = u ? u->dz16[0] : nullptr;
  *lo_off = u ? u->dz_elems[0] : 0;
}

void umma_dz3_planes(b200dqn_net* n, __half** hi, int64_t* lo_off) {
  UmmaState* u = ust(n);
  *hi = u ? u->dz16[1] : nullptr;
  *lo_off = u ? u->dz_elems[1] : 0;
}

template <int W>
static int fc1_fwd_umma(b200dqn_net* n, const PlanePair h3[3], int nets, int rows, cudaStream_t st) {
  UmmaState* u = ust(n);
  V2Fc1Fwd<W> p;
  for (int z = 0; z < 2; ++z) p.wimg[z] = u->img_fwd[z][3];
  for (int z = 0; z < 3; ++z) p.in16[z] = h3[z];
  p.part = n->d_fc1part; p.rows = rows; p.splits = fc1_splits_for(rows);
  return umma2::launch_umma2("fc1_fwd", p, W, rows, nets * p.splits, st, false);
}

int umma_forward(b200dqn_net* n, const uint8_t* const src[2], const int32_t* const idx[2], const int shift[2],
                 const int32_t* const crop[2], int nets, int rows, cudaStream_t st, bool release_early, bool trunk_only) {
  // Early release is applied to conv1_fwd and conv3_fwd only: on an H100 80GB HBM3 (400 W) taking it away from either
  // one slowed the batch-32 step by 0.6-1.4 us, while conv2_fwd and fc1_fwd gained nothing from it.  conv23_fwd keeps
  // its own release point.
  UmmaState* u = ust(n);
  auto planes = [&](int i, int z) { return PlanePair{u->h16[i][z], u->h_elems[i]}; };
  auto conv1 = [&](auto& p) {
    for (int z = 0; z < 2; ++z) {
      p.src[z] = src[z]; p.idx[z] = idx[z]; p.shift[z] = shift[z];
      p.wimg[z] = u->img_fwd[z][0]; p.out[z] = n->d_h1[z];
    }
    for (int z = 0; z < 3; ++z) p.out16[z] = planes(0, z);
    p.out[2] = nullptr;                                                  // slot 2 keeps no fp32 activations
    p.rows = rows;
    p.im2col = (nets >= 2 && rows == n->nb) ? u->im2col1 : nullptr;   // only a train step feeds conv1_wgrad
    return umma2::launch_umma2("conv1_fwd", p, rows * kP1 * kP1, kC1, nets, st, release_early);
  };
  int rc = with_hist(n->cfg.history_length, [&](auto h) {
    constexpr int H = decltype(h)::value;
    if (crop[0]) {
      V2Conv1FwdCrop<H> p;
      p.crop[0] = crop[0]; p.crop[1] = crop[1];
      return conv1(p);
    }
    V2Conv1Fwd<H> p;
    return conv1(p);
  });
  if (rc) return rc;
  if (rows <= kConv23MaxRows) {
    Conv23Fwd p{};
    for (int z = 0; z < 2; ++z) { p.c2.wimg[z] = u->img_fwd[z][1]; p.c3.wimg[z] = u->img_fwd[z][2]; }
    for (int z = 0; z < 3; ++z) {
      p.c2.in16[z] = planes(0, z); p.c3.out16[z] = planes(2, z);
      p.c3.out[z] = z ? nullptr : n->d_h3[z];   // nothing reads the fp32 activations of slots 1 and 2
    }
    if (trunk_only) p.c3.out[1] = n->d_h3[1];   // IQN: the target's psi for its modulation
    p.c2.out[0] = n->d_h2[0]; p.c2.out16[0] = planes(1, 0);   // the kernel stores H2 of the online net only
    p.c2.rows = p.c3.rows = rows;
    if ((rc = launch_conv23(p, rows, nets, st))) return rc;
  } else {
    {
      using P = V2ConvFwd<kP1, kC1, 4, 2, kC2>;
      P p;
      for (int z = 0; z < 2; ++z) p.wimg[z] = u->img_fwd[z][1];
      for (int z = 0; z < 3; ++z) {
        p.in16[z] = planes(0, z); p.out16[z] = planes(1, z);
        p.out[z] = z ? nullptr : n->d_h2[z];     // nothing reads the fp32 activations of slots 1 and 2
      }
      p.rows = rows;
      if ((rc = umma2::launch_umma2("conv2_fwd", p, rows * kP2 * kP2, kC2, nets, st, false))) return rc;
    }
    {
      using P = V2ConvFwd<kP2, kC2, 3, 1, kC3>;
      P p;
      for (int z = 0; z < 2; ++z) p.wimg[z] = u->img_fwd[z][2];
      for (int z = 0; z < 3; ++z) {
        p.in16[z] = planes(1, z); p.out16[z] = planes(2, z);
        p.out[z] = z ? nullptr : n->d_h3[z];
      }
      if (trunk_only) p.out[1] = n->d_h3[1];
      p.rows = rows;
      if ((rc = umma2::launch_umma2("conv3_fwd", p, rows * kP3 * kP3, kC3, nets, st, release_early))) return rc;
    }
  }
  if (trunk_only) return B200DQN_OK;
  // data-parallel learners: this rank's H3 rows start travelling to every rank's fc1_wgrad now
  if (nets >= 2 && rows == n->nb && comm_gather_active(n, st) && (rc = umma_push_h3(n, st))) return rc;
  const PlanePair h3[3] = {planes(2, 0), planes(2, 1), planes(2, 2)};
  return n->dueling ? fc1_fwd_umma<kDuelHidden>(n, h3, nets, rows, st) : fc1_fwd_umma<kHidden>(n, h3, nets, rows, st);
}

// X planes of slot z: [hi ld x 3136 | lo ld x 3136] at d_x16 + z * 2 * ld * 3136 (k_iqn_mod writes them)
static PlanePair iqn_x_planes(b200dqn_net* n, int z) {
  const int64_t slot = int64_t(n->iqn_rows) * kFlat;
  return PlanePair{n->d_x16 + 2 * z * slot, slot};
}

int umma_fc1_fwd_iqn(b200dqn_net* n, int nets, int rows, int splits, cudaStream_t st) {
  UmmaState* u = ust(n);
  V2Fc1Fwd<kHidden> p;   // 512 wide: an IQN net is not a dueling one
  for (int z = 0; z < 2; ++z) p.wimg[z] = u->img_fwd[z][3];
  for (int z = 0; z < 3; ++z) p.in16[z] = iqn_x_planes(n, z == 1 ? 1 : 0);
  p.part = n->d_fc1part; p.rows = rows; p.splits = splits;
  return umma2::launch_umma2("fc1_fwd", p, kHidden, rows, nets * splits, st, false);
}

int umma_fc1_fwd_fqf_boundary(b200dqn_net* n, int rows, int splits, cudaStream_t st) {
  UmmaState* u = ust(n);
  V2Fc1Fwd<kHidden> p;   // the online network only (nets = 1)
  p.wimg[0] = p.wimg[1] = u->img_fwd[0][3];
  const PlanePair x{n->d_bx16, int64_t(n->nb) * (n->fqf_n - 1) * kFlat};
  for (int z = 0; z < 3; ++z) p.in16[z] = x;
  p.part = n->d_fc1part; p.rows = rows; p.splits = splits;
  return umma2::launch_umma2("fc1_fwd", p, kHidden, rows, splits, st, false);
}

// The Munchausen target pass: umma_forward's launches with one network slot (nets = 1) and remapped pointers.  Device
// slot 0 reads the target network's weight images and the prestates (slot 0's frames) and writes the third slot's
// fp16 planes and fc1 partials; no fp32 activation is kept.  The kernels specialise slot 0 in two places: conv1_fwd
// dumps no im2col tiles (nets < 2), and conv23_fwd stores its H2 planes (here slot 2's) and, with a null `out`, no
// fp32 H2.
int umma_forward_target_pre(b200dqn_net* n, const uint8_t* src, const int32_t* idx, int shift, const int32_t* crop,
                            int rows, cudaStream_t st) {
  UmmaState* u = ust(n);
  auto planes = [&](int i) { return PlanePair{u->h16[i][2], u->h_elems[i]}; };
  auto conv1 = [&](auto& p) {
    p.src[0] = p.src[1] = src; p.idx[0] = p.idx[1] = idx; p.shift[0] = p.shift[1] = shift;
    p.wimg[0] = p.wimg[1] = u->img_fwd[1][0];
    p.out16[0] = planes(0);
    p.rows = rows;
    p.im2col = nullptr;
    return umma2::launch_umma2("conv1_fwd", p, rows * kP1 * kP1, kC1, 1, st, false);
  };
  int rc = with_hist(n->cfg.history_length, [&](auto h) {
    constexpr int H = decltype(h)::value;
    if (crop) {
      V2Conv1FwdCrop<H> p{};
      p.crop[0] = p.crop[1] = crop;
      return conv1(p);
    }
    V2Conv1Fwd<H> p{};
    return conv1(p);
  });
  if (rc) return rc;
  if (rows <= kConv23MaxRows) {
    Conv23Fwd p{};
    p.c2.wimg[0] = p.c2.wimg[1] = u->img_fwd[1][1];
    p.c3.wimg[0] = p.c3.wimg[1] = u->img_fwd[1][2];
    p.c2.in16[0] = planes(0);
    p.c2.out16[0] = planes(1);
    p.c3.out16[0] = planes(2);
    p.c2.rows = p.c3.rows = rows;
    if ((rc = launch_conv23(p, rows, 1, st))) return rc;
  } else {
    {
      V2ConvFwd<kP1, kC1, 4, 2, kC2> p{};
      p.wimg[0] = p.wimg[1] = u->img_fwd[1][1];
      p.in16[0] = planes(0); p.out16[0] = planes(1);
      p.rows = rows;
      if ((rc = umma2::launch_umma2("conv2_fwd", p, rows * kP2 * kP2, kC2, 1, st, false))) return rc;
    }
    {
      V2ConvFwd<kP2, kC2, 3, 1, kC3> p{};
      p.wimg[0] = p.wimg[1] = u->img_fwd[1][2];
      p.in16[0] = planes(1); p.out16[0] = planes(2);
      p.rows = rows;
      if ((rc = umma2::launch_umma2("conv3_fwd", p, rows * kP3 * kP3, kC3, 1, st, false))) return rc;
    }
  }
  // fc1 (512 wide: a Munchausen net is not a dueling one) into slot 2's region of the three-slot partial buffer
  V2Fc1Fwd<kHidden> p{};
  p.wimg[0] = p.wimg[1] = u->img_fwd[1][3];
  p.in16[0] = planes(2);
  p.splits = fc1_splits_for(rows);
  p.part = n->d_fc1part + int64_t(2) * p.splits * rows * kHidden;
  p.rows = rows;
  return umma2::launch_umma2("fc1_fwd", p, kHidden, rows, p.splits, st, false);
}

template <int W>
static int fc1_wgrad_umma(b200dqn_net* n, int rows, cudaStream_t st, bool release_early) {
  UmmaState* u = ust(n);
  WFc1Wgrad<W> p{PlanePair{u->h16[2][0], u->h_elems[2]}, PlanePair{u->dz16[0], u->dz_elems[0]},
                 n->d_part + n->lt.part_off[3], rows};
  return umma_mn::launch_umma_mn("fc1_wgrad", p, kFlat, W, 1, st, release_early);
}

template <int W>
static int fc1_dgrad_umma(b200dqn_net* n, int rows, cudaStream_t st, bool release_early) {
  UmmaState* u = ust(n);
  // the fp32 copies of dZ3/dZ2/dZ1 have no reader in this engine (wgrads and dgrads take the fp16 planes)
  V2Fc1Dgrad<W> p{u->img_dgr[0], PlanePair{u->dz16[0], u->dz_elems[0]}, n->d_h3[0], n->keep_grads ? n->d_dz3 : nullptr,
                  PlanePair{u->dz16[1], u->dz_elems[1]}, rows};
  return umma2::launch_umma2("fc1_dgrad", p, kFlat, rows, 1, st, release_early);
}

int umma_backward_op(b200dqn_net* n, int op, const uint8_t* src, const int32_t* idx, int shift, int rows,
                     cudaStream_t st, bool release_early) {
  const LayerTable& lt = n->lt;
  const float* w = n->d_w;
  switch (op) {
    case 0:
      if (n->iqn_n) {   // IQN: fc1 ran on X at rows N expanded rows, reduced in chunks of kIqnWgradRows rows, one
        // partial each (lt.splits[3]): one fp32 accumulation chain over 4096 rows exceeded the hi/lo scheme's bound
        UmmaState* u = ust(n);
        const int R = rows * n->iqn_n;
        const PlanePair x = iqn_x_planes(n, 0);
        const int64_t wsize = lt.off[4] - lt.off[3];
        for (int s = 0; s < lt.splits[3]; ++s) {
          const int r0 = s * kIqnWgradRows;
          WFc1Wgrad<kHidden> p{PlanePair{x.hi + int64_t(r0) * kFlat, x.lo_off},
                               PlanePair{u->dz16[0] + int64_t(r0) * kHidden, u->dz_elems[0]},
                               n->d_part + lt.part_off[3] + s * wsize, std::min(kIqnWgradRows, R - r0)};
          const int rc = umma_mn::launch_umma_mn("fc1_wgrad", p, kFlat, kHidden, 1, st, release_early);
          if (rc) return rc;
        }
        return B200DQN_OK;
      }
      return n->dueling ? fc1_wgrad_umma<kDuelHidden>(n, rows, st, release_early)
                        : fc1_wgrad_umma<kHidden>(n, rows, st, release_early);
    case 1:
      if (n->iqn_n) {   // IQN: dX in fp32 (masked by X > 0, harmless: b200dqn.h rule 11); its fp16 planes have no
        // reader and go to slot 1's X planes, which nothing reads after the forward
        UmmaState* u = ust(n);
        V2Fc1Dgrad<kHidden> p{u->img_dgr[0], PlanePair{u->dz16[0], u->dz_elems[0]}, n->d_x, n->d_dx,
                              iqn_x_planes(n, 1), rows * n->iqn_n};
        return umma2::launch_umma2("fc1_dgrad", p, kFlat, rows * n->iqn_n, 1, st, release_early);
      }
      return n->dueling ? fc1_dgrad_umma<kDuelHidden>(n, rows, st, release_early)
                        : fc1_dgrad_umma<kHidden>(n, rows, st, release_early);
    case 2: {
      UmmaState* u = ust(n);
      using P = WConvWgrad<kP2, kC2, 3, 1, kC3>;
      P p{PlanePair{u->h16[1][0], u->h_elems[1]}, PlanePair{u->dz16[1], u->dz_elems[1]},
          n->d_part + lt.part_off[2], rows, umma_wgrad_kb(2, rows)};
      return umma_mn::launch_umma_mn("conv3_wgrad", p, P::KW, kC3, lt.splits[2], st, release_early);
    }
    case 3: {
      UmmaState* u = ust(n);
      using P = V2ConvDgrad<kP2, kC2, 3, 1, kC3>;
      P p{PlanePair{u->dz16[1], u->dz_elems[1]}, u->img_dgr[1], n->d_h2[0], n->keep_grads ? n->d_dz2 : nullptr,
          PlanePair{u->dz16[2], u->dz_elems[2]}, rows};
      return umma2::launch_umma2("conv3_dgrad", p, rows * P::HC * P::HC, kC2, 1, st, release_early);
    }
    case 4: {
      UmmaState* u = ust(n);
      using P = WConvWgrad<kP1, kC1, 4, 2, kC2>;
      P p{PlanePair{u->h16[0][0], u->h_elems[0]}, PlanePair{u->dz16[2], u->dz_elems[2]},
          n->d_part + lt.part_off[1], rows, umma_wgrad_kb(1, rows)};
      return umma_mn::launch_umma_mn("conv2_wgrad", p, P::KW, kC2, lt.splits[1], st, release_early);
    }
    case 5: {
      UmmaState* u = ust(n);
      using P = V2ConvDgrad<kP1, kC1, 4, 2, kC2>;
      using P2 = V2ConvDgrad<kP1, kC1, 4, 2, kC2, 2>;
      // One GPU: a 2-stage operand ring, 81 KB per CTA instead of 161 KB, so the 100 CTAs take 50 SMs instead of 100
      // while conv3_wgrad / conv2_wgrad / conv1_wgrad look for SMs.  On an H100 80GB HBM3 at 700 W this is 1.5 %
      // faster than the deepest ring at batch 256 and the same at 32; shallow rings for the conv3/conv2 wgrads as
      // well cost 1-2 %.  With data-parallel learners the deepest ring was faster (on an earlier GPU generation;
      // multi-GPU schedules have not been re-measured on H100).
      if (n->world == 1) {
        P2 p{PlanePair{u->dz16[2], u->dz_elems[2]}, u->img_dgr[2], n->d_h1[0], n->keep_grads ? n->d_dz1 : nullptr,
             PlanePair{u->dz16[3], u->dz_elems[3]}, rows};
        return umma2::launch_umma2("conv2_dgrad", p, rows * P::HC * P::HC, kC1, 4, st, release_early);
      }
      P p{PlanePair{u->dz16[2], u->dz_elems[2]}, u->img_dgr[2], n->d_h1[0], n->keep_grads ? n->d_dz1 : nullptr,
          PlanePair{u->dz16[3], u->dz_elems[3]}, rows};
      return umma2::launch_umma2("conv2_dgrad", p, rows * P::HC * P::HC, kC1, 4, st, release_early);
    }
    default: {
      UmmaState* u = ust(n);
      (void)src; (void)idx; (void)shift;   // the frames were already gathered by conv1_fwd (im2col image)
      return with_hist(n->cfg.history_length, [&](auto h) {
        constexpr int H = decltype(h)::value;
        WConv1Wgrad<H> p{u->im2col1, PlanePair{u->dz16[3], u->dz_elems[3]}, n->d_part + lt.part_off[0], rows,
                           umma_wgrad_kb(0, rows)};
        return umma_mn::launch_umma_mn("conv1_wgrad", p, 64 * H, kC1, lt.splits[0], st, release_early);
      });
    }
  }
}

int umma_fc1_splits(int rows) { return fc1_splits_for(rows); }
// ---- gather schedule hooks (data-parallel learners, comm_p2p.cuh) ---------------------------------------
int umma_push_h3(b200dqn_net* n, cudaStream_t st) {
  UmmaState* u = ust(n);
  cudaStream_t sN = n->side[3];
  B2_CHECK_CUDA(cudaEventRecord(n->ev[13], st));          // conv23_fwd done: the online net's H3 planes are final
  B2_CHECK_CUDA(cudaStreamWaitEvent(sN, n->ev[13], 0));
  const int rc = comm_push_planes(n, 0, u->h16[2][0], u->h_elems[2], sN);
  if (rc) return rc;
  B2_CHECK_CUDA(cudaEventRecord(n->ev[14], sN));
  return B200DQN_OK;
}
int umma_push_dz4(b200dqn_net* n, cudaStream_t st) {
  UmmaState* u = ust(n);
  return comm_push_planes(n, 1, u->dz16[0], u->dz_elems[0], st);
}
int umma_gather_dz4_ll(b200dqn_net* n, cudaStream_t st) {
  UmmaState* u = ust(n);
  return comm_gather_dz4_ll(n, u->dz16[0], u->dz_elems[0], st, true);   // also waits for the peers' H3 rows
}
int umma_fc1_wgrad_gathered(b200dqn_net* n, cudaStream_t st) {
  WFc1WgradGather p{reinterpret_cast<const __half*>(n->d_xbuf + n->x_h3_off),
                    reinterpret_cast<const __half*>(n->d_xbuf + n->x_dz_off),
                    n->x_h3_parity / 2, n->x_h3_lo, n->x_dz_parity / 2, n->x_dz_lo,
                    n->d_xpush_epoch, n->d_part + n->lt.part_off[3], n->nb * n->world};
  return umma_mn::launch_umma_mn("fc1_wgrad", p, kFlat, kHidden, 1, st, false);
}

}  // namespace b200

extern "C" int b200dqn_debug_trace(unsigned long long* host_out, int n) {
  cudaDeviceSynchronize();
  return b200::umma2::read_trace(host_out, n);
}
