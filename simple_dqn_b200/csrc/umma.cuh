// umma.cuh — Hopper (sm_90a) warpgroup-MMA building blocks shared by the kernels of umma2.cuh (K-major
// operands: forward, dgrad) and umma_mn.cuh (MN-major operands: wgrad).
//
//   D[128 x BN] (fp32, registers) = A[128 x K] * B[BN x K]^T        A, B: fp16 in SWIZZLE_128B shared memory
//
// A CTA tile of 128 rows is computed by two consumer warpgroups, each issuing wgmma.mma_async with M = 64 on its
// half of the A tile; the fp32 accumulators live in the registers of the warpgroup that issued the MMAs.
//
// Every fp32 operand x is split ONCE, by its producer, into hi = fp16(x) and lo' = fp16((x - hi) * 2^11);
// a k-step issues  [acc0 | acc1] += A_hi x [B_hi ; B_lo']  (one MMA with N = 2*BN: the hi and lo tiles
// are adjacent in shared memory) and  acc2 += A_lo' x B_hi;  the epilogue returns acc0 + (acc1 + acc2) * 2^-11.
// That reproduces fp32 products to ~2^-22 (SURVEY §7 "Precision vs the 1e-3 bar": plain fp16 fails the
// parity bar, the split is indistinguishable from fp32) for 1.5-2x the tensor work of plain fp16.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"

namespace b200 {
namespace umma {

constexpr int kBM = 128;        // CTA tile M = two warpgroups x wgmma M = 64
constexpr int kWgM = 64;        // rows of the tile owned by one warpgroup
constexpr int kBK = 64;         // fp16 elements per k-block = one 128-byte swizzle row
constexpr int kThreads = 256;   // 2 warpgroups: all stage operands, issue the MMAs of their half, run the epilogue
constexpr float kLoScale = 2048.0f, kLoInv = 1.0f / 2048.0f;

// ---- wgmma shared-memory matrix descriptor, K-major SWIZZLE_128B:
//   [0,14) start>>4 | [16,30) LBO>>4 (unused for swizzled K-major: 1) | [32,46) SBO>>4 (8 rows * 128 B = 1024 -> 64) |
//   [49,52) base offset (0: tiles are 1024-byte aligned) | [62,64) layout = 1 (SWIZZLE_128B)
__device__ __forceinline__ uint64_t make_desc_sw128(uint32_t smem_addr) {
  return uint64_t((smem_addr >> 4) & 0x3FFF) | (uint64_t(1) << 16) | (uint64_t(64) << 32) | (uint64_t(1) << 62);
}

// MN-major SWIZZLE_128B descriptor: LBO = byte stride between 64-element MN chunks, SBO = byte stride
// between groups of 8 k rows (1024 when rows are packed).  A [64 k-rows x 128 B] sub-tile written in the K-major
// SW128 pattern with "row = k" IS this layout — which is why the row-oriented fc1 weight image (rows = flat index,
// 64 hidden units per 128-byte row) serves the dgrad as a K-major operand and the forward as an MN-major one.
__device__ __forceinline__ uint64_t make_desc_mn(uint32_t smem_addr, uint32_t lbo_bytes) {
  return uint64_t((smem_addr >> 4) & 0x3FFF) | (uint64_t((lbo_bytes >> 4) & 0x3FFF) << 16) | (uint64_t(64) << 32) |
         (uint64_t(1) << 62);
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// D[64 x N] += A[64 x 16] * B[N x 16]^T, fp16 operands from shared memory, fp32 accumulators in registers.
// TA / TB = 1: the operand is MN-major (transposed) in shared memory.  Register i of the fragment holds
// row (warp % 4) * 16 + lane / 4 + 8 * ((i >> 1) & 1), column (i >> 2) * 8 + (lane % 4) * 2 + (i & 1).
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n32(float* d, uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(1), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n64(float* d, uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(1), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n128(float* d, uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, %67, %68;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(1), "n"(TA), "n"(TB));
}

template <int N, int TA = 0, int TB = 0>
__device__ __forceinline__ void wgmma_f16(float* d, uint64_t da, uint64_t db) {
  static_assert(N == 32 || N == 64 || N == 128, "instantiated wgmma shapes");
  if constexpr (N == 32) wgmma_n32<TA, TB>(d, da, db);
  else if constexpr (N == 64) wgmma_n64<TA, TB>(d, da, db);
  else wgmma_n128<TA, TB>(d, da, db);
}
__device__ __forceinline__ int frag_row(int i, int lane, int warp) { return (warp & 3) * 16 + (lane >> 2) + 8 * ((i >> 1) & 1); }
__device__ __forceinline__ int frag_col(int i, int lane) { return (i >> 2) * 8 + (lane & 3) * 2 + (i & 1); }

// The combined tile (acc0 + (acc1 + acc2) * 2^-11) of this warpgroup into shared memory at `tile` (row pitch `pitch`
// bytes, rows of this warpgroup start at wg * 64).  acc holds the N = 2*BN fragment [acc0 | acc1] (registers
// [0, BN/2) and [BN/2, BN)), acc2 the N = BN fragment of A_lo x B_hi (nullptr: A is exact).  A_lo x B_hi has an
// accumulator of its own: a wgmma accumulating into part of another in-flight wgmma's fragment makes ptxas
// serialize the whole wgmma pipeline.
template <int BN>
__device__ __forceinline__ void stage_acc(const float* acc, const float* acc2, uint8_t* tile, int pitch, int wg, int warp,
                                          int lane) {
#pragma unroll
  for (int i = 0; i < BN / 2; i += 2) {
    const int r = wg * kWgM + frag_row(i, lane, warp), c = frag_col(i, lane);
    const float l0 = acc2 ? acc[BN / 2 + i] + acc2[i] : acc[BN / 2 + i];
    const float l1 = acc2 ? acc[BN / 2 + i + 1] + acc2[i + 1] : acc[BN / 2 + i + 1];
    const float2 v = make_float2(fmaf(l0, kLoInv, acc[i]), fmaf(l1, kLoInv, acc[i + 1]));
    *reinterpret_cast<float2*>(tile + r * pitch + c * 4) = v;
  }
}

// fp32 x[8] -> 16-byte chunks of fp16 hi and scaled fp16 lo
__device__ __forceinline__ void split8(const float x[8], uint4& hi, uint4& lo) {
  __half2 h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const __half2 hh = __floats2half2_rn(x[2 * i], x[2 * i + 1]);
    const float2 back = __half22float2(hh);
    h[i] = hh;
    l[i] = __floats2half2_rn((x[2 * i] - back.x) * kLoScale, (x[2 * i + 1] - back.y) * kLoScale);
  }
  hi = *reinterpret_cast<uint4*>(h);
  lo = *reinterpret_cast<uint4*>(l);
}

// byte offset of 16-byte chunk c (0..7) of row r inside a [rows x 64] fp16 SW128 tile
__device__ __forceinline__ uint32_t sw128_off(int r, int c) {
  return uint32_t((r >> 3) * 1024 + (r & 7) * 128 + ((c ^ (r & 7)) << 4));
}

}  // namespace umma
}  // namespace b200
