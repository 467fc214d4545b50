// net_simt.cuh — CUDA-core fp32 implicit-GEMM engine (math_mode FP32_SIMT).
//
// One tiled FFMA GEMM kernel, C[M,N] = A[M,K] * B[K,N], whose operands are produced element by
// element by a "problem" functor, so every GEMM-shaped op of the Nature-DQN step (im2col forward,
// dgrad, wgrad, dense layers) is the same kernel with a different functor.  It is the exact-fp32
// mode of the library and the on-device cross-check of the tensor-core path.
//
// Geometry is the reference's (src/deepqnetwork.py:77-92): 84x84xH u8 (H = history_length frames as input
// channels) -> conv 8x8x32 s4 -> conv 4x4x64 s2 -> conv 3x3x64 s1 -> fc 512 -> fc A; no bias, no padding.
// A dueling net (b200dqn_net_config::dueling) has fc 1024 -> fc A + 1 in place of the last two.
//
// Internal layouts (HBM):
//   activations  NHWC fp32:  H1[n][20][20][32]  H2[n][9][9][64]  H3[n][7][7][64]  H4[n][512]
//   weights      [K][N] fp32 with N (output feature) contiguous and K ordered to match the
//                producer's NHWC patch: W1[(c,r,s)][32] (64*H rows, == Neon CRSK), W2[(r,s,c)][64],
//                W3[(r,s,c)][64], W4[(p,q,c)][512], W5[512][A]
#pragma once
#include "common.cuh"

namespace b200 {

constexpr int kFrameH = 84, kFrameW = 84;
constexpr int kHist = 4;                        // the reference's default history length (main.py:34)
constexpr int kMaxHist = 16;                    // history lengths 1..kMaxHist are implemented
constexpr int kFrameBytes = kFrameH * kFrameW;  // 7056 = 441 * 16
constexpr int kP1 = 20, kC1 = 32;               // conv1 output
constexpr int kP2 = 9, kC2 = 64;                // conv2 output
constexpr int kP3 = 7, kC3 = 64;                // conv3 output
constexpr int kFlat = kP3 * kP3 * kC3;          // 3136
constexpr int kHidden = 512;
constexpr int kDuelHidden = 2 * kHidden;      // dueling fc1: advantage units [0, 512), value units [512, 1024)
constexpr int kK2 = 4 * 4 * kC1;                // 512
constexpr int kK3 = 3 * 3 * kC2;                // 576

// ------------------------------------------------------------------------------------------
// Generic kernel.  grid = (ceil(M/BM), ceil(N/BN), Z).  Problem P provides:
//   int M(z), N(z); void krange(z, kb, ke); float a(z,m,k); float b(z,k,n); void store(z,m,n,v)
//   static constexpr bool kAKContig / kBKContig : which index is contiguous in memory (coalescing)
// ------------------------------------------------------------------------------------------
template <class P, int BM, int BN, int BK, int TM, int TN>
__global__ void __launch_bounds__((BM / TM) * (BN / TN)) k_simt_gemm(const P p) {
  constexpr int NT = (BM / TM) * (BN / TN);
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  const int z = blockIdx.z;
  const int M = p.M(z), N = p.N(z);
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  if (m0 >= M || n0 >= N) return;
  int kb, ke;
  p.krange(z, kb, ke);
  const int tid = threadIdx.x;
  const int tx = tid % (BN / TN), ty = tid / (BN / TN);
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  for (int k0 = kb; k0 < ke; k0 += BK) {
#pragma unroll 2
    for (int i = tid; i < BM * BK; i += NT) {
      int mm, kk;
      if (P::kAKContig) { kk = i % BK; mm = i / BK; } else { mm = i % BM; kk = i / BM; }
      const int m = m0 + mm, k = k0 + kk;
      As[kk][mm] = (m < M && k < ke) ? p.a(z, m, k) : 0.f;
    }
#pragma unroll 2
    for (int i = tid; i < BN * BK; i += NT) {
      int nn, kk;
      if (P::kBKContig) { kk = i % BK; nn = i / BK; } else { nn = i % BN; kk = i / BN; }
      const int n = n0 + nn, k = k0 + kk;
      Bs[kk][nn] = (n < N && k < ke) ? p.b(z, k, n) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float av[TM], bv[TN];
#pragma unroll
      for (int i = 0; i < TM; ++i) av[i] = As[kk][ty * TM + i];
#pragma unroll
      for (int j = 0; j < TN; ++j) bv[j] = Bs[kk][tx * TN + j];
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int m = m0 + ty * TM + i, n = n0 + tx * TN + j;
      if (m < M && n < N) p.store(z, m, n, acc[i][j]);
    }
}

// Network slot z of a forward launch: 0 = online weights on the prestates, 1 = target weights on the poststates,
// 2 = online weights on the poststates (Double DQN's action choice, launched only when it is on).  Per-slot kernel
// parameters are picked with selects, never indexed by z, so they stay in the parameter bank instead of a local copy.
template <class T>
__device__ __forceinline__ T slot3(const T (&x)[3], int z) { return z == 2 ? x[2] : z ? x[1] : x[0]; }
template <class T>   // weights of slot z where only two networks exist: the target's for slot 1, the online's otherwise
__device__ __forceinline__ T wslot(const T (&x)[2], int z) { return z == 1 ? x[1] : x[0]; }

// ------------------------------------------------------------------------------------------
// Forward problems.  z selects the network slot: 0 = online (prestates), 1 = target (poststates), 2 = online on the
// poststates (the Double DQN action choice; only launched when it is on).
// ------------------------------------------------------------------------------------------

// conv1: A = u8 frames read in place (ring or staged states), k = (c, r, s) with c the frame of the
// history window; the /255 of _setInput (src/deepqnetwork.py:100) is applied to the fp32 accumulator, ReLU fused.
struct Conv1Fwd {
  const uint8_t* src[3];   // base of the frame array
  const int32_t* idx[3];   // per-sample frame index
  int shift[3];            // first frame of sample n is idx[n] + shift
  const float* w[3];
  float* out[3];
  int nb;
  int k1;                  // 64 * history_length
  static constexpr bool kAKContig = true, kBKContig = false;
  __device__ int M(int) const { return nb * kP1 * kP1; }
  __device__ int N(int) const { return kC1; }
  __device__ void krange(int, int& kb, int& ke) const { kb = 0; ke = k1; }
  __device__ float a(int z, int m, int k) const {
    const int n = m / (kP1 * kP1), pq = m % (kP1 * kP1), p = pq / kP1, q = pq % kP1;
    const int c = k >> 6, r = (k >> 3) & 7, s = k & 7;
    const int64_t f = static_cast<int64_t>(slot3(idx, z)[n]) + slot3(shift, z) + c;
    return static_cast<float>(slot3(src, z)[f * kFrameBytes + (p * 4 + r) * kFrameW + q * 4 + s]);
  }
  __device__ float b(int z, int k, int n) const { return slot3(w, z)[k * kC1 + n]; }
  __device__ void store(int z, int m, int n, float v) const {
    slot3(out, z)[m * kC1 + n] = fmaxf(v * (1.0f / 255.0f), 0.f);
  }
};

// Random-shift augmentation (b200dqn_net_config::random_shift): pixel (y, x) of a sample whose crop offsets are
// (dy, dx) = (crop[2n], crop[2n + 1]) reads frame pixel (clamp(y + dy, 0, 83), clamp(x + dx, 0, 83)): edge-replicate
// padding followed by a crop, without leaving the 84x84 frame.
__device__ __forceinline__ int crop_pixel(const int32_t* crop, int n, int y, int x) {
  const int yy = min(max(y + crop[2 * n], 0), kFrameH - 1), xx = min(max(x + crop[2 * n + 1], 0), kFrameW - 1);
  return yy * kFrameW + xx;
}

// conv1 forward on shifted states: crop[z] = the crop offsets of slot z ([nb][2] int32); slot 2 (Double DQN) reads
// slot 1's frames and therefore slot 1's offsets, which the caller sets explicitly in crop[2].
struct Conv1FwdCrop : Conv1Fwd {
  const int32_t* crop[3];
  __device__ float a(int z, int m, int k) const {
    const int n = m / (kP1 * kP1), pq = m % (kP1 * kP1), p = pq / kP1, q = pq % kP1;
    const int c = k >> 6, r = (k >> 3) & 7, s = k & 7;
    const int64_t f = static_cast<int64_t>(slot3(idx, z)[n]) + slot3(shift, z) + c;
    return static_cast<float>(slot3(src, z)[f * kFrameBytes + crop_pixel(slot3(crop, z), n, p * 4 + r, q * 4 + s)]);
  }
};

// conv2 / conv3: NHWC fp32 input, k = (r, s, c) so one filter row is (S*C) contiguous floats.
template <int H, int C, int R, int ST, int KO>
struct ConvFwd {
  static constexpr int P = (H - R) / ST + 1, K = R * R * C;
  const float* in[3];
  const float* w[3];
  float* out[3];
  int nb;
  static constexpr bool kAKContig = true, kBKContig = false;
  __device__ int M(int) const { return nb * P * P; }
  __device__ int N(int) const { return KO; }
  __device__ void krange(int, int& kb, int& ke) const { kb = 0; ke = K; }
  __device__ float a(int z, int m, int k) const {
    const int n = m / (P * P), pq = m % (P * P), p = pq / P, q = pq % P;
    const int r = k / (R * C), sc = k % (R * C);
    return slot3(in, z)[((n * H + p * ST + r) * H + q * ST) * C + sc];
  }
  __device__ float b(int z, int k, int n) const { return slot3(w, z)[k * KO + n]; }
  __device__ void store(int z, int m, int n, float v) const { slot3(out, z)[m * KO + n] = fmaxf(v, 0.f); }
};

// fc1 forward with split-K: z = net * splits + split; partial[z][m][n].  ReLU is applied by the
// consumer (the head) after it sums the splits.  W = fc1's width: kHidden, or kDuelHidden on a dueling net.
template <int W>
struct Fc1Fwd {
  const float* in[3];   // H3 flat [nb][3136]
  const float* w[3];    // W4 [3136][W]
  float* part;          // [nets*splits][nb][W]
  int nb, splits, kchunk;
  static constexpr bool kAKContig = true, kBKContig = false;
  __device__ int M(int) const { return nb; }
  __device__ int N(int) const { return W; }
  __device__ void krange(int z, int& kb, int& ke) const {
    kb = (z % splits) * kchunk;
    ke = min(kb + kchunk, kFlat);
  }
  __device__ float a(int z, int m, int k) const { return slot3(in, z / splits)[m * kFlat + k]; }
  __device__ float b(int z, int k, int n) const { return slot3(w, z / splits)[k * W + n]; }
  __device__ void store(int z, int m, int n, float v) const { part[(z * nb + m) * W + n] = v; }
};

// ------------------------------------------------------------------------------------------
// Backward problems (online network only).  "dZ" tensors already carry the ReLU mask of the layer
// that produced them: every dgrad store multiplies by (activation > 0) — Neon's Rectlin.bprop.
// ------------------------------------------------------------------------------------------

// fc1 dgrad: dZ3[b][k] = (sum_n dZ4[b][n] * W4[k][n]) * (H3[b][k] > 0)
template <int W>
struct Fc1Dgrad {
  const float* dz4;  // [nb][W]
  const float* w4;   // [3136][W]
  const float* h3;   // [nb][3136]
  float* dz3;        // [nb][3136]
  int nb;
  static constexpr bool kAKContig = true, kBKContig = true;
  __device__ int M(int) const { return nb; }
  __device__ int N(int) const { return kFlat; }
  __device__ void krange(int, int& kb, int& ke) const { kb = 0; ke = W; }
  __device__ float a(int, int m, int k) const { return dz4[m * W + k]; }
  __device__ float b(int, int k, int n) const { return w4[n * W + k]; }
  __device__ void store(int, int m, int n, float v) const {
    const int i = m * kFlat + n;
    dz3[i] = h3[i] > 0.f ? v : 0.f;
  }
};

// fc1 wgrad: dW4[k][n] = sum_b H3[b][k] * dZ4[b][n]   (reduction dim = batch, no split)
template <int W>
struct Fc1Wgrad {
  const float* h3;
  const float* dz4;
  float* dw4;  // [3136][W]
  int nb;
  static constexpr bool kAKContig = false, kBKContig = false;
  __device__ int M(int) const { return kFlat; }
  __device__ int N(int) const { return W; }
  __device__ void krange(int, int& kb, int& ke) const { kb = 0; ke = nb; }
  __device__ float a(int, int m, int k) const { return h3[k * kFlat + m]; }
  __device__ float b(int, int k, int n) const { return dz4[k * W + n]; }
  __device__ void store(int, int m, int n, float v) const { dw4[m * W + n] = v; }
};

// conv dgrad (input gradient of a stride-ST RxR conv, NHWC), decomposed by output-parity class
// z = (y % ST) * ST + (x % ST) so that only the R/ST x R/ST taps that can reach a pixel of that
// class are multiplied:  dX[n,y,x,c] = sum_{r',s',ko} dZ[n, yy-r', xx-s', ko] * W[(r,s,c)][ko],
// y = ST*yy + py, r = ST*r' + py (same for x/s).  Masked by (X > 0) on store.
template <int H, int C, int R, int ST, int KO>
struct ConvDgrad {
  static constexpr int P = (H - R) / ST + 1;
  static constexpr int RT = R / ST;          // taps per axis per class (R % ST == 0 here)
  static constexpr int HC = (H + ST - 1) / ST;  // pixels per axis per class
  static constexpr int K = RT * RT * KO;
  const float* dz;  // [nb][P][P][KO]
  const float* w;   // [(r,s,c)][KO]
  const float* x;   // [nb][H][H][C]  forward activation (mask)
  float* dx;        // [nb][H][H][C]
  int nb;
  static constexpr bool kAKContig = true, kBKContig = true;
  __device__ int M(int) const { return nb * HC * HC; }
  __device__ int N(int) const { return C; }
  __device__ void krange(int, int& kb, int& ke) const { kb = 0; ke = K; }
  __device__ float a(int z, int m, int k) const {
    const int n = m / (HC * HC), yx = m % (HC * HC), yy = yx / HC, xx = yx % HC;
    const int rp = k / (RT * KO), sp = (k / KO) % RT, ko = k % KO;
    const int py = z / ST, px = z % ST;
    if (yy * ST + py >= H || xx * ST + px >= H) return 0.f;
    const int p = yy - rp, q = xx - sp;
    if (p < 0 || p >= P || q < 0 || q >= P) return 0.f;
    return dz[((n * P + p) * P + q) * KO + ko];
  }
  __device__ float b(int z, int k, int c) const {
    const int rp = k / (RT * KO), sp = (k / KO) % RT, ko = k % KO;
    const int r = rp * ST + z / ST, s = sp * ST + z % ST;
    return w[((r * R + s) * C + c) * KO + ko];
  }
  __device__ void store(int z, int m, int c, float v) const {
    const int n = m / (HC * HC), yx = m % (HC * HC), yy = yx / HC, xx = yx % HC;
    const int y = yy * ST + z / ST, xq = xx * ST + z % ST;
    if (y >= H || xq >= H) return;
    const int i = ((n * H + y) * H + xq) * C + c;
    dx[i] = x[i] > 0.f ? v : 0.f;
  }
};

// conv wgrad (conv2, conv3): dW[(r,s,c)][ko] = sum_{n,p,q} X[n,p*ST+r,q*ST+s,c] * dZ[n,p,q,ko];
// split-K over z, partial[z][(r,s,c)][ko] summed (in fixed order) by the optimizer kernel.
template <int H, int C, int R, int ST, int KO>
struct ConvWgrad {
  static constexpr int P = (H - R) / ST + 1, KW = R * R * C;
  const float* x;   // [nb][H][H][C]
  const float* dz;  // [nb][P][P][KO]
  float* part;      // [splits][KW][KO]
  int nb, kchunk;
  static constexpr bool kAKContig = false, kBKContig = false;
  __device__ int M(int) const { return KW; }
  __device__ int N(int) const { return KO; }
  __device__ void krange(int z, int& kb, int& ke) const {
    kb = z * kchunk;
    ke = min(kb + kchunk, nb * P * P);
  }
  __device__ float a(int, int m, int k) const {
    const int n = k / (P * P), pq = k % (P * P), p = pq / P, q = pq % P;
    const int r = m / (R * C), sc = m % (R * C);
    return x[((n * H + p * ST + r) * H + q * ST) * C + sc];
  }
  __device__ float b(int, int k, int n) const { return dz[k * KO + n]; }
  __device__ void store(int z, int m, int n, float v) const { part[(z * KW + m) * KO + n] = v; }
};

// conv1 wgrad: the input is the u8 frame window (x = pixel / 255), k = (c, r, s) as in Conv1Fwd.
struct Conv1Wgrad {
  const uint8_t* src;
  const int32_t* idx;
  int shift;
  const float* dz;  // dZ1 [nb][20][20][32]
  float* part;      // [splits][k1][32]
  int nb, kchunk;
  int k1;           // 64 * history_length
  static constexpr bool kAKContig = false, kBKContig = false;
  __device__ int M(int) const { return k1; }
  __device__ int N(int) const { return kC1; }
  __device__ void krange(int z, int& kb, int& ke) const {
    kb = z * kchunk;
    ke = min(kb + kchunk, nb * kP1 * kP1);
  }
  __device__ float a(int, int m, int k) const {
    const int n = k / (kP1 * kP1), pq = k % (kP1 * kP1), p = pq / kP1, q = pq % kP1;
    const int c = m >> 6, r = (m >> 3) & 7, s = m & 7;
    const int64_t f = static_cast<int64_t>(idx[n]) + shift + c;
    return static_cast<float>(src[f * kFrameBytes + (p * 4 + r) * kFrameW + q * 4 + s]);
  }
  __device__ float b(int, int k, int n) const { return dz[k * kC1 + n]; }
  __device__ void store(int z, int m, int n, float v) const { part[(z * k1 + m) * kC1 + n] = v * (1.0f / 255.0f); }
};

// conv1 wgrad on shifted prestates: it re-reads the pixels, so it takes slot 0's crop offsets, as slot 0's forward did.
struct Conv1WgradCrop : Conv1Wgrad {
  const int32_t* crop;
  __device__ float a(int, int m, int k) const {
    const int n = k / (kP1 * kP1), pq = k % (kP1 * kP1), p = pq / kP1, q = pq % kP1;
    const int c = m >> 6, r = (m >> 3) & 7, s = m & 7;
    const int64_t f = static_cast<int64_t>(idx[n]) + shift + c;
    return static_cast<float>(src[f * kFrameBytes + crop_pixel(crop, n, p * 4 + r, q * 4 + s)]);
  }
};

}  // namespace b200
