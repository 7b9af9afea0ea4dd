// fp32 building blocks of the parallel-in-time stages around the AR kernel: the NAR refiner
// (reference nn/nar.py:13-116, model.py:307-347) and the prefill (model.py:172-216, nn/text.py:16-44,
// nn/speaker.py:64-85, nn/ref.py:16-160).  Their results are integer ids (NAR argmax) or inputs of the
// id-exact AR kernel (cond_ar, txt_seq), so every contraction is fp32 on the FMA pipe (element pairs, fp32
// accumulate) -- no tensor cores, no reduced precision.
//
//   dense_tile_kernel    C[M][N] = epi(prologue(A)[M][K] . W[N][K]^T): 128x128x16 tiles, 8x8 outputs per thread
//   dense_skinny_kernel  the same contract for M <= 16 rows (streaming windows, time-to-first-audio): the rows
//                        live in shared memory, one warp per output column, lanes split K; more rows in blocks of 16
//                        (grid.y), where a row's reduction order must not depend on M (Token2SV of a batch)
//   prologue             optional RMSNorm of the A rows (nn/blocks.py:32-37) and/or a vector added to every row
//   epilogues            bias | bias+GELU(erf) | bias+residual | GLU (value . sigmoid(gate), nn/blocks.py:16-23) |
//                        argmax partials (value desc, index asc == torch.argmax's first maximum)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dense {

// fma of an element pair, one rounding per element
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }

enum { EPI_BIAS = 0, EPI_GELU = 1, EPI_RES = 2, EPI_GLU = 3, EPI_ARGMAX = 4, EPI_RES_GATE = 5 };

struct DenseOp {
  const float* A;       // [M][K]
  const float* W;       // [N][K] (nn.Linear layout)
  const float* bias;    // [N] or null
  const float* norm_w;  // RMSNorm weight [K] applied to the rows of A on load, or null
  const float* a_add;   // [K] added to every row of A on load (after the norm), or null
  const float* R;       // residual [M][ldc] (EPI_RES / EPI_RES_GATE)
  float* C;             // [M][ldc]; GLU: [M][N/2]
  float* amax_val;      // EPI_ARGMAX: [M][parts]
  int* amax_idx;
  float gate;           // EPI_RES_GATE: C = R + gate * acc
  int M, N, K, ldc, epi, parts;
  // grouped launch (blockIdx.z = group, e.g. the heads of a NAR stage): per-group element strides of W / bias /
  // a_add; the argmax partials of group z start at z * M * parts
  size_t zW, zBias, zAdd;
};

__device__ __forceinline__ DenseOp group_of(const DenseOp& in) {
  DenseOp op = in;
  const size_t z = blockIdx.z;
  if (z) {
    op.W += z * in.zW;
    if (op.bias) op.bias += z * in.zBias;
    if (op.a_add) op.a_add += z * in.zAdd;
    if (op.amax_val) {
      op.amax_val += z * (size_t)in.M * in.parts;
      op.amax_idx += z * (size_t)in.M * in.parts;
    }
  }
  return op;
}

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }
__device__ __forceinline__ float sigmoid_ref(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ bool before(float av, int ai, float bv, int bi) { return av > bv || (av == bv && ai < bi); }

// weight row of tile column j (GLU: the first half of a tile are value rows, the second half their gate rows)
__device__ __forceinline__ int w_row(const DenseOp& op, int n0, int j, int BN) {
  if (op.epi != EPI_GLU) return n0 + j;
  const int half = BN / 2, D = op.N / 2, base = (n0 / BN) * half;
  return j < half ? base + j : D + base + (j - half);
}

constexpr int kBM = 128, kBN = 128, kBK = 16, kTileThreads = 256;

// BM x BN x 16 tiles, 256 threads as a 16 x 16 grid, (BM/16) x (BN/16) outputs per thread.  Three sizes
// (128x128 / 64x64 / 32x32): the host picks the largest one that still gives every SM a CTA.  Every output is ONE
// fma chain over k = 0 .. K-1 whatever the tile size, so the choice never changes a bit of the result.
template <int BM, int BN>
__global__ void __launch_bounds__(kTileThreads, 2) dense_tile_kernel(const DenseOp op_in) {
  constexpr int TM = BM / 16, TN = BN / 16, TP = TN / 2;  // thread tile; accumulators paired over columns
  static_assert((TM == 8 || TM == 4 || TM == 2) && (TN == 8 || TN == 4 || TN == 2), "tile sizes 128 / 64 / 32");
  constexpr int HA = BM >= 64 ? BM / 64 : 1, HB = BN >= 64 ? BN / 64 : 1;  // loader passes over the rows / columns
  const DenseOp op = group_of(op_in);
  __shared__ __align__(16) float As[2][kBK][BM + 4];
  __shared__ __align__(16) float Bs[2][kBK][BN + 4];
  __shared__ float inv_rms[BM];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int K = op.K;
  // ---- prologue: 1/rms of this tile's rows (one warp per row)
  if (op.norm_w) {
    for (int r = warp; r < BM; r += kTileThreads / 32) {
      const int m = m0 + r;
      float ss = 0.f;
      if (m < op.M) {
        const float* a = op.A + (size_t)m * K;
        for (int k = lane * 4; k < K; k += 128) {
          const float4 v = *reinterpret_cast<const float4*>(a + k);
          ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
      if (lane == 0) inv_rms[r] = 1.0f / sqrtf(ss / (float)K + 1e-6f);
    }
    __syncthreads();
  }
  // loader mapping: row = tid / 4 (+64 per pass), 4 consecutive k at (tid % 4) * 4
  const int lrow = tid >> 2, lk = (tid & 3) * 4;
  const bool la = lrow < BM, lb = lrow < BN;  // 32-wide tiles: only the first 128 threads load
  int wrow[HB];
#pragma unroll
  for (int h = 0; h < HB; ++h) {
    const int j = lrow + 64 * h;
    const int r = w_row(op, n0, j, BN);
    const bool ok = lb && (op.epi == EPI_GLU ? (n0 / BN) * (BN / 2) + (j % (BN / 2)) < op.N / 2 : r < op.N);
    wrow[h] = ok ? r : -1;
  }
  auto load_a = [&](int k0, int h) -> float4 {
    const int m = m0 + lrow + 64 * h;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (la && m < op.M) {
      v = *reinterpret_cast<const float4*>(op.A + (size_t)m * K + k0 + lk);
      if (op.norm_w) {
        const float inv = inv_rms[lrow + 64 * h];
        const float4 w = __ldg(reinterpret_cast<const float4*>(op.norm_w + k0 + lk));
        v.x = (v.x * inv) * w.x;
        v.y = (v.y * inv) * w.y;
        v.z = (v.z * inv) * w.z;
        v.w = (v.w * inv) * w.w;
      }
      if (op.a_add) {
        const float4 e = __ldg(reinterpret_cast<const float4*>(op.a_add + k0 + lk));
        v.x += e.x;
        v.y += e.y;
        v.z += e.z;
        v.w += e.w;
      }
    }
    return v;
  };
  auto load_b = [&](int k0, int h) -> float4 {
    return wrow[h] >= 0 ? __ldg(reinterpret_cast<const float4*>(op.W + (size_t)wrow[h] * K + k0 + lk)) : make_float4(0.f, 0.f, 0.f, 0.f);
  };
  auto store = [&](int buf, const float4 (&a)[HA], const float4 (&b)[HB]) {
#pragma unroll
    for (int h = 0; h < HA; ++h) {
      const int r = lrow + 64 * h;
      if (la) {
        As[buf][lk + 0][r] = a[h].x;
        As[buf][lk + 1][r] = a[h].y;
        As[buf][lk + 2][r] = a[h].z;
        As[buf][lk + 3][r] = a[h].w;
      }
    }
#pragma unroll
    for (int h = 0; h < HB; ++h) {
      const int r = lrow + 64 * h;
      if (lb) {
        Bs[buf][lk + 0][r] = b[h].x;
        Bs[buf][lk + 1][r] = b[h].y;
        Bs[buf][lk + 2][r] = b[h].z;
        Bs[buf][lk + 3][r] = b[h].w;
      }
    }
  };
  // thread tile rows.  128: {ty*4..+3, 64+ty*4..+3}; 64: ty*4..+3; 32: ty*2, ty*2+1.  Columns.  128: {tx*4..+3, 64+tx*4..+3};
  // 64: {tx*2, tx*2+1, 32+tx*2, 32+tx*2+1} (a GLU thread holds a channel's value AND gate column); 32: tx*2, tx*2+1 (no GLU)
  const int ty = tid >> 4, tx = tid & 15;
  auto row_of = [&](int i) { return TM == 8 ? (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4)) : ty * TM + i; };
  auto col_of = [&](int j) {  // first column of accumulator pair j
    return TN == 8 ? (j < 2 ? tx * 4 + 2 * j : 64 + tx * 4 + 2 * (j - 2)) : TN == 4 ? (j == 0 ? tx * 2 : 32 + tx * 2) : tx * 2;
  };
  float2 acc[TM][TP];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TP; ++j) acc[i][j] = make_float2(0.f, 0.f);
  float4 ra[HA], rb[HB];
#pragma unroll
  for (int h = 0; h < HA; ++h) ra[h] = load_a(0, h);
#pragma unroll
  for (int h = 0; h < HB; ++h) rb[h] = load_b(0, h);
  store(0, ra, rb);
  __syncthreads();
  const int nk = K / kBK;
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) {
#pragma unroll
      for (int h = 0; h < HA; ++h) ra[h] = load_a((kt + 1) * kBK, h);
#pragma unroll
      for (int h = 0; h < HB; ++h) rb[h] = load_b((kt + 1) * kBK, h);
    }
#pragma unroll
    for (int k = 0; k < kBK; ++k) {
      float a[TM];
      float2 b[TP];
      if constexpr (TM == 8) {
        const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
        const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
        a[0] = a0.x, a[1] = a0.y, a[2] = a0.z, a[3] = a0.w, a[4] = a1.x, a[5] = a1.y, a[6] = a1.z, a[7] = a1.w;
      } else if constexpr (TM == 4) {
        const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
        a[0] = a0.x, a[1] = a0.y, a[2] = a0.z, a[3] = a0.w;
      } else {
        const float2 a0 = *reinterpret_cast<const float2*>(&As[buf][k][ty * 2]);
        a[0] = a0.x, a[1] = a0.y;
      }
      if constexpr (TN == 8) {
        const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
        const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
        b[0] = make_float2(b0.x, b0.y), b[1] = make_float2(b0.z, b0.w), b[2] = make_float2(b1.x, b1.y), b[3] = make_float2(b1.z, b1.w);
      } else if constexpr (TN == 4) {
        b[0] = *reinterpret_cast<const float2*>(&Bs[buf][k][tx * 2]);
        b[1] = *reinterpret_cast<const float2*>(&Bs[buf][k][32 + tx * 2]);
      } else {
        b[0] = *reinterpret_cast<const float2*>(&Bs[buf][k][tx * 2]);
      }
#pragma unroll
      for (int i = 0; i < TM; ++i) {
        const float2 aa = make_float2(a[i], a[i]);
#pragma unroll
        for (int j = 0; j < TP; ++j) acc[i][j] = ffma2(aa, b[j], acc[i][j]);
      }
    }
    if (kt + 1 < nk) store(buf ^ 1, ra, rb);
    __syncthreads();
  }
  // ---- epilogue
  constexpr int half = BN / 2;
  if (op.epi == EPI_ARGMAX) {
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      float bv = -INFINITY;
      int bi = 0x7fffffff;
#pragma unroll
      for (int j = 0; j < TP; ++j) {
        const int c = n0 + col_of(j);
        const float v0 = acc[i][j].x + (op.bias && c < op.N ? __ldg(op.bias + c) : 0.f);
        const float v1 = acc[i][j].y + (op.bias && c + 1 < op.N ? __ldg(op.bias + c + 1) : 0.f);
        if (c < op.N && before(v0, c, bv, bi)) bv = v0, bi = c;
        if (c + 1 < op.N && before(v1, c + 1, bv, bi)) bv = v1, bi = c + 1;
      }
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) {  // the 16 threads of a row group are 16 consecutive lanes
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (before(ov, oi, bv, bi)) bv = ov, bi = oi;
      }
      const int m = m0 + row_of(i);
      if (tx == 0 && m < op.M) {
        op.amax_val[(size_t)m * op.parts + blockIdx.y] = bv;
        op.amax_idx[(size_t)m * op.parts + blockIdx.y] = bi;
      }
    }
    return;
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int m = m0 + row_of(i);
    if (m >= op.M) continue;
    if (op.epi == EPI_GLU) {
      // columns [0, BN/2) of the tile are value rows, [BN/2, BN) the gate rows of the same channels: the value pairs
      // j < TP/2 of a thread meet their gate pairs j + TP/2 (TN == 2: value and gate live in different threads -> not used)
      const int D = op.N / 2;
      if constexpr (TP >= 2) {
#pragma unroll
        for (int j = 0; j < TP / 2; ++j) {
          const int c = (n0 / BN) * half + (TN == 8 ? tx * 4 + 2 * j : tx * 2);
          const float v0 = acc[i][j].x + (c < D ? __ldg(op.bias + c) : 0.f), g0 = acc[i][j + TP / 2].x + (c < D ? __ldg(op.bias + D + c) : 0.f);
          const float v1 = acc[i][j].y + (c + 1 < D ? __ldg(op.bias + c + 1) : 0.f), g1 = acc[i][j + TP / 2].y + (c + 1 < D ? __ldg(op.bias + D + c + 1) : 0.f);
          if (c < D) op.C[(size_t)m * op.ldc + c] = v0 * sigmoid_ref(g0);
          if (c + 1 < D) op.C[(size_t)m * op.ldc + c + 1] = v1 * sigmoid_ref(g1);
        }
      }
      continue;
    }
#pragma unroll
    for (int j = 0; j < TP; ++j) {
      const int c = n0 + col_of(j);
      float v[2] = {acc[i][j].x, acc[i][j].y};
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        if (c + e >= op.N) continue;
        float x = v[e];
        if (op.bias) x += __ldg(op.bias + c + e);
        if (op.epi == EPI_GELU) x = gelu_erf(x);
        else if (op.epi == EPI_RES) x = op.R[(size_t)m * op.ldc + c + e] + x;
        else if (op.epi == EPI_RES_GATE) x = op.R[(size_t)m * op.ldc + c + e] + op.gate * x;
        op.C[(size_t)m * op.ldc + c + e] = x;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// M <= 16 rows.  The (normalised) rows are staged in shared memory once per CTA; each warp owns output columns
// n = first + warp, first + warp + 8, ...: lanes split K in float4 steps (coalesced weight reads straight from
// L2), 16 row accumulators per lane, transposed shuffle reduction, epilogue by the lane that ends up owning the row.
// grid.x CTAs x kCols columns each.  GLU: a "column" is a channel (value row + gate row).
// ---------------------------------------------------------------------------------------------
constexpr int kSkinnyRows = 16, kSkinnyThreads = 256;

template <int N>
__device__ __forceinline__ float reduce_transposed(float (&v)[N], int lane) {
  int n = N;
#pragma unroll
  for (int s = 16; s >= 1; s >>= 1) {
    if (n > 1) {
      const int half = n >> 1;
      const bool up = (lane & s) != 0;
#pragma unroll
      for (int i = 0; i < N / 2; ++i) {
        if (i < half) {
          const float keep = up ? v[i + half] : v[i];
          const float send = up ? v[i] : v[i + half];
          v[i] = keep + __shfl_xor_sync(0xffffffffu, send, s);
        }
      }
      n = half;
    } else {
      v[0] += __shfl_xor_sync(0xffffffffu, v[0], s);
    }
  }
  return v[0];
}

__global__ void __launch_bounds__(kSkinnyThreads) dense_skinny_kernel(const DenseOp op_in, int cols_per_cta) {
  DenseOp op = group_of(op_in);
  // more than 16 rows (never with the argmax epilogue): blockIdx.y = block of 16 rows, each row computed exactly as in
  // a launch of its own
  if (blockIdx.y) {
    const size_t r0 = (size_t)blockIdx.y * kSkinnyRows;
    op.A += r0 * op.K;
    op.C += r0 * op.ldc;
    if (op.R) op.R += r0 * op.ldc;
    op.M -= (int)r0;
  }
  extern __shared__ __align__(16) float xs[];  // [16][K]
  __shared__ float s_best_v[kSkinnyThreads / 32][kSkinnyRows];
  __shared__ int s_best_i[kSkinnyThreads / 32][kSkinnyRows];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int K = op.K, M = op.M;
  for (int r = warp; r < kSkinnyRows; r += kSkinnyThreads / 32) {
    float* d = xs + (size_t)r * K;
    if (r >= M) {
      for (int k = lane * 4; k < K; k += 128) *reinterpret_cast<float4*>(d + k) = make_float4(0.f, 0.f, 0.f, 0.f);
      continue;
    }
    const float* a = op.A + (size_t)r * K;
    float inv = 1.f;
    if (op.norm_w) {
      float ss = 0.f;
      for (int k = lane * 4; k < K; k += 128) {
        const float4 v = *reinterpret_cast<const float4*>(a + k);
        ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
      inv = 1.0f / sqrtf(ss / (float)K + 1e-6f);
    }
    for (int k = lane * 4; k < K; k += 128) {
      float4 v = *reinterpret_cast<const float4*>(a + k);
      if (op.norm_w) {
        const float4 w = __ldg(reinterpret_cast<const float4*>(op.norm_w + k));
        v.x = (v.x * inv) * w.x;
        v.y = (v.y * inv) * w.y;
        v.z = (v.z * inv) * w.z;
        v.w = (v.w * inv) * w.w;
      }
      if (op.a_add) {
        const float4 e = __ldg(reinterpret_cast<const float4*>(op.a_add + k));
        v.x += e.x;
        v.y += e.y;
        v.z += e.z;
        v.w += e.w;
      }
      *reinterpret_cast<float4*>(d + k) = v;
    }
  }
  __syncthreads();
  const bool glu = op.epi == EPI_GLU;
  const int ncol = glu ? op.N / 2 : op.N;
  const int c_lo = blockIdx.x * cols_per_cta, c_hi = min(ncol, c_lo + cols_per_cta);
  // after the transposed reduction lane L holds row (L >> 1) & 15
  const int my_row = (lane >> 1) & 15;
  const bool writer = (lane & 1) == 0 && my_row < M;
  float best_v = -INFINITY;
  int best_i = 0x7fffffff;
  for (int c = c_lo + warp; c < c_hi; c += kSkinnyThreads / 32) {
    const float* w0 = op.W + (size_t)c * K;
    const float* w1 = glu ? op.W + (size_t)(ncol + c) * K : nullptr;
    float acc[kSkinnyRows], accg[kSkinnyRows];
#pragma unroll
    for (int r = 0; r < kSkinnyRows; ++r) acc[r] = accg[r] = 0.f;
    for (int k = lane * 4; k < K; k += 128) {
      const float4 wv = __ldg(reinterpret_cast<const float4*>(w0 + k));
      float4 wg = make_float4(0.f, 0.f, 0.f, 0.f);
      if (glu) wg = __ldg(reinterpret_cast<const float4*>(w1 + k));
#pragma unroll
      for (int r = 0; r < kSkinnyRows; ++r) {
        const float4 x = *reinterpret_cast<const float4*>(xs + (size_t)r * K + k);
        acc[r] = fmaf(wv.x, x.x, acc[r]);
        acc[r] = fmaf(wv.y, x.y, acc[r]);
        acc[r] = fmaf(wv.z, x.z, acc[r]);
        acc[r] = fmaf(wv.w, x.w, acc[r]);
        if (glu) {
          accg[r] = fmaf(wg.x, x.x, accg[r]);
          accg[r] = fmaf(wg.y, x.y, accg[r]);
          accg[r] = fmaf(wg.z, x.z, accg[r]);
          accg[r] = fmaf(wg.w, x.w, accg[r]);
        }
      }
    }
    float v = reduce_transposed<kSkinnyRows>(acc, lane);
    float gv = 0.f;
    if (glu) gv = reduce_transposed<kSkinnyRows>(accg, lane);
    if (!writer) continue;
    const int m = my_row;
    if (glu) {
      v = (v + __ldg(op.bias + c)) * sigmoid_ref(gv + __ldg(op.bias + ncol + c));
      op.C[(size_t)m * op.ldc + c] = v;
      continue;
    }
    if (op.bias) v += __ldg(op.bias + c);
    if (op.epi == EPI_ARGMAX) {
      if (before(v, c, best_v, best_i)) best_v = v, best_i = c;
      continue;
    }
    if (op.epi == EPI_GELU) v = gelu_erf(v);
    else if (op.epi == EPI_RES) v = op.R[(size_t)m * op.ldc + c] + v;
    else if (op.epi == EPI_RES_GATE) v = op.R[(size_t)m * op.ldc + c] + op.gate * v;
    op.C[(size_t)m * op.ldc + c] = v;
  }
  if (op.epi == EPI_ARGMAX) {
    if ((lane & 1) == 0) {
      s_best_v[warp][my_row] = best_v;
      s_best_i[warp][my_row] = best_i;
    }
    __syncthreads();
    if (tid < M) {
      float bv = -INFINITY;
      int bi = 0x7fffffff;
      for (int w = 0; w < kSkinnyThreads / 32; ++w)
        if (before(s_best_v[w][tid], s_best_i[w][tid], bv, bi)) bv = s_best_v[w][tid], bi = s_best_i[w][tid];
      op.amax_val[(size_t)tid * op.parts + blockIdx.x] = bv;
      op.amax_idx[(size_t)tid * op.parts + blockIdx.x] = bi;
    }
  }
}

// final argmax over the per-tile partials of group z = blockIdx.y: out[m * out_stride + z] = index of the first maximum
__global__ void argmax_finish_kernel(const float* __restrict__ val, const int* __restrict__ idx, int M, int parts,
                                     int* __restrict__ out, int out_stride) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  const size_t z = blockIdx.y;
  if (m >= M) return;
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int p = 0; p < parts; ++p) {
    const float v = val[(z * M + m) * parts + p];
    const int i = idx[(z * M + m) * parts + p];
    if (before(v, i, bv, bi)) bv = v, bi = i;
  }
  out[(size_t)m * out_stride + z] = bi;
}

// ---------------------------------------------------------------------------------------------
// depthwise dilated Conv1d ("same" padding for the non-causal blocks, nn/blocks.py:63-74) + residual:
//   out[b][t][c] = x[b][t][c] + bias[c] + sum_j h[b][t + j*dil - left][c] * w[c][j]      (rows outside [0, len_b) are 0)
// rows are [B][Tmax][D]; len[b] <= Tmax valid rows per utterance (null = Tmax).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) dwconv_res_kernel(const float* __restrict__ h, const float* __restrict__ x,
                                                         const float* __restrict__ w, const float* __restrict__ bias,
                                                         float* __restrict__ out, const int* __restrict__ len, int Tmax, int D,
                                                         int k, int dil, int left) {
  const int t = blockIdx.x, b = blockIdx.y;
  const int L = len ? len[b] : Tmax;
  if (t >= L) return;
  const size_t base = (size_t)b * Tmax * D;
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    float acc = 0.f;
    for (int j = 0; j < k; ++j) {
      const int r = t + j * dil - left;
      if (r >= 0 && r < L) acc = fmaf(h[base + (size_t)r * D + c], __ldg(w + c * k + j), acc);
    }
    out[base + (size_t)t * D + c] = x[base + (size_t)t * D + c] + (acc + __ldg(bias + c));
  }
}

// RMSNorm of rows (one warp per row): y = (x * rsqrt(mean(x^2) + 1e-6)) * w, optionally followed by the FiLM-style
// modulation y * mul[c] + add[c] (NARStageAdapter: mul = 1 + tanh(g), add = tanh(b); nn/nar.py:28-32)
__global__ void __launch_bounds__(256) rmsnorm_rows_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                           const float* __restrict__ mul, const float* __restrict__ add,
                                                           float* __restrict__ y, long long rows, int D) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* xr = x + row * D;
  float ss = 0.f;
  for (int k = lane * 4; k < D; k += 128) {
    const float4 v = *reinterpret_cast<const float4*>(xr + k);
    ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float inv = 1.0f / sqrtf(ss / (float)D + 1e-6f);
  for (int k = lane; k < D; k += 32) {
    float v = (xr[k] * inv) * __ldg(w + k);
    if (mul) v = v * __ldg(mul + k) + __ldg(add + k);
    y[row * D + k] = v;
  }
}

}  // namespace dense
