// Mimi codec DECODE path on sm_90a: codes [B, Q, T] -> wav [B, T*1920].
//
// Replaces transformers.MimiModel.decode as called by the reference (codec/mimi.py:65-72):
// RVQ lookup-sum + 1x1 projections, depthwise 2x ConvTranspose upsample, 8-layer causal
// sliding-window transformer, SEANet decoder (modeling_mimi.py 5.5.0: _decode_frame :1613-1631,
// MimiSplitResidualVectorQuantizer.decode :1340-1350, MimiTransformerLayer :966-993,
// MimiAttention :681-738, MimiDecoder :1143-1173, MimiConvTranspose1d :402-409, MimiConv1d :331-351,
// MimiResnetBlock :437-451).
//
// Round-1 design (DESIGN.md §5): every dense block is an implicit GEMM over channel-last
// activations [T, C]: Linear, causal Conv1d (K = taps x Cin gathered from shifted rows) and causal
// ConvTranspose1d (stride s, kernel 2s == a 2-tap conv producing s*Cout columns, which IS the
// channel-last upsampled tensor), with ELU fused on the operand load and bias / GELU / LayerScale
// residual fused in the epilogue.  This first version runs the contractions in fp32 on the FMA
// pipe (parity 1e-4 against the fp32 oracle).  SOPRO_MIMI_BF16_TC mode (mimi_tc.cuh) runs every
// contraction after the RVQ projection on the tensor cores (wgmma) with bf16 operands, fp32
// accumulation in registers and the same fused epilogues; the fp32 kernels stay for the exact mode
// and for the small RVQ projection.
//
// The one-shot decode, the streaming step and the encoder's transformer share one host-side layer
// sequence (run_layers, seanet_f32 / seanet_tc); they differ only in data: the batch, the rows of left
// context in front of each conv operand and a stream's K/V rings.
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/sopro_b200.h"
#include "common.cuh"
#include "mimi_tc.cuh"

namespace mimi {

enum { EPI_NONE = 0, EPI_GELU = 1, EPI_RES_SCALE = 2, EPI_RES = 3 };

struct GemmOp {
  const float* A;   // channel-last input [B][Min][Cin]
  const float* W;   // [N][K], K = taps*Cin ordered (tap, ci)
  const float* bias;  // [bias_mod] or null
  const float* R;     // residual [B][M][N] or null
  const float* scale; // [N] LayerScale or null
  float* C;           // [B][M][ldc]
  long long a_bs, c_bs, r_bs;  // batch strides (floats)
  int M, N, K, Min, Cin, taps, dil, pad, ldc, bias_mod, epi, a_elu;
};

__device__ __forceinline__ float elu1(float x) { return x > 0.f ? x : expm1f(x); }
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

// C[m][n] = epi( sum_k A'[m][k] * W[n][k] + bias ),  A'[m][(j,ci)] = act(X[m + j*dil - pad][ci]) (0 outside)
template <int BN>
__global__ void __launch_bounds__(256) igemm_kernel(const GemmOp op) {
  constexpr int BM = 64, BK = 16, TM = 4, TN = BN / 16;
  __shared__ float As[2][BK][BM + 4];
  __shared__ float Bs[2][BK][BN + 4];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN, b = blockIdx.z;
  const float* X = op.A + (size_t)b * op.a_bs;
  const int lrow = tid >> 2, lk = (tid & 3) * 4;  // loader mapping: 64 rows x 4 float4 along k
  const int ty = tid >> 4, tx = tid & 15;
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  auto load_a = [&](int k0) -> float4 {
    const int kk = k0 + lk;
    const int j = kk / op.Cin, ci = kk - j * op.Cin;
    const int m = m0 + lrow;
    const int rin = m + j * op.dil - op.pad;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (m < op.M && rin >= 0 && rin < op.Min) {
      v = *reinterpret_cast<const float4*>(X + (size_t)rin * op.Cin + ci);
      if (op.a_elu) {
        v.x = elu1(v.x);
        v.y = elu1(v.y);
        v.z = elu1(v.z);
        v.w = elu1(v.w);
      }
    }
    return v;
  };
  auto load_b = [&](int k0) -> float4 {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (lrow < BN && n0 + lrow < op.N) v = __ldg(reinterpret_cast<const float4*>(op.W + (size_t)(n0 + lrow) * op.K + k0 + lk));
    return v;
  };
  auto store_tiles = [&](int buf, const float4& a, const float4& bq) {
    As[buf][lk + 0][lrow] = a.x;
    As[buf][lk + 1][lrow] = a.y;
    As[buf][lk + 2][lrow] = a.z;
    As[buf][lk + 3][lrow] = a.w;
    if (lrow < BN) {
      Bs[buf][lk + 0][lrow] = bq.x;
      Bs[buf][lk + 1][lrow] = bq.y;
      Bs[buf][lk + 2][lrow] = bq.z;
      Bs[buf][lk + 3][lrow] = bq.w;
    }
  };
  float4 ra = load_a(0), rb = load_b(0);
  store_tiles(0, ra, rb);
  __syncthreads();
  const int nk = op.K / BK;
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) {
      ra = load_a((kt + 1) * BK);
      rb = load_b((kt + 1) * BK);
    }
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a4 = *reinterpret_cast<const float4*>(&As[buf][k][ty * TM]);
      const float a[4] = {a4.x, a4.y, a4.z, a4.w};
      float bv[TN];
      if (TN == 4) {
        const float4 b4 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * TN]);
        bv[0] = b4.x;
        bv[1] = b4.y;
        bv[TN - 2] = b4.z;
        bv[TN - 1] = b4.w;
      } else {
        const float2 b2 = *reinterpret_cast<const float2*>(&Bs[buf][k][tx * TN]);
        bv[0] = b2.x;
        bv[TN - 1] = b2.y;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], bv[j], acc[i][j]);
    }
    if (kt + 1 < nk) store_tiles(buf ^ 1, ra, rb);
    __syncthreads();
  }
  float* Cb = op.C + (size_t)b * op.c_bs;
  const float* Rb = op.R ? op.R + (size_t)b * op.r_bs : nullptr;
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int m = m0 + ty * TM + i;
    if (m >= op.M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int n = n0 + tx * TN + j;
      if (n >= op.N) continue;
      float v = acc[i][j];
      if (op.bias) v += __ldg(op.bias + (n % op.bias_mod));
      if (op.epi == EPI_GELU) v = gelu_erf(v);
      else if (op.epi == EPI_RES_SCALE) v = Rb[(size_t)m * op.N + n] + __ldg(op.scale + n) * v;
      else if (op.epi == EPI_RES) v = Rb[(size_t)m * op.N + n] + v;
      Cb[(size_t)m * op.ldc + n] = v;
    }
  }
}

// RVQ lookup-sum: codes [B][Q][code_T] (frames [0, T) of each row) -> S [B][T][2*Dc] = [semantic sum | acoustic sum]
// A code outside [0, vocab) (an uncut EOS id, a negative pad) is clamped and recorded in *bad (sticky, read by
// sopro_mimi_check): the gather never leaves the table.  The reference's embedding lookup raises IndexError there.
__global__ void rvq_gather_kernel(const int* __restrict__ codes, const float* __restrict__ embed, float* __restrict__ S,
                                  int Q, int T, int code_T, int Dc, int vocab, int n_sem, int* __restrict__ bad) {
  const int t = blockIdx.x, b = blockIdx.y;
  for (int c = threadIdx.x; c < Dc; c += blockDim.x) {
    float s0 = 0.f, s1 = 0.f;
    for (int q = 0; q < Q; ++q) {
      int code = codes[((size_t)b * Q + q) * code_T + t];
      if (code < 0 || code >= vocab) {
        if (c == 0) atomicOr(bad, 1);
        code = min(max(code, 0), vocab - 1);
      }
      const float e = __ldg(embed + ((size_t)q * vocab + code) * Dc + c);
      if (q < n_sem) s0 += e;
      else s1 += e;
    }
    float* o = S + ((size_t)b * T + t) * (2 * Dc);
    o[c] = s0;
    o[Dc + c] = s1;
  }
}

// depthwise ConvTranspose k=4 s=2, causal: y[2t+r][c] = x[t][c]*w[c][r] + x[t-1][c]*w[c][r+2]
// `prev` (streaming): [B][C], each row's frame before x[0] (zeros at the start of a stream), else null
__global__ void upsample_kernel(const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ y, int T,
                                int C, const float* __restrict__ prev) {
  const int to = blockIdx.x, b = blockIdx.y;  // output row 0..2T-1
  const int t = to >> 1, r = to & 1;
  const float* xb = x + (size_t)b * T * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float v = xb[(size_t)t * C + c] * __ldg(w + c * 4 + r);
    if (t > 0) v += xb[(size_t)(t - 1) * C + c] * __ldg(w + c * 4 + r + 2);
    else if (prev) v += prev[(size_t)b * C + c] * __ldg(w + c * 4 + r + 2);
    y[((size_t)b * 2 * T + to) * C + c] = v;
  }
}

// LayerNorm over C (one warp per row)
__device__ __forceinline__ void put(float* p, float v) { *p = v; }
__device__ __forceinline__ void put(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }

template <typename OutT>
__global__ void layernorm_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bb,
                                 OutT* __restrict__ y, long long rows, int C, float eps) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* xr = x + row * C;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += xr[c];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / (float)C;
  float v = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float d = xr[c] - mean;
    v += d * d;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const float inv = 1.0f / sqrtf(v / (float)C + eps);
  for (int c = lane; c < C; c += 32) put(y + row * C + c, (xr[c] - mean) * inv * __ldg(w + c) + __ldg(bb + c));
}

// n4 float4s of item blockIdx.y: x + item * x_bs -> y + item * y_bs (strides in elements, multiples of 4)
__global__ void cast_bf16_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, long long n4, long long x_bs, long long y_bs) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float4 v = reinterpret_cast<const float4*>(x + blockIdx.y * x_bs)[i];
  const __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
  reinterpret_cast<uint2*>(y + blockIdx.y * y_bs)[i] = make_uint2(*reinterpret_cast<const uint32_t*>(&a), *reinterpret_cast<const uint32_t*>(&b));
}

// RoPE in place on the q and k thirds of QKV [rows][3C]; rope table [T2][Dh/2] cos, then sin
// Streaming (kring != null): row t sits at absolute position pos0 + t; its rotated key and its value are also
// appended to item b's ring of the layer, [B][R][C], at slot (pos0 + t) % R.
__global__ void rope_kernel(float* __restrict__ qkv, const float* __restrict__ cs, int T2, int tab_T2, int C, int H,
                            int pos0, float* __restrict__ kring, float* __restrict__ vring, int R) {
  const int t = blockIdx.x, b = blockIdx.y;
  const int Dh = C / H, half = Dh / 2;
  float* row = qkv + ((size_t)b * T2 + t) * 3 * C;
  const float* cosr = cs + (size_t)(pos0 + t) * half;
  const float* sinr = cs + (size_t)(tab_T2 + pos0 + t) * half;  // table: [cos rows 0..tab_T2) | sin rows 0..tab_T2)]
  for (int i = threadIdx.x; i < 2 * H * half; i += blockDim.x) {
    const int which = i / (H * half);  // 0 = q, 1 = k
    const int rem = i - which * H * half;
    const int h = rem / half, d = rem - h * half;
    float* p = row + which * C + h * Dh;
    const float x1 = p[d], x2 = p[d + half];
    const float c = cosr[d], s = sinr[d];
    p[d] = x1 * c - x2 * s;          // q*cos + rotate_half(q)*sin, first half: -x2
    p[d + half] = x2 * c + x1 * s;   // second half: +x1
  }
  if (kring) {
    __syncthreads();
    const size_t slot = ((size_t)b * R + (pos0 + t) % R) * C;
    for (int c4 = threadIdx.x * 4; c4 < C; c4 += blockDim.x * 4) {
      *reinterpret_cast<float4*>(kring + slot + c4) = *reinterpret_cast<const float4*>(row + C + c4);
      *reinterpret_cast<float4*>(vring + slot + c4) = *reinterpret_cast<const float4*>(row + 2 * C + c4);
    }
  }
}

// Tensor-core attention operands from the fp32 QKV rows [B][T2][3C]: rotated q and k as bf16 [B][T2][C], v transposed
// as bf16 [B][C][T2p] (keys contiguous: the K-major B operand of P.V).  32 rows per block.
template <int DH>
__global__ void __launch_bounds__(256) rope_pack_kernel(const float* __restrict__ qkv, const float* __restrict__ cs,
                                                        __nv_bfloat16* __restrict__ qh, __nv_bfloat16* __restrict__ kh,
                                                        __nv_bfloat16* __restrict__ vt, int T2, long long T2p, int tab_T2, int C, int H) {
  extern __shared__ __nv_bfloat16 sv[];  // [32][C + 2]
  constexpr int half = DH / 2;
  const int t0 = blockIdx.x * 32, b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rows = min(32, T2 - t0);
  for (int tt = warp; tt < rows; tt += 8) {  // one warp per row
    const int t = t0 + tt;
    const float* row = qkv + ((size_t)b * T2 + t) * 3 * C;
    const float* cosr = cs + (size_t)t * half;
    const float* sinr = cs + (size_t)(tab_T2 + t) * half;
#pragma unroll
    for (int which = 0; which < 2; ++which) {
      __nv_bfloat16* o = (which ? kh : qh) + ((size_t)b * T2 + t) * C;
      for (int i = lane; i < H * half; i += 32) {
        const int h = i / half, d = i % half;
        const float x1 = row[which * C + h * DH + d], x2 = row[which * C + h * DH + d + half];
        const float c = cosr[d], s = sinr[d];
        o[h * DH + d] = __float2bfloat16_rn(x1 * c - x2 * s);
        o[h * DH + d + half] = __float2bfloat16_rn(x2 * c + x1 * s);
      }
    }
    for (int c = lane * 4; c < C; c += 128) {
      const float4 v = *reinterpret_cast<const float4*>(row + 2 * C + c);
      __nv_bfloat16* d = sv + tt * (C + 2) + c;
      d[0] = __float2bfloat16_rn(v.x);
      d[1] = __float2bfloat16_rn(v.y);
      d[2] = __float2bfloat16_rn(v.z);
      d[3] = __float2bfloat16_rn(v.w);
    }
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < 32 * C; idx += blockDim.x) {
    const int c = idx >> 5, tt = idx & 31;
    if (t0 + tt < T2p) vt[((size_t)b * C + c) * T2p + t0 + tt] = tt < rows ? sv[tt * (C + 2) + c] : __float2bfloat16_rn(0.f);  // pad stays finite
  }
}

// causal sliding-window attention, one warp per (b, h, query); QKV rotated; out [B][T2][C]
// Streaming (kring != null): query row i sits at absolute position pos0 + i and the keys / values of positions
// [pos - window + 1, pos] are read from item b's ring of the layer (slot = position % R); the arithmetic and its order
// are the full decode's, so a chunked decode equals the full decode's prefix bit for bit in fp32 mode.
template <typename OutT>
__global__ void __launch_bounds__(256) attn_kernel(const float* __restrict__ qkv, OutT* __restrict__ out, int T2, int C,
                                                   int H, int window, int pos0, const float* __restrict__ kring,
                                                   const float* __restrict__ vring, int R) {
  extern __shared__ float sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int Dh = C / H;
  const int i = blockIdx.x * 8 + warp, h = blockIdx.y, b = blockIdx.z;
  float* qs = sm + warp * (Dh + window);
  float* sc = qs + Dh;
  if (i >= T2) return;
  const float* base = qkv + (size_t)b * T2 * 3 * C;
  const float* q = base + (size_t)i * 3 * C + h * Dh;
  // keys / values of position p: row p % R of item b's ring (streaming), else row p of the QKV rows
  const float* kb = kring ? kring + (size_t)b * R * C + h * Dh : base + C + h * Dh;
  const float* vb = vring ? vring + (size_t)b * R * C + h * Dh : base + 2 * C + h * Dh;
  const int kv_ld = kring ? C : 3 * C, kv_mod = kring ? R : INT_MAX;
  for (int d = lane; d < Dh; d += 32) qs[d] = q[d];
  __syncwarp();
  const int ia = pos0 + i;  // absolute position
  const int j0 = max(0, ia - window + 1);
  const int nk = ia - j0 + 1;
  const float scale = 1.0f / sqrtf((float)Dh);
  float mx = -INFINITY;
  for (int jj = lane; jj < nk; jj += 32) {
    const float* kr = kb + (size_t)((j0 + jj) % kv_mod) * kv_ld;
    float s = 0.f;
    for (int d = 0; d < Dh; d += 4) {
      const float4 kk = *reinterpret_cast<const float4*>(kr + d);
      s += kk.x * qs[d] + kk.y * qs[d + 1] + kk.z * qs[d + 2] + kk.w * qs[d + 3];
    }
    s *= scale;
    sc[jj] = s;
    mx = fmaxf(mx, s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
  for (int jj = lane; jj < nk; jj += 32) {
    const float e = expf(sc[jj] - mx);
    sc[jj] = e;
    sum += e;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  __syncwarp();
  const float inv = 1.0f / sum;
  for (int d = lane; d < Dh; d += 32) {
    float o = 0.f;
    for (int jj = 0; jj < nk; ++jj) o += (sc[jj] * inv) * vb[(size_t)((j0 + jj) % kv_mod) * kv_ld + d];
    put(out + ((size_t)b * T2 + i) * C + h * Dh + d, o);
  }
}

// final conv: ELU -> causal conv k taps, Cin -> 1
// rows r >= lo are readable (lo = 0: the causal zero pad; streaming: lo = -(taps-1), the carried context rows sit in
// front of x); item b of x starts at x + b * x_bs, its output at y + b * y_bs
__global__ void final_conv_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                  float* __restrict__ y, long long Tn, int Cin, int taps, int lo, long long x_bs, long long y_bs) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (t >= Tn) return;
  const float* xb = x + (size_t)b * x_bs;
  float acc = __ldg(bias);
  for (int j = 0; j < taps; ++j) {
    const long long r = t + j - (taps - 1);
    if (r < lo) continue;
    const float* xr = xb + r * Cin;
    for (int c = 0; c < Cin; c += 4) {
      const float4 v = *reinterpret_cast<const float4*>(xr + c);
      const float4 ww = __ldg(reinterpret_cast<const float4*>(w + j * Cin + c));
      acc += elu1(v.x) * ww.x + elu1(v.y) * ww.y + elu1(v.z) * ww.z + elu1(v.w) * ww.w;
    }
  }
  y[(size_t)b * y_bs + t] = acc;
}

// final conv on the bf16 activation [B][Tn][Cin] that already went through ELU (tensor-core mode): one thread per
// input row computes the row's dot product with every tap's weights (each row is read once), the taps are combined
// through shared memory.  256 - (taps-1) outputs per block.
__global__ void __launch_bounds__(256) final_conv_h_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ w,
                                                           const float* __restrict__ bias, float* __restrict__ y, long long Tn,
                                                           int Cin, int taps, int lo, long long x_bs, long long y_bs) {
  extern __shared__ float fsm[];  // [taps][256] partial dots, then [taps*Cin] weights
  float* sp = fsm;
  float* sw = fsm + taps * 256;
  const int tid = threadIdx.x, halo = taps - 1, per = 256 - halo, b = blockIdx.y;
  for (int i = tid; i < taps * Cin; i += 256) sw[i] = __ldg(w + i);
  __syncthreads();
  const long long r = (long long)blockIdx.x * per - halo + tid;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  if (r >= lo && r < Tn) {
    const uint4* xr = reinterpret_cast<const uint4*>(x + (long long)b * x_bs + r * Cin);
    for (int c = 0; c < Cin; c += 8) {
      const uint4 v = xr[c >> 3];
      const uint32_t u[4] = {v.x, v.y, v.z, v.w};
      float f[8];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        f[2 * e] = __uint_as_float(u[e] << 16);
        f[2 * e + 1] = __uint_as_float(u[e] & 0xffff0000u);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (j < taps) {
          const float* wj = sw + j * Cin + c;
#pragma unroll
          for (int e = 0; e < 8; ++e) acc[j] = fmaf(f[e], wj[e], acc[j]);
        }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j)
    if (j < taps) sp[j * 256 + tid] = acc[j];
  __syncthreads();
  if (tid >= halo && r < Tn) {  // output sample r: tap j reads row r + j - halo
    float o = __ldg(bias);
    for (int j = 0; j < taps; ++j) o += sp[j * 256 + tid - halo + j];
    y[(size_t)b * y_bs + r] = o;
  }
}

}  // namespace mimi

using namespace mimi;

namespace {
uint16_t bf16_rne(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);  // NaN stays NaN
  u += 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}

// bf16 copies of the GEMM weight matrices (tensor-core mode); offsets in elements, 256-B aligned
struct Bf16Arena {
  std::vector<uint16_t> host;
  size_t add(const float* p, size_t n) {
    const size_t off = (host.size() + 127) / 128 * 128;
    host.resize(off + n);
    for (size_t i = 0; i < n; ++i) host[off + i] = bf16_rne(p[i]);
    return off;
  }
};

struct DevArena {
  std::vector<float> host;
  size_t add(const float* p, size_t n) {
    const size_t off = (host.size() + 63) / 64 * 64;
    host.resize(off + n);
    if (p) memcpy(host.data() + off, p, n * 4);
    return off;
  }
};
}  // namespace

struct sopro_mimi {
  int device = 0;
  sopro_mimi_config_t cfg{};
  float* dev = nullptr;
  size_t n_floats = 0;
  // offsets (floats) into dev
  size_t embed = 0, rvq_w = 0, up_w = 0;
  struct Layer {
    size_t ln1w, ln1b, qkv, wo, ls1, ln2w, ln2b, fc1, fc2, ls2;
    size_t qkv_h, wo_h, fc1_h, fc2_h;  // bf16 arena
  };
  std::vector<Layer> layers;
  size_t c0w = 0, c0b = 0, c0w_h = 0;
  struct Stage {
    size_t tw, tb, r1w, r1b, r2w, r2b;
    size_t tw_h, r1w_h, r2w_h;  // bf16 arena
    int ratio, cin, cout;
  };
  __nv_bfloat16* dev_h = nullptr;  // bf16 weight arena
  int precision = SOPRO_MIMI_BF16_TC;
  std::vector<Stage> stages;
  size_t lw = 0, lb = 0;
  // rope table + workspace
  float* rope = nullptr;
  int rope_T2 = 0;
  float* ws = nullptr;
  size_t ws_bytes = 0;
  int* codes_dev = nullptr;
  size_t codes_cap = 0;
  int* bad_code = nullptr;  // sticky flag: a decode saw a code outside [0, vocab)
  // launch-bound small decodes (streaming chunks, time-to-first-audio) are replayed from CUDA graphs captured over
  // internal static buffers; every graph dies when the workspace or the rope table is reallocated
  struct Replay {
    int B, T, precision;
    cudaGraphExec_t exec;
  };
  std::vector<Replay> replays;
  int* g_codes = nullptr;   // [kGraphFrames * n_q]
  float* g_wav = nullptr;   // [kGraphFrames * hop]
  bool graphs = true;
  cudaStream_t cap_stream = nullptr;
};

namespace {
// one transformer layer's weights: fp32 into A (q, k and v concatenated into one [3C][C] matrix) and, when Hh is given,
// bf16 copies of its four GEMM matrices into Hh
sopro_mimi::Layer pack_layer(const sopro_mimi_layer_weights_t& L, int C, int FF, DevArena& A, Bf16Arena* Hh) {
  sopro_mimi::Layer d{};
  d.ln1w = A.add(L.ln1_w, C);
  d.ln1b = A.add(L.ln1_b, C);
  std::vector<float> qkv((size_t)3 * C * C);
  memcpy(qkv.data(), L.q_w, (size_t)C * C * 4);
  memcpy(qkv.data() + (size_t)C * C, L.k_w, (size_t)C * C * 4);
  memcpy(qkv.data() + (size_t)2 * C * C, L.v_w, (size_t)C * C * 4);
  d.qkv = A.add(qkv.data(), qkv.size());
  d.wo = A.add(L.o_w, (size_t)C * C);
  d.ls1 = A.add(L.ls1, C);
  d.ln2w = A.add(L.ln2_w, C);
  d.ln2b = A.add(L.ln2_b, C);
  d.fc1 = A.add(L.fc1_w, (size_t)FF * C);
  d.fc2 = A.add(L.fc2_w, (size_t)C * FF);
  d.ls2 = A.add(L.ls2, C);
  if (Hh) {
    d.qkv_h = Hh->add(qkv.data(), qkv.size());
    d.wo_h = Hh->add(L.o_w, (size_t)C * C);
    d.fc1_h = Hh->add(L.fc1_w, (size_t)FF * C);
    d.fc2_h = Hh->add(L.fc2_w, (size_t)C * FF);
  }
  return d;
}
}  // namespace

extern "C" {

int sopro_mimi_create(const sopro_mimi_config_t* cfg, const sopro_mimi_weights_t* w, int device, sopro_mimi_t** out) {
  if (!cfg || !w || !out) return fail(SOPRO_ERR_INVALID, "null argument");
  *out = nullptr;
  const int rc = open_device(device, "the Mimi decoder");
  if (rc != SOPRO_OK) return rc;
  const int C = cfg->hidden, Dc = cfg->codebook_dim, Q = cfg->n_q, V = cfg->vocab, NL = cfg->n_layers, FF = cfg->ffn;
  if (C % 64 || Dc % 4 || C != 2 * Dc || NL < 1 || cfg->n_ratios < 1 || cfg->n_ratios > 8 || cfg->n_heads < 1 || C % cfg->n_heads ||
      (C / cfg->n_heads) % 4 || FF % 16)
    return fail(SOPRO_ERR_INVALID, "unsupported Mimi geometry (hidden=%d codebook_dim=%d)", C, Dc);
  sopro_mimi* m = new sopro_mimi();
  m->device = device;
  m->cfg = *cfg;
  DevArena A;
  Bf16Arena Hh;
  m->embed = A.add(w->embed, (size_t)Q * V * Dc);
  {  // [C][2*Dc] = [W_sem | W_ac]
    std::vector<float> cat((size_t)C * 2 * Dc);
    for (int n = 0; n < C; ++n)
      for (int k = 0; k < Dc; ++k) {
        cat[(size_t)n * 2 * Dc + k] = w->sem_out_proj[(size_t)n * Dc + k];
        cat[(size_t)n * 2 * Dc + Dc + k] = w->ac_out_proj[(size_t)n * Dc + k];
      }
    m->rvq_w = A.add(cat.data(), cat.size());
  }
  m->up_w = A.add(w->upsample_w, (size_t)C * 4);
  for (int l = 0; l < NL; ++l) m->layers.push_back(pack_layer(w->layer[l], C, FF, A, &Hh));
  // conv weights [Cout][Cin][k] -> [Cout][(tap, ci)]
  auto repack_conv = [&](const float* src, int cout, int cin, int k, size_t* half_off) {
    std::vector<float> r((size_t)cout * k * cin);
    for (int co = 0; co < cout; ++co)
      for (int ci = 0; ci < cin; ++ci)
        for (int j = 0; j < k; ++j) r[((size_t)co * k + j) * cin + ci] = src[((size_t)co * cin + ci) * k + j];
    if (half_off) *half_off = Hh.add(r.data(), r.size());
    return A.add(r.data(), r.size());
  };
  int ch = cfg->num_filters << cfg->n_ratios;  // 1024
  m->c0w = repack_conv(w->conv0_w, ch, C, cfg->kernel, &m->c0w_h);
  m->c0b = A.add(w->conv0_b, ch);
  for (int s = 0; s < cfg->n_ratios; ++s) {
    const sopro_mimi_stage_weights_t& S = w->stage[s];
    sopro_mimi::Stage d;
    const int r = cfg->ratios[s], cin = ch, cout = ch / 2;
    d.ratio = r;
    d.cin = cin;
    d.cout = cout;
    // ConvTranspose weight [Cin][Cout][2r] -> [(phase, co)][(tap, ci)]: tap 0 <-> x[t-1] <-> w[.., phase + r], tap 1 <-> x[t] <-> w[.., phase]
    std::vector<float> tw((size_t)r * cout * 2 * cin);
    for (int ph = 0; ph < r; ++ph)
      for (int co = 0; co < cout; ++co)
        for (int ci = 0; ci < cin; ++ci) {
          const size_t n = (size_t)ph * cout + co;
          tw[(n * 2 + 0) * cin + ci] = S.convt_w[((size_t)ci * cout + co) * 2 * r + ph + r];
          tw[(n * 2 + 1) * cin + ci] = S.convt_w[((size_t)ci * cout + co) * 2 * r + ph];
        }
    d.tw = A.add(tw.data(), tw.size());
    d.tw_h = Hh.add(tw.data(), tw.size());
    d.tb = A.add(S.convt_b, cout);
    d.r1w = repack_conv(S.res1_w, cout / cfg->compress, cout, cfg->res_kernel, &d.r1w_h);
    d.r1b = A.add(S.res1_b, cout / cfg->compress);
    d.r2w = repack_conv(S.res2_w, cout, cout / cfg->compress, 1, &d.r2w_h);
    d.r2b = A.add(S.res2_b, cout);
    m->stages.push_back(d);
    ch = cout;
  }
  m->lw = repack_conv(w->last_w, 1, ch, cfg->last_kernel, nullptr);
  m->lb = A.add(w->last_b, 1);
  m->n_floats = A.host.size();
  cudaError_t err = cudaMalloc(&m->dev, m->n_floats * 4);
  if (err == cudaSuccess) err = cudaMemcpy(m->dev, A.host.data(), m->n_floats * 4, cudaMemcpyHostToDevice);
  if (err == cudaSuccess) err = cudaMalloc(&m->bad_code, 256);
  if (err == cudaSuccess) err = cudaMemset(m->bad_code, 0, 256);
  if (err == cudaSuccess) err = cudaMalloc(&m->dev_h, Hh.host.size() * 2);
  if (err == cudaSuccess) err = cudaMemcpy(m->dev_h, Hh.host.data(), Hh.host.size() * 2, cudaMemcpyHostToDevice);
  if (err == cudaSuccess && !tc::encode_tiled_fn()) {
    cudaFree(m->dev);
    cudaFree(m->dev_h);
    delete m;
    return fail(SOPRO_ERR_UNSUPPORTED, "driver has no cuTensorMapEncodeTiled entry point");
  }
  if (err != cudaSuccess) {
    if (m->dev) cudaFree(m->dev);
    if (m->dev_h) cudaFree(m->dev_h);
    delete m;
    return fail(SOPRO_ERR_CUDA, "Mimi weight upload failed: %s", cudaGetErrorString(err));
  }
  *out = m;
  return SOPRO_OK;
}

int sopro_mimi_destroy(sopro_mimi_t* m) {
  if (!m) return SOPRO_OK;
  cudaSetDevice(m->device);
  cudaFree(m->dev);
  cudaFree(m->dev_h);
  cudaFree(m->rope);
  cudaFree(m->ws);
  cudaFree(m->codes_dev);
  cudaFree(m->bad_code);
  for (auto& r : m->replays) cudaGraphExecDestroy(r.exec);
  cudaFree(m->g_codes);
  cudaFree(m->g_wav);
  if (m->cap_stream) cudaStreamDestroy(m->cap_stream);
  delete m;
  return SOPRO_OK;
}

int64_t sopro_mimi_samples_per_frame(const sopro_mimi_t* m) {
  if (!m) return 0;
  int64_t s = 2;
  for (int i = 0; i < m->cfg.n_ratios; ++i) s *= m->cfg.ratios[i];
  return s;
}

int sopro_mimi_set_precision(sopro_mimi_t* m, int precision) {
  if (!m) return fail(SOPRO_ERR_INVALID, "null argument");
  if (precision != SOPRO_MIMI_FP32 && precision != SOPRO_MIMI_BF16_TC) return fail(SOPRO_ERR_INVALID, "unknown precision %d", precision);
  m->precision = precision;
  return SOPRO_OK;
}

}  // extern "C"

namespace {
constexpr long long kGraphFrames = 64;  // decodes of at most this many frames (B*T) go through the graph cache

void drop_replays(sopro_mimi* m) {
  for (auto& r : m->replays) cudaGraphExecDestroy(r.exec);
  m->replays.clear();
}

// RoPE table [cos rows 0..n) | sin rows 0..n)] of n positions, replacing *tab (n rows recorded in *tab_n); uploads and
// synchronises, so never inside a stream capture
int make_rope(const sopro_mimi_config_t& c, int n, float** tab, int* tab_n, cudaStream_t st) {
  const int Dh = c.hidden / c.n_heads;
  cudaFree(*tab);
  *tab = nullptr;
  *tab_n = 0;
  std::vector<float> h((size_t)2 * n * (Dh / 2));
  for (int t = 0; t < n; ++t)
    for (int d = 0; d < Dh / 2; ++d) {
      const float inv = 1.0f / powf(c.rope_theta, (float)(2 * d) / (float)Dh);
      const float f = (float)t * inv;
      h[(size_t)t * (Dh / 2) + d] = cosf(f);
      h[(size_t)(n + t) * (Dh / 2) + d] = sinf(f);
    }
  CK(cudaMalloc(tab, h.size() * 4));
  CK(cudaMemcpyAsync(*tab, h.data(), h.size() * 4, cudaMemcpyHostToDevice, st));
  CK(cudaStreamSynchronize(st));
  *tab_n = n;
  return SOPRO_OK;
}

// Allocations and table uploads a decode of [B, T] needs; never called inside a stream capture.
// RoPE table covering at least T2 positions
int ensure_rope(sopro_mimi* m, int T2, cudaStream_t st) {
  if (m->rope_T2 >= T2) return SOPRO_OK;
  drop_replays(m);
  return make_rope(m->cfg, T2, &m->rope, &m->rope_T2, st);
}

int mimi_prepare(sopro_mimi* m, int B, int T, cudaStream_t st) {
  const sopro_mimi_config_t& c = m->cfg;
  const int C = c.hidden, T2 = 2 * T, FF = c.ffn;
  {
    // streams share the table: never shrink it, grow with headroom
    const int rc = ensure_rope(m, T2, st);
    if (rc) return rc;
  }
  long long up = 2;
  for (int i = 0; i < c.n_ratios; ++i) up *= c.ratios[i];
  const size_t big = (size_t)B * T * up * c.num_filters;
  const size_t tr = (size_t)B * T2 * (size_t)std::max(3 * C, FF);
  const size_t bufsz = (std::max(std::max(big, tr), (size_t)B * T2 * (c.num_filters << c.n_ratios)) + 63) / 64 * 64;
  const size_t xsz = ((size_t)B * T2 * C + 63) / 64 * 64;
  const size_t need = (3 * bufsz + 2 * xsz) * 4 + 3 * bufsz * 2;
  if (m->ws_bytes < need) {
    drop_replays(m);
    cudaFree(m->ws);
    m->ws = nullptr;
    m->ws_bytes = 0;
    cudaError_t e = cudaMalloc(&m->ws, need);
    if (e != cudaSuccess) return fail(SOPRO_ERR_CUDA, "Mimi workspace %zu MB: %s", need >> 20, cudaGetErrorString(e));
    m->ws_bytes = need;
  }
  return SOPRO_OK;
}

// Tensor-core mode runs every contraction after the RVQ projection on the wgmma tiles; a geometry they cannot take
// (none of Mimi's layers) is refused before the first launch.  The fp32 mode takes any geometry.
int check_tc_geometry(const sopro_mimi* m) {
  const sopro_mimi_config_t& c = m->cfg;
  const int C = c.hidden, FF = c.ffn;
  bool ok = tc::supported(3 * C, C, C) && tc::supported(C, C, C) && tc::supported(FF, C, C) && tc::supported(C, FF, FF) &&
            tc::supported(c.num_filters << c.n_ratios, c.kernel * C, C) && c.num_filters % 8 == 0 && c.last_kernel <= 8;
  for (const sopro_mimi::Stage& S : m->stages) {
    const int hid = S.cout / c.compress;
    ok = ok && tc::supported(S.ratio * S.cout, 2 * S.cin, S.cin) && tc::supported(hid, c.res_kernel * S.cout, S.cout) &&
         tc::supported(S.cout, hid, hid);
  }
  return ok ? (int)SOPRO_OK : fail(SOPRO_ERR_UNSUPPORTED, "tensor-core mode: unsupported Mimi geometry (use SOPRO_MIMI_FP32)");
}

// ---- the layer sequence shared by the one-shot decode, the streaming step and the encoder.  These routines only
//      enqueue kernels (no allocation, upload or synchronisation): the one-shot decode runs them under graph capture.

int launch_gemm(const GemmOp& op, int B, cudaStream_t st) {
  if (op.K % 16 || op.Cin % 4) return fail(SOPRO_ERR_INVALID, "igemm: K=%d Cin=%d not aligned", op.K, op.Cin);
  if (op.N % 64 == 0 || op.N > 32) {
    dim3 grid((op.M + 63) / 64, (op.N + 63) / 64, B);
    igemm_kernel<64><<<grid, 256, 0, st>>>(op);
  } else {
    dim3 grid((op.M + 63) / 64, (op.N + 31) / 32, B);
    igemm_kernel<32><<<grid, 256, 0, st>>>(op);
  }
  CK(cudaGetLastError());
  return SOPRO_OK;
}

// A channel-last GEMM operand: B items of [ctx + M] rows each, item b at p + b * pitch rows (pitch 0: ctx + M, the
// items back to back).  The first ctx rows of an item are left context (the rows a stream carried over from its
// previous chunk); with ctx = 0 the causal zero padding stands in for them.
struct Operand {
  const void* p;  // first context row of item 0
  long long M;
  int ctx, B;
  long long pitch;
  long long rows_per_item() const { return pitch > 0 ? pitch : M + ctx; }
};

// fp32 implicit GEMM (a causal conv of `taps` taps; a Linear with taps = 1) over an operand of cin channels:
// pad = taps - 1 - ctx zero rows, Min = M + ctx readable rows.  elu: ELU on the operand load.  Item b of the output
// (and of R) starts c_pitch (r_pitch) rows of N after item b - 1 (0: M rows).
int gemm_f32(const Operand& a, int cin, int taps, const float* W, const float* bias, int N, int bias_mod, int epi, const float* R,
             const float* scale, float* out, int elu, cudaStream_t st, long long c_pitch = 0, long long r_pitch = 0) {
  GemmOp g{};
  g.A = static_cast<const float*>(a.p); g.W = W; g.C = out; g.R = R; g.bias = bias; g.scale = scale;
  g.M = (int)a.M; g.N = N; g.K = taps * cin; g.Min = (int)(a.M + a.ctx); g.Cin = cin; g.taps = taps; g.dil = 1; g.pad = taps - 1 - a.ctx;
  g.ldc = N; g.bias_mod = bias_mod; g.epi = epi; g.a_elu = elu;
  g.a_bs = a.rows_per_item() * cin; g.c_bs = (c_pitch > 0 ? c_pitch : a.M) * N; g.r_bs = (r_pitch > 0 ? r_pitch : a.M) * N;
  return launch_gemm(g, a.B, st);
}

// tensor-core implicit GEMM over a bf16 operand (ELU already applied by its producer where the layer wants it), same
// operand geometry; fp32 and / or bf16 output (the same pitch), the bf16 copy through ELU when out_elu
int gemm_tc(const Operand& a, int cin, int taps, const __nv_bfloat16* W, const float* bias, int N, int bias_mod, int epi, const float* R,
            const float* scale, float* of, __nv_bfloat16* oh, int out_elu, cudaStream_t st, long long c_pitch = 0, long long r_pitch = 0) {
  tc::TcOp o{};
  o.bias = bias; o.R = R; o.scale = scale; o.out_f32 = of; o.out_bf16 = oh;
  o.c_bs = (c_pitch > 0 ? c_pitch : a.M) * N; o.r_bs = (r_pitch > 0 ? r_pitch : a.M) * N; o.a_pitch = a.rows_per_item();
  o.M = (int)a.M; o.N = N; o.K = taps * cin; o.Cin = cin; o.dil = 1; o.pad = taps - 1 - a.ctx;
  o.bias_mod = bias_mod; o.epi = epi; o.out_elu = out_elu;
  cudaError_t e = tc::launch(a.p, a.M + a.ctx, W, o, a.B, st);
  if (e != cudaSuccess) return fail(SOPRO_ERR_CUDA, "tensor-core GEMM (N=%d K=%d): %s", N, o.K, cudaGetErrorString(e));
  return SOPRO_OK;
}
static_assert((int)EPI_NONE == tc::EPI_NONE && (int)EPI_GELU == tc::EPI_GELU && (int)EPI_RES_SCALE == tc::EPI_RES_SCALE &&
                  (int)EPI_RES == tc::EPI_RES,
              "both GEMMs take the same epilogue codes");

// Scratch of the transformer layers.  ln, att and hid are fp32 in fp32 mode and bf16 in tensor-core mode; k and vt
// take the tensor-core attention's keys and transposed values (written by rope_pack_kernel with the queries in ln).
struct LayerBufs {
  void *ln, *att, *hid;  // LayerNorm output [rows][C], attention output [rows][C], MLP hidden [rows][FF]
  float* qkv;            // [rows][3C]
  __nv_bfloat16 *k, *vt;  // [rows][C], [B][C][T2 rounded up to 8]
};

// A stream's K/V rings [n_layers][B][R][C]: item b of layer l holds the rotated key / the value of position p in row
// p % R of k / v + (l*B + b)*R*C; row 0 of the chunk is position pos0
struct KVRing {
  float *k, *v;
  int R, pos0;
};

// Transformer layers (MimiTransformerLayer: x += LS1 * attn(LN1(x)); x += LS2 * MLP(LN2(x))) in place on the residual
// stream x [B][T2][C].  Attention: given a ring, the chunk's keys and values are appended to it and the queries attend
// over it; without one, tensor-core mode runs rope_pack_kernel + the tensor-core attention when its tiles take the
// geometry; otherwise the plain RoPE and attention kernels run.
int run_layers(const sopro_mimi_config_t& c, const std::vector<sopro_mimi::Layer>& layers, bool tcm, const float* Wd,
               const __nv_bfloat16* Wh, const float* rope, int rope_T2, float* x, int B, int T2, const LayerBufs& b,
               const KVRing* ring, cudaStream_t st) {
  const int C = c.hidden, H = c.n_heads, Dh = C / H, FF = c.ffn;
  const long long rows = (long long)B * T2;
  const unsigned ln_grid = (unsigned)((rows + 7) / 8);
  const size_t asm_bytes = (size_t)8 * (Dh + c.window) * 4, pack_bytes = (size_t)32 * (C + 2) * 2;
  const bool tc_attn = tcm && !ring && tc::attn_supported(C, H, c.window) && pack_bytes <= 48 * 1024;
  const long long T2p = (T2 + 7) / 8 * 8;  // v^T row pitch: tensor-map strides are multiples of 16 bytes
  const int pos0 = ring ? ring->pos0 : 0, R = ring ? ring->R : 1;
  // the layers over the LayerNorm output `ln`, the attention output `att` and the MLP hidden `hid`: bf16 in tensor-core
  // mode, fp32 otherwise
  auto run = [&](auto* ln, auto* att, auto* hid) -> int {
    using T = std::remove_pointer_t<decltype(ln)>;
    constexpr bool tc_mode = std::is_same<T, __nv_bfloat16>::value;
    // one Linear over the rows; with `scale` its result, times the LayerScale, is added to x.  Output: fp32 `of`, or
    // `oh` (the MLP hidden)
    auto lin = [&](const T* A, int K, size_t w, size_t w_h, int N, int epi, const float* scale, float* of, T* oh) -> int {
      const Operand a{A, T2, 0, B};
      const float* res = scale ? x : nullptr;
      if constexpr (tc_mode) return gemm_tc(a, K, 1, Wh + w_h, nullptr, N, N, epi, res, scale, of, oh, 0, st);
      else return gemm_f32(a, K, 1, Wd + w, nullptr, N, N, epi, res, scale, of ? of : oh, 0, st);
    };
    int rc;
    for (size_t li = 0; li < layers.size(); ++li) {
      const sopro_mimi::Layer& L = layers[li];
      layernorm_kernel<<<ln_grid, 256, 0, st>>>(x, Wd + L.ln1w, Wd + L.ln1b, ln, rows, C, c.norm_eps);
      if ((rc = lin(ln, C, L.qkv, L.qkv_h, 3 * C, EPI_NONE, nullptr, b.qkv, nullptr))) return rc;
      if (tc_attn) {
        if constexpr (tc_mode) {  // q goes to ln (dead until the next LayerNorm)
          rope_pack_kernel<tc::kAttnDh><<<dim3((T2 + 31) / 32, B), 256, pack_bytes, st>>>(b.qkv, rope, ln, b.k, b.vt, T2, T2p, rope_T2, C, H);
          CK(cudaGetLastError());
          cudaError_t ae = tc::launch_attn(ln, b.k, b.vt, att, B, T2, T2p, C, H, c.window, st);
          if (ae != cudaSuccess) return fail(SOPRO_ERR_CUDA, "tensor-core attention: %s", cudaGetErrorString(ae));
        }
      } else {
        float* kr = ring ? ring->k + li * (size_t)B * R * C : nullptr;
        float* vr = ring ? ring->v + li * (size_t)B * R * C : nullptr;
        rope_kernel<<<dim3(T2, B), 256, 0, st>>>(b.qkv, rope, T2, rope_T2, C, H, pos0, kr, vr, R);
        attn_kernel<<<dim3((T2 + 7) / 8, H, B), 256, asm_bytes, st>>>(b.qkv, att, T2, C, H, c.window, pos0, kr, vr, R);
        CK(cudaGetLastError());
      }
      if ((rc = lin(att, C, L.wo, L.wo_h, C, EPI_RES_SCALE, Wd + L.ls1, x, nullptr))) return rc;
      layernorm_kernel<<<ln_grid, 256, 0, st>>>(x, Wd + L.ln2w, Wd + L.ln2b, ln, rows, C, c.norm_eps);
      if ((rc = lin(ln, C, L.fc1, L.fc1_h, FF, EPI_GELU, nullptr, nullptr, hid))) return rc;
      if ((rc = lin(hid, FF, L.fc2, L.fc2_h, C, EPI_RES_SCALE, Wd + L.ls2, x, nullptr))) return rc;
    }
    return SOPRO_OK;
  };
  using bf16 = __nv_bfloat16;
  if (tcm) return run(static_cast<bf16*>(b.ln), static_cast<bf16*>(b.att), static_cast<bf16*>(b.hid));
  return run(static_cast<float*>(b.ln), static_cast<float*>(b.att), static_cast<float*>(b.hid));
}

}  // namespace

// Context rows a stream moves to the front of each row's slice of its conv operand buffers after a step (the
// parameter of tail_shift_kernel, so outside the anonymous namespace)
struct TailShift {
  void* base[16];
  long long pitch_bytes[16];             // one stream row's slice of the buffer
  int row_bytes[16], ctx[16], rows[16];  // rows = new rows written behind the ctx rows this step
  int n;
};

namespace {

// A SEANet activation buffer: `ctx` rows of left context in front of the rows a pass writes, item b at p + b * pitch
// rows (pitch 0: ctx + the pass's rows, the items back to back)
struct Buf {
  void* p;
  int ctx;
  long long pitch;
  template <typename T>
  T* rows(int cols) const { return static_cast<T*>(p) + (size_t)ctx * cols; }  // the first row item 0's pass writes
  Operand operand(long long M, int B) const { return {p, M, ctx, B, pitch}; }
};

// Buffers of one SEANet decoder pass.  fp32 mode: every buffer is fp32 and `h` holds the raw ResnetBlock hidden.
// Tensor-core mode: `in`, `a0`, `z`, `o` hold bf16 activations with their consumer's ELU applied, `zf` the fp32 skip
// (the ConvTranspose output) and `h` the bf16 ELU'd hidden of a block that does not take the fused kernel.
struct SeanetBufs {
  Buf in;  // conv0 operand [ctx + T2][C]: the residual stream itself (fp32) or its bf16 copy (tensor-core mode)
  Buf a0;  // conv0 output
  struct Stage {
    Buf z, h, o;  // ConvTranspose output, ResnetBlock hidden, block output
    float* zf;
  } stage[SOPRO_MIMI_MAX_RATIOS];
};

// records that `rows` new rows were written behind b's context rows (no-op without a record)
void carry(TailShift* ts, const Buf& b, int row_bytes, long long rows) {
  if (!ts) return;
  ts->base[ts->n] = b.p;
  ts->pitch_bytes[ts->n] = b.pitch * row_bytes;
  ts->row_bytes[ts->n] = row_bytes;
  ts->ctx[ts->n] = b.ctx;
  ts->rows[ts->n] = (int)rows;
  ++ts->n;
}

// SEANet decoder in fp32: conv0, per stage ELU -> ConvTranspose (stride r, kernel 2r: a 2-tap GEMM with r*Cout columns)
// and the ResnetBlock z + conv1(ELU(conv3(ELU(z)))), then ELU -> final conv into wav [B][T2 * prod(ratios)].  The
// tail shift of every buffer that holds a conv operand is recorded in *ts when ts is given.
int seanet_f32(const sopro_mimi* m, const SeanetBufs& b, int B, long long T2, TailShift* ts, float* wav, long long wav_pitch, cudaStream_t st) {
  const sopro_mimi_config_t& c = m->cfg;
  const float* Wd = m->dev;
  long long Tn = T2;
  int ch = c.num_filters << c.n_ratios, rc;
  if ((rc = gemm_f32(b.in.operand(Tn, B), c.hidden, c.kernel, Wd + m->c0w, Wd + m->c0b, ch, ch, EPI_NONE, nullptr, nullptr,
                     b.a0.rows<float>(ch), 0, st, b.a0.pitch)))
    return rc;
  carry(ts, b.in, c.hidden * 4, Tn);
  carry(ts, b.a0, ch * 4, Tn);
  Buf cur = b.a0;
  for (size_t si = 0; si < m->stages.size(); ++si) {
    const sopro_mimi::Stage& S = m->stages[si];
    const SeanetBufs::Stage& sb = b.stage[si];
    const int hid = S.cout / c.compress;
    // the ConvTranspose's S.ratio output rows of an input row are its S.ratio * S.cout columns: the output pitch in
    // input rows is z's pitch / S.ratio (stream layouts keep it whole)
    if ((rc = gemm_f32(cur.operand(Tn, B), S.cin, 2, Wd + S.tw, Wd + S.tb, S.ratio * S.cout, S.cout, EPI_NONE, nullptr, nullptr,
                       sb.z.rows<float>(S.cout), 1, st, sb.z.pitch / S.ratio)))
      return rc;
    Tn *= S.ratio;
    if ((rc = gemm_f32(sb.z.operand(Tn, B), S.cout, c.res_kernel, Wd + S.r1w, Wd + S.r1b, hid, hid, EPI_NONE, nullptr, nullptr,
                       sb.h.rows<float>(hid), 1, st, sb.h.pitch)))
      return rc;
    if ((rc = gemm_f32(sb.h.operand(Tn, B), hid, 1, Wd + S.r2w, Wd + S.r2b, S.cout, S.cout, EPI_RES, sb.z.rows<float>(S.cout), nullptr,
                       sb.o.rows<float>(S.cout), 1, st, sb.o.pitch, sb.z.pitch)))
      return rc;
    carry(ts, sb.z, S.cout * 4, Tn);
    carry(ts, sb.o, S.cout * 4, Tn);
    cur = sb.o;
    ch = S.cout;
  }
  final_conv_kernel<<<dim3((unsigned)((Tn + 255) / 256), B), 256, 0, st>>>(cur.rows<float>(ch), Wd + m->lw, Wd + m->lb, wav, Tn, ch,
                                                                            c.last_kernel, -cur.ctx, cur.operand(Tn, B).rows_per_item() * ch,
                                                                            wav_pitch > 0 ? wav_pitch : Tn);
  CK(cudaGetLastError());
  return SOPRO_OK;
}

// SEANet decoder in tensor-core mode (check_tc_geometry passed), from the fp32 residual stream x [B][T2][C].
// Activations that feed a contraction travel as bf16 with the consumer's ELU already applied; the ResnetBlock skip
// stays fp32.  A ResnetBlock runs in one launch when the fused kernel takes its geometry, else conv by conv.
int seanet_tc(const sopro_mimi* m, const float* x, const SeanetBufs& b, int B, long long T2, TailShift* ts, float* wav, long long wav_pitch,
              cudaStream_t st) {
  const sopro_mimi_config_t& c = m->cfg;
  const int C = c.hidden;
  const float* Wd = m->dev;
  const __nv_bfloat16* Wh = m->dev_h;
  long long Tn = T2;
  int ch = c.num_filters << c.n_ratios, rc;
  const long long n4 = T2 * C / 4;  // x [B][T2][C] packed -> each item's rows of `in`
  cast_bf16_kernel<<<dim3((unsigned)((n4 + 255) / 256), B), 256, 0, st>>>(x, b.in.rows<__nv_bfloat16>(C), n4, T2 * C,
                                                                          b.in.operand(Tn, B).rows_per_item() * C);
  CK(cudaGetLastError());
  if ((rc = gemm_tc(b.in.operand(Tn, B), C, c.kernel, Wh + m->c0w_h, Wd + m->c0b, ch, ch, tc::EPI_NONE, nullptr, nullptr, nullptr,
                    b.a0.rows<__nv_bfloat16>(ch), 1, st, b.a0.pitch)))
    return rc;
  carry(ts, b.in, C * 2, Tn);
  carry(ts, b.a0, ch * 2, Tn);
  Buf cur = b.a0;
  for (size_t si = 0; si < m->stages.size(); ++si) {
    const sopro_mimi::Stage& S = m->stages[si];
    const SeanetBufs::Stage& sb = b.stage[si];
    const int hid = S.cout / c.compress;
    // ELU -> ConvTranspose: fp32 skip zf, bf16 ELU(z) for the ResnetBlock
    // (zf, which has no context rows, is laid out with z's pitch: one GEMM writes both)
    if ((rc = gemm_tc(cur.operand(Tn, B), S.cin, 2, Wh + S.tw_h, Wd + S.tb, S.ratio * S.cout, S.cout, tc::EPI_NONE, nullptr, nullptr,
                      sb.zf, sb.z.rows<__nv_bfloat16>(S.cout), 1, st, sb.z.pitch / S.ratio)))
      return rc;
    Tn *= S.ratio;
    if (tc::resblock_supported(hid, S.cout) && (S.cout * c.res_kernel) % 64 == 0) {
      tc::ResOp ro{};
      ro.bias1 = Wd + S.r1b;
      ro.bias2 = Wd + S.r2b;
      ro.Z = sb.zf;
      ro.out_bf16 = sb.o.rows<__nv_bfloat16>(S.cout);
      ro.M = (int)Tn;
      ro.Min = (int)Tn + sb.z.ctx;
      ro.taps = c.res_kernel;
      ro.pad = c.res_kernel - 1 - sb.z.ctx;
      ro.out_elu = 1;
      ro.a_pitch = sb.z.pitch;
      ro.z_bs = sb.z.pitch * S.cout;
      ro.o_bs = sb.o.pitch * S.cout;
      cudaError_t fe = tc::launch_resblock(sb.z.p, Wh + S.r1w_h, Wh + S.r2w_h, hid, ro, B, st);
      if (fe != cudaSuccess) return fail(SOPRO_ERR_CUDA, "fused ResnetBlock (stage %zu): %s", si, cudaGetErrorString(fe));
    } else {  // conv k=3 -> ELU(h) bf16, then the 1x1 conv + fp32 skip
      if ((rc = gemm_tc(sb.z.operand(Tn, B), S.cout, c.res_kernel, Wh + S.r1w_h, Wd + S.r1b, hid, hid, tc::EPI_NONE, nullptr, nullptr,
                        nullptr, sb.h.rows<__nv_bfloat16>(hid), 1, st, sb.h.pitch)))
        return rc;
      if ((rc = gemm_tc(sb.h.operand(Tn, B), hid, 1, Wh + S.r2w_h, Wd + S.r2b, S.cout, S.cout, tc::EPI_RES, sb.zf, nullptr, nullptr,
                        sb.o.rows<__nv_bfloat16>(S.cout), 1, st, sb.o.pitch, sb.z.pitch)))
        return rc;
    }
    carry(ts, sb.z, S.cout * 2, Tn);
    carry(ts, sb.o, S.cout * 2, Tn);
    cur = sb.o;
    ch = S.cout;
  }
  const int per = 256 - (c.last_kernel - 1);
  final_conv_h_kernel<<<dim3((unsigned)((Tn + per - 1) / per), B), 256, (size_t)(c.last_kernel * 256 + c.last_kernel * ch) * 4, st>>>(
      cur.rows<__nv_bfloat16>(ch), Wd + m->lw, Wd + m->lb, wav, Tn, ch, c.last_kernel, -cur.ctx, cur.operand(Tn, B).rows_per_item() * ch,
      wav_pitch > 0 ? wav_pitch : Tn);
  CK(cudaGetLastError());
  return SOPRO_OK;
}

// One-shot decode of codes [B][Q][T] into the workspace mimi_prepare sized: RVQ, projection, upsample, transformer,
// SEANet.  Enqueues only (it runs under graph capture).
int mimi_enqueue(sopro_mimi* m, const int32_t* codes, int B, int T, float* wav, cudaStream_t st) {
  const sopro_mimi_config_t& c = m->cfg;
  const int C = c.hidden, T2 = 2 * T, FF = c.ffn;
  const float* Wd = m->dev;
  const bool use_tc = m->precision == SOPRO_MIMI_BF16_TC;
  // ---- workspace (mimi_prepare): three fp32 ping-pong buffers sized for the widest SEANet activation + transformer
  //      scratch, the residual stream and its normalised copy, three bf16 buffers for the tensor-core operands
  long long up = 2;
  for (int i = 0; i < c.n_ratios; ++i) up *= c.ratios[i];
  const size_t big = (size_t)B * T * up * c.num_filters;                     // [T*1920][64]
  const size_t tr = (size_t)B * T2 * (size_t)std::max(3 * C, FF);            // QKV / MLP hidden
  const size_t bufsz = (std::max(std::max(big, tr), (size_t)B * T2 * (c.num_filters << c.n_ratios)) + 63) / 64 * 64;
  const size_t xsz = ((size_t)B * T2 * C + 63) / 64 * 64;
  float* b0 = m->ws;
  float* b1 = b0 + bufsz;
  float* b2 = b1 + bufsz;
  float* x = b2 + bufsz;    // residual stream [B][T2][C]
  float* ln = x + xsz;      // normalised copy (fp32 mode)
  __nv_bfloat16* h0 = reinterpret_cast<__nv_bfloat16*>(ln + xsz);
  __nv_bfloat16* h1 = h0 + bufsz;
  __nv_bfloat16* h2 = h1 + bufsz;
  // ---- RVQ + projection + upsample (small; fp32 in both modes)
  rvq_gather_kernel<<<dim3(T, B), 256, 0, st>>>(codes, Wd + m->embed, b0, c.n_q, T, T, c.codebook_dim, c.vocab, c.n_sem, m->bad_code);
  CK(cudaGetLastError());
  int rc;
  if ((rc = gemm_f32({b0, T, 0, B}, C, 1, Wd + m->rvq_w, nullptr, C, C, EPI_NONE, nullptr, nullptr, b1, 0, st))) return rc;
  upsample_kernel<<<dim3(T2, B), 256, 0, st>>>(b1, Wd + m->up_w, x, T, C, nullptr);
  CK(cudaGetLastError());
  // ---- transformer: b1 (idle until the SEANet) takes the attention output; tensor-core mode: the LayerNorm copy and
  //      q in h0, k in h1, v^T and the MLP hidden in h2
  LayerBufs lb{};
  lb.ln = use_tc ? (void*)h0 : ln;
  lb.qkv = b0;
  lb.att = b1;
  lb.hid = use_tc ? (void*)h2 : b0;
  lb.k = h1;
  lb.vt = h2;
  if ((rc = run_layers(c, m->layers, use_tc, Wd, m->dev_h, m->rope, m->rope_T2, x, B, T2, lb, nullptr, st))) return rc;
  // ---- SEANet decoder over ping-pong buffers, no context rows.  fp32: x -> b0, per stage b0 -> b1 -> b2 -> b0.
  //      Tensor-core: bf16 copy of x in h2 -> h0, per stage h0 -> h1 (+ fp32 skip b1) -> [h2] -> h0
  SeanetBufs sb{};
  sb.in = {use_tc ? (void*)h2 : x, 0, 0};
  sb.a0 = {use_tc ? (void*)h0 : b0, 0, 0};
  for (int i = 0; i < c.n_ratios; ++i)
    sb.stage[i] = use_tc ? SeanetBufs::Stage{{h1, 0, 0}, {h2, 0, 0}, {h0, 0, 0}, b1} : SeanetBufs::Stage{{b1, 0, 0}, {b2, 0, 0}, {b0, 0, 0}, nullptr};
  return use_tc ? seanet_tc(m, x, sb, B, T2, nullptr, wav, 0, st) : seanet_f32(m, sb, B, T2, nullptr, wav, 0, st);
}
}  // namespace

extern "C" {

int sopro_mimi_decode(sopro_mimi_t* m, const int32_t* codes, int B, int T, float* wav, void* stream) {
  if (!m || !codes || !wav) return fail(SOPRO_ERR_INVALID, "null argument");
  if (B < 1 || T < 1) return fail(SOPRO_ERR_INVALID, "B and T must be >= 1");
  if (B > 65535) return fail(SOPRO_ERR_INVALID, "B must be <= 65535");
  if ((long long)T * sopro_mimi_samples_per_frame(m) > 0x7fffffffLL) return fail(SOPRO_ERR_INVALID, "sequence too long for one launch");
  int rc;
  if (m->precision == SOPRO_MIMI_BF16_TC && (rc = check_tc_geometry(m))) return rc;
  CK(cudaSetDevice(m->device));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if ((rc = mimi_prepare(m, B, T, st))) return rc;
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  CK(cudaStreamIsCapturing(st, &cap));
  if (!m->graphs || (long long)B * T > kGraphFrames || cap != cudaStreamCaptureStatusNone) return mimi_enqueue(m, codes, B, T, wav, st);
  const size_t nc = (size_t)B * m->cfg.n_q * T, nw = (size_t)B * T * (size_t)sopro_mimi_samples_per_frame(m);
  if (!m->g_codes) {
    CK(cudaMalloc(&m->g_codes, (size_t)kGraphFrames * m->cfg.n_q * 4));
    CK(cudaMalloc(&m->g_wav, (size_t)kGraphFrames * (size_t)sopro_mimi_samples_per_frame(m) * 4));
  }
  cudaGraphExec_t exec = nullptr;
  for (auto& r : m->replays)
    if (r.B == B && r.T == T && r.precision == m->precision) exec = r.exec;
  if (!exec) {
    if (m->replays.size() >= 32) drop_replays(m);
    // captured on a private stream (the caller's may be the legacy default stream, which cannot capture)
    if (!m->cap_stream) CK(cudaStreamCreateWithFlags(&m->cap_stream, cudaStreamNonBlocking));
    CK(cudaStreamBeginCapture(m->cap_stream, cudaStreamCaptureModeThreadLocal));
    rc = mimi_enqueue(m, m->g_codes, B, T, m->g_wav, m->cap_stream);
    cudaGraph_t graph = nullptr;
    cudaError_t ce = cudaStreamEndCapture(m->cap_stream, &graph);
    if (rc) {
      if (graph) cudaGraphDestroy(graph);
      return rc;
    }
    if (ce != cudaSuccess) return fail(SOPRO_ERR_CUDA, "Mimi graph capture: %s", cudaGetErrorString(ce));
    ce = cudaGraphInstantiate(&exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ce != cudaSuccess) return fail(SOPRO_ERR_CUDA, "Mimi graph instantiate: %s", cudaGetErrorString(ce));
    m->replays.push_back({B, T, m->precision, exec});
  }
  CK(cudaMemcpyAsync(m->g_codes, codes, nc * 4, cudaMemcpyDeviceToDevice, st));
  CK(cudaGraphLaunch(exec, st));
  CK(cudaMemcpyAsync(wav, m->g_wav, nw * 4, cudaMemcpyDeviceToDevice, st));
  return SOPRO_OK;
}

}  // extern "C"


// ---------------------------------------------------------------------------------------------
// Streaming decode with persistent state (reference codec/mimi.py:83-181 MimiStreamDecoder; transformers
// modeling_mimi.py:77-170 MimiConv1dPaddingCache is the per-conv left context this replaces).
//
// A stream owns (a) one K/V ring per transformer layer holding the rotated keys and the values of the last
// `window` positions, (b) the previous RVQ frame (the depthwise ConvTranspose upsampler reads x[t-1]) and (c) for every
// causal conv of the SEANet decoder the last (taps-1) input rows.  (c) is stored IN PLACE: each conv input buffer is
// laid out [context rows | rows of this chunk]; the conv runs as a "valid" convolution over it (pad = 0,
// Min = M + taps - 1) and afterwards the buffer's last context-many rows are moved to its front.  At the start of a
// stream the context rows are zero, which is exactly the causal zero padding of the full decode, and every kernel
// computes each output element in the same order as the full decode: in fp32 mode the chunks are bit-identical to the
// full decode's prefix.  Work per chunk is O(chunk), not O(prefix).
// ---------------------------------------------------------------------------------------------
// one block per (buffer, stream row): rows [rows, rows + ctx) -> [0, ctx) of the row's slice (through shared memory:
// the ranges may overlap)
__global__ void __launch_bounds__(256) tail_shift_kernel(const TailShift ts) {
  extern __shared__ uint4 tsm[];
  const int i = blockIdx.x;
  const int n16 = ts.ctx[i] * ts.row_bytes[i] / 16;
  unsigned char* base = reinterpret_cast<unsigned char*>(ts.base[i]) + (size_t)blockIdx.y * (size_t)ts.pitch_bytes[i];
  const uint4* src = reinterpret_cast<const uint4*>(base + (size_t)ts.rows[i] * ts.row_bytes[i]);
  uint4* dst = reinterpret_cast<uint4*>(base);
  for (int e = threadIdx.x; e < n16; e += blockDim.x) tsm[e] = src[e];
  __syncthreads();
  for (int e = threadIdx.x; e < n16; e += blockDim.x) dst[e] = tsm[e];
}

// `rows` utterances decoded side by side, frame count shared.  Every per-utterance buffer is [rows][pitch][...] with a
// pitch fixed at create time, so a stream row's state never moves and every kernel reads and writes only its own row.
struct sopro_mimi_stream {
  sopro_mimi* m = nullptr;
  int max_n = 0, precision = 0, R = 0, rows = 1;
  long long frames = 0;
  unsigned char* slab = nullptr;
  size_t slab_bytes = 0, state_bytes = 0;
  // ---- state (zeroed by reset): [up_prev | K rings | V rings | conv-context rows at the front of the buffers below]
  float* up_prev = nullptr;                  // [rows][C]
  float *kring = nullptr, *vring = nullptr;  // [n_layers][rows][R][C]
  // ---- chunk buffers
  float *S = nullptr, *E = nullptr, *X = nullptr;  // [rows][n][2Dc], [rows][n][C], residual stream [rows][2n][C]
  LayerBufs tr{};  // transformer scratch (ln, att, hid: bf16 views in tensor-core mode)
  // SEANet buffers, each conv operand [rows][taps-1 context rows | Tn rows] (fp32 raw | bf16 ELU'd): in [2 + T2][C]
  // (a copy of X), a0 [1 + T2][16F], z [2 + Tn][cout], o [ctx + Tn][cout] with ctx = 1 (next ConvTranspose) or taps-1
  // (final conv); h [Tn][cout/2] has no context, zf [Tn][cout] (tensor-core mode) none either but z's pitch
  SeanetBufs sea{};
  int* codes_dev = nullptr;
  float* wav_dev = nullptr;
};

namespace {
struct SlabPlan {
  size_t off = 0;
  size_t take(size_t bytes) {
    const size_t o = off;
    off = (off + bytes + 255) / 256 * 256;
    return o;
  }
};

// lays the stream's slab out; with base == nullptr only sizes are computed
void stream_layout(sopro_mimi_stream* s, unsigned char* base) {
  const sopro_mimi_config_t& c = s->m->cfg;
  const bool tcm = s->precision == SOPRO_MIMI_BF16_TC;
  const size_t C = c.hidden, FF = c.ffn, n = s->max_n, T2 = 2 * n, NL = c.n_layers, rows = s->rows;
  const size_t es = tcm ? 2 : 4;  // element size of the conv operands
  SlabPlan P;
  auto at = [&](size_t o) { return base ? base + o : nullptr; };
  // a buffer of `ctx` context rows and up to Tn chunk rows per stream row, the pitch a multiple of `unit` rows
  auto buf = [&](int ctx, size_t Tn, size_t cols, size_t esz, size_t unit) -> Buf {
    const size_t pitch = (ctx + Tn + unit - 1) / unit * unit;
    return {at(P.take(rows * pitch * cols * esz)), ctx, (long long)pitch};
  };
  // state first
  s->up_prev = (float*)at(P.take(rows * C * 4));
  s->kring = (float*)at(P.take(NL * rows * s->R * C * 4));
  s->vring = (float*)at(P.take(NL * rows * s->R * C * 4));
  // conv operand buffers: the context rows at their fronts are state too, so they come next.  A ConvTranspose output's
  // pitch is a whole number of its input rows (the GEMM writes ratio rows per input row).
  s->sea.in = buf(c.kernel - 1, T2, C, es, 1);
  size_t ch = (size_t)c.num_filters << c.n_ratios, Tn = T2;
  s->sea.a0 = buf(1, Tn, ch, es, 1);
  for (int i = 0; i < c.n_ratios; ++i) {
    const size_t cout = ch / 2;
    Tn *= c.ratios[i];
    const int ctx_o = i + 1 == c.n_ratios ? c.last_kernel - 1 : 1;
    s->sea.stage[i].z = buf(c.res_kernel - 1, Tn, cout, es, c.ratios[i]);
    s->sea.stage[i].o = buf(ctx_o, Tn, cout, es, 1);
    ch = cout;
  }
  s->state_bytes = P.off;  // everything up to here is zeroed by reset (a superset of the state proper)
  ch = (size_t)c.num_filters << c.n_ratios;
  Tn = T2;
  for (int i = 0; i < c.n_ratios; ++i) {
    const size_t cout = ch / 2;
    Tn *= c.ratios[i];
    const size_t zp = s->sea.stage[i].z.pitch;
    s->sea.stage[i].zf = tcm ? (float*)at(P.take(rows * zp * cout * 4)) : nullptr;
    s->sea.stage[i].h = buf(0, Tn, cout / c.compress, 4, 1);  // fp32 mode: fp32; tensor-core mode: bf16 (unfused blocks)
    ch = cout;
  }
  s->S = (float*)at(P.take(rows * n * C * 4));
  s->E = (float*)at(P.take(rows * n * C * 4));
  s->X = (float*)at(P.take(rows * T2 * C * 4));
  s->tr.ln = at(P.take(rows * T2 * C * 4));
  s->tr.qkv = (float*)at(P.take(rows * T2 * 3 * C * 4));
  s->tr.att = at(P.take(rows * T2 * C * 4));
  s->tr.hid = at(P.take(rows * T2 * FF * 4));
  s->slab_bytes = P.off;
}

// n <= max_n frames of every row: codes [rows][n_q][code_T], frames [0, n) -> wav [rows][wav_pitch], samples [0, n*hop)
int stream_step(sopro_mimi_stream* s, const int32_t* codes, int n, int code_T, float* wav, long long wav_pitch, cudaStream_t st) {
  sopro_mimi* m = s->m;
  const sopro_mimi_config_t& c = m->cfg;
  const int C = c.hidden, T2 = 2 * n, B = s->rows;
  const float* Wd = m->dev;
  const bool tcm = s->precision == SOPRO_MIMI_BF16_TC;
  const int pos0 = (int)(2 * s->frames);
  int rc = ensure_rope(m, std::max(4096, 2 * (pos0 + T2)), st);
  if (rc) return rc;
  // ---- RVQ + projection + upsample; each row's last frame is the next step's upsampler context
  rvq_gather_kernel<<<dim3(n, B), 256, 0, st>>>(codes, Wd + m->embed, s->S, c.n_q, n, code_T, c.codebook_dim, c.vocab, c.n_sem,
                                                m->bad_code);
  CK(cudaGetLastError());
  if ((rc = gemm_f32({s->S, n, 0, B, 0}, C, 1, Wd + m->rvq_w, nullptr, C, C, EPI_NONE, nullptr, nullptr, s->E, 0, st))) return rc;
  upsample_kernel<<<dim3(T2, B), 256, 0, st>>>(s->E, Wd + m->up_w, s->X, n, C, s->up_prev);
  CK(cudaGetLastError());
  CK(cudaMemcpy2DAsync(s->up_prev, (size_t)C * 4, s->E + (size_t)(n - 1) * C, (size_t)n * C * 4, (size_t)C * 4, B,
                       cudaMemcpyDeviceToDevice, st));
  // ---- transformer: K/V of the new positions go to each row's rings, queries attend over them
  const KVRing ring{s->kring, s->vring, s->R, pos0};
  if ((rc = run_layers(c, m->layers, tcm, Wd, m->dev_h, m->rope, m->rope_T2, s->X, B, T2, s->tr, &ring, st))) return rc;
  // ---- SEANet decoder over [context | chunk] buffers, then every buffer's last context rows move to its front.  fp32
  //      mode: the residual stream goes behind conv0's context rows here (tensor-core mode: its bf16 cast does)
  if (!tcm)
    CK(cudaMemcpy2DAsync(s->sea.in.rows<float>(C), (size_t)s->sea.in.pitch * C * 4, s->X, (size_t)T2 * C * 4, (size_t)T2 * C * 4, B,
                         cudaMemcpyDeviceToDevice, st));
  TailShift ts{};
  if ((rc = tcm ? seanet_tc(m, s->X, s->sea, B, T2, &ts, wav, wav_pitch, st) : seanet_f32(m, s->sea, B, T2, &ts, wav, wav_pitch, st)))
    return rc;
  tail_shift_kernel<<<dim3(ts.n, B), 256, 16384, st>>>(ts);
  CK(cudaGetLastError());
  s->frames += n;
  return SOPRO_OK;
}
}  // namespace

extern "C" {

int sopro_mimi_stream_create_rows(sopro_mimi_t* m, int max_chunk_frames, int rows, sopro_mimi_stream_t** out) {
  if (!m || !out) return fail(SOPRO_ERR_INVALID, "null argument");
  *out = nullptr;
  if (max_chunk_frames < 1 || max_chunk_frames > 256) return fail(SOPRO_ERR_INVALID, "max_chunk_frames must be in [1, 256]");
  if (rows < 1 || rows > 65535) return fail(SOPRO_ERR_INVALID, "rows must be in [1, 65535]");
  CK(cudaSetDevice(m->device));
  sopro_mimi_stream* s = new sopro_mimi_stream();
  s->m = m;
  s->max_n = max_chunk_frames;
  s->rows = rows;
  s->precision = m->precision;
  s->R = (m->cfg.window + 2 * max_chunk_frames + 7) / 8 * 8;
  stream_layout(s, nullptr);
  if ((size_t)(m->cfg.kernel - 1) * m->cfg.hidden * 4 > 16384) {
    delete s;
    return fail(SOPRO_ERR_UNSUPPORTED, "conv context rows exceed the tail-shift staging buffer");
  }
  cudaError_t e = cudaMalloc(&s->slab, s->slab_bytes);
  if (e != cudaSuccess) {
    const size_t mb = s->slab_bytes >> 20;
    delete s;
    return fail(SOPRO_ERR_CUDA, "stream state %zu MB: %s", mb, cudaGetErrorString(e));
  }
  stream_layout(s, s->slab);
  e = cudaMemset(s->slab, 0, s->state_bytes);
  if (e != cudaSuccess) {
    cudaFree(s->slab);
    delete s;
    return fail(SOPRO_ERR_CUDA, "stream state init: %s", cudaGetErrorString(e));
  }
  *out = s;
  return SOPRO_OK;
}

int sopro_mimi_stream_create(sopro_mimi_t* m, int max_chunk_frames, sopro_mimi_stream_t** out) {
  return sopro_mimi_stream_create_rows(m, max_chunk_frames, 1, out);
}

int sopro_mimi_stream_destroy(sopro_mimi_stream_t* s) {
  if (!s) return SOPRO_OK;
  cudaSetDevice(s->m->device);
  cudaFree(s->slab);
  cudaFree(s->codes_dev);
  delete s;
  return SOPRO_OK;
}

int sopro_mimi_stream_reset(sopro_mimi_stream_t* s, void* stream) {
  if (!s) return fail(SOPRO_ERR_INVALID, "null argument");
  CK(cudaSetDevice(s->m->device));
  if (s->precision != s->m->precision) {  // the buffers are laid out per arithmetic mode
    s->precision = s->m->precision;
    size_t old = s->slab_bytes;
    stream_layout(s, nullptr);
    if (s->slab_bytes > old) {
      CK(cudaStreamSynchronize(reinterpret_cast<cudaStream_t>(stream)));
      cudaFree(s->slab);
      s->slab = nullptr;
      CK(cudaMalloc(&s->slab, s->slab_bytes));
    }
    stream_layout(s, s->slab);
  }
  CK(cudaMemsetAsync(s->slab, 0, s->state_bytes, reinterpret_cast<cudaStream_t>(stream)));
  s->frames = 0;
  return SOPRO_OK;
}

int64_t sopro_mimi_stream_frames(const sopro_mimi_stream_t* s) { return s ? s->frames : -1; }

int64_t sopro_mimi_stream_rows(const sopro_mimi_stream_t* s) { return s ? s->rows : -1; }

int64_t sopro_mimi_stream_bytes(const sopro_mimi_stream_t* s) { return s ? (int64_t)s->slab_bytes : -1; }

int sopro_mimi_decode_step(sopro_mimi_stream_t* s, const int32_t* codes, int n, float* wav, void* stream) {
  if (!s || !codes || !wav) return fail(SOPRO_ERR_INVALID, "null argument");
  if (n < 1) return fail(SOPRO_ERR_INVALID, "n must be >= 1");
  if (s->precision != s->m->precision)
    return fail(SOPRO_ERR_STATE, "the decoder's precision changed since this stream started: call sopro_mimi_stream_reset");
  if (2 * (s->frames + n) > 0x3fffffffLL) return fail(SOPRO_ERR_INVALID, "stream too long");
  const int64_t hop = sopro_mimi_samples_per_frame(s->m);
  if ((long long)n * hop > 0x7fffffffLL) return fail(SOPRO_ERR_INVALID, "n too large for one call");
  if (s->precision == SOPRO_MIMI_BF16_TC) {
    const int rc = check_tc_geometry(s->m);
    if (rc) return rc;
  }
  CK(cudaSetDevice(s->m->device));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  for (int done = 0; done < n; done += s->max_n) {  // codes are [rows][n_q][n]: a sub-chunk starts at column `done`
    const int k = std::min(s->max_n, n - done);
    const int rc = stream_step(s, codes + done, k, n, wav + (size_t)done * hop, (long long)n * hop, st);
    if (rc) return rc;
  }
  return SOPRO_OK;
}

int sopro_mimi_decode_step_host(sopro_mimi_stream_t* s, const int32_t* codes_host, int n, float* wav_host, void* stream) {
  if (!s || !codes_host || !wav_host) return fail(SOPRO_ERR_INVALID, "null argument");
  if (n < 1 || n > 65536) return fail(SOPRO_ERR_INVALID, "n must be in [1, 65536]");
  const sopro_mimi_config_t& c = s->m->cfg;
  for (size_t i = 0; i < (size_t)s->rows * n * c.n_q; ++i)
    if (codes_host[i] < 0 || codes_host[i] >= c.vocab)
      return fail(SOPRO_ERR_INVALID, "code %d at flat index %zu is outside [0, %d)", codes_host[i], i, c.vocab);
  CK(cudaSetDevice(s->m->device));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t nc = (size_t)s->rows * n * c.n_q, nw = (size_t)s->rows * n * (size_t)sopro_mimi_samples_per_frame(s->m);
  cudaFree(s->codes_dev);
  s->codes_dev = nullptr;
  CK(cudaMalloc(&s->codes_dev, nc * 4 + nw * 4));
  s->wav_dev = reinterpret_cast<float*>(s->codes_dev + nc);
  CK(cudaMemcpyAsync(s->codes_dev, codes_host, nc * 4, cudaMemcpyHostToDevice, st));
  const int rc = sopro_mimi_decode_step(s, s->codes_dev, n, s->wav_dev, stream);
  if (rc) return rc;
  CK(cudaMemcpyAsync(wav_host, s->wav_dev, nw * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return SOPRO_OK;
}

}  // extern "C"

extern "C" {

int sopro_mimi_check(sopro_mimi_t* m, void* stream) {
  if (!m) return fail(SOPRO_ERR_INVALID, "null argument");
  CK(cudaSetDevice(m->device));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int flag = 0;
  CK(cudaMemcpyAsync(&flag, m->bad_code, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaMemsetAsync(m->bad_code, 0, 4, st));
  CK(cudaStreamSynchronize(st));
  if (flag) return fail(SOPRO_ERR_INVALID, "a decode since the last check read a code outside [0, %d) (clamped)", m->cfg.vocab);
  return SOPRO_OK;
}

int sopro_mimi_set_graphs(sopro_mimi_t* m, int enabled) {
  if (!m) return fail(SOPRO_ERR_INVALID, "null argument");
  m->graphs = enabled != 0;
  return SOPRO_OK;
}

int sopro_debug_tc_gemm_pitched(const void* X, int B, int M, int ctx, int64_t a_pitch, int cin, int taps, const void* W, int N,
                                const float* bias, int bias_mod, int epi, const float* R, int64_t r_pitch, const float* scale,
                                float* out_f32, void* out_bf16, int64_t c_pitch, int out_elu, void* stream) {
  const bool res = epi == tc::EPI_RES || epi == tc::EPI_RES_SCALE;
  if (!X || !W || (!out_f32 && !out_bf16) || (res && !R) || (epi == tc::EPI_RES_SCALE && !scale))
    return fail(SOPRO_ERR_INVALID, "null argument");
  auto misaligned = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) != 0; };
  if (misaligned(X) || misaligned(W) || misaligned(bias) || misaligned(R) || misaligned(scale) || misaligned(out_f32) ||
      misaligned(out_bf16))
    return fail(SOPRO_ERR_INVALID, "tc gemm: every pointer must be 16-byte aligned");
  if (B < 1 || B > 65535 || M < 1 || taps < 1 || ctx < 0 || ctx > taps - 1 || a_pitch < (int64_t)ctx + M || c_pitch < M ||
      (res && r_pitch < M) || epi < tc::EPI_NONE || epi > tc::EPI_RES || (bias && (bias_mod < 4 || bias_mod % 4 || bias_mod > N)) ||
      !tc::supported(N, taps * cin, cin))
    return fail(SOPRO_ERR_INVALID, "tc gemm: unsupported shape (B=%d M=%d ctx=%d a_pitch=%lld cin=%d taps=%d N=%d c_pitch=%lld)", B, M,
                ctx, (long long)a_pitch, cin, taps, N, (long long)c_pitch);
  // the decoder's own launcher: pad = taps - 1 - ctx, dil = 1 and the item strides come from the same code
  const Operand a{X, M, ctx, B, a_pitch};
  return gemm_tc(a, cin, taps, static_cast<const __nv_bfloat16*>(W), bias, N, bias ? bias_mod : N, epi, R, scale, out_f32,
                 static_cast<__nv_bfloat16*>(out_bf16), out_elu, reinterpret_cast<cudaStream_t>(stream), c_pitch, res ? r_pitch : 0);
}

// the packed one-shot geometry (no context rows, items back to back) of sopro_debug_tc_gemm_pitched; dil and pad stay in
// the signature for its callers, and only what the decoder issues (dil = 1, pad = taps - 1) is taken
int sopro_debug_tc_gemm(const void* X, int B, int64_t rows, int cin, int taps, int dil, int pad, const void* W, int N,
                        const float* bias, int bias_mod, int epi, const float* R, const float* scale, float* out_f32,
                        void* out_bf16, int out_elu, void* stream) {
  if (rows < 1 || rows > 0x7fffffffLL || dil != 1 || pad != taps - 1)
    return fail(SOPRO_ERR_INVALID, "tc gemm: rows=%lld dil=%d pad=%d (the decoder issues dil = 1, pad = taps - 1)", (long long)rows, dil,
                pad);
  return sopro_debug_tc_gemm_pitched(X, B, (int)rows, 0, rows, cin, taps, W, N, bias, bias_mod > 0 ? bias_mod : N, epi, R, rows, scale,
                                     out_f32, out_bf16, rows, out_elu, stream);
}

int sopro_debug_tc_attn(const void* q, const void* k, const void* vt, void* out, int B, int T2, int64_t T2p, int C, int H, int window,
                        void* stream) {
  if (!q || !k || !vt || !out) return fail(SOPRO_ERR_INVALID, "null argument");
  if (B < 1 || B > 65535 || T2 < 1 || T2p < T2 || T2p % 8 != 0 || !tc::attn_supported(C, H, window))
    return fail(SOPRO_ERR_INVALID, "tc attention: unsupported shape (B=%d T2=%d T2p=%lld C=%d H=%d window=%d)", B, T2, (long long)T2p,
                C, H, window);
  cudaError_t e = tc::launch_attn(q, k, vt, static_cast<__nv_bfloat16*>(out), B, T2, T2p, C, H, window,
                                  reinterpret_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return fail(SOPRO_ERR_CUDA, "tensor-core attention launch: %s", cudaGetErrorString(e));
  return SOPRO_OK;
}

int sopro_debug_tc_resblock_pitched(const void* X, const void* W1, const void* W2, const float* bias1, const float* bias2,
                                    const float* Z, float* out_f32, void* out_bf16, int B, int M, int ctx, int64_t a_pitch, int64_t z_pitch,
                                    int64_t o_pitch, int hid, int taps, int out_elu, void* stream) {
  if (!X || !W1 || !W2 || !bias1 || !bias2 || !Z || (!out_f32 && !out_bf16)) return fail(SOPRO_ERR_INVALID, "null argument");
  if (B < 1 || B > 65535 || M < 1 || taps < 1 || ctx < 0 || ctx > taps - 1 || (long long)M + ctx > 0x7fffffffLL ||
      a_pitch < (int64_t)M + ctx || z_pitch < M || o_pitch < M || !tc::resblock_supported(hid, 2 * hid) || (2 * hid * taps) % 64 != 0)
    return fail(SOPRO_ERR_INVALID, "fused ResnetBlock: unsupported shape (B=%d M=%d ctx=%d hid=%d taps=%d)", B, M, ctx, hid, taps);
  // the operand geometry of seanet_tc: ctx context rows in front of the M rows, the causal zero pad covers the rest;
  // item b of X, Z and the outputs a_pitch, z_pitch and o_pitch rows after item b - 1 (the stream's buffers)
  tc::ResOp ro{};
  ro.a_pitch = a_pitch;
  ro.z_bs = z_pitch * 2 * hid;
  ro.o_bs = o_pitch * 2 * hid;
  ro.bias1 = bias1;
  ro.bias2 = bias2;
  ro.Z = Z;
  ro.out_f32 = out_f32;
  ro.out_bf16 = static_cast<__nv_bfloat16*>(out_bf16);
  ro.M = M;
  ro.Min = M + ctx;
  ro.taps = taps;
  ro.pad = taps - 1 - ctx;
  ro.out_elu = out_elu;
  cudaError_t e = tc::launch_resblock(X, W1, W2, hid, ro, B, reinterpret_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return fail(SOPRO_ERR_CUDA, "fused ResnetBlock launch: %s", cudaGetErrorString(e));
  return SOPRO_OK;
}

// packed items: X [B][ctx + M][2*hid], Z and the outputs [B][M][2*hid]
int sopro_debug_tc_resblock(const void* X, const void* W1, const void* W2, const float* bias1, const float* bias2, const float* Z,
                            float* out_f32, void* out_bf16, int B, int M, int ctx, int hid, int taps, int out_elu, void* stream) {
  return sopro_debug_tc_resblock_pitched(X, W1, W2, bias1, bias2, Z, out_f32, out_bf16, B, M, ctx, (int64_t)M + ctx, M, M, hid, taps,
                                         out_elu, stream);
}

int sopro_debug_rope_pack(const float* qkv, const float* table, int tab_T2, void* qh, void* kh, void* vt, int B, int T2, int C, int H,
                          void* stream) {
  if (!qkv || !table || !qh || !kh || !vt) return fail(SOPRO_ERR_INVALID, "null argument");
  const size_t pack_bytes = (size_t)32 * (C + 2) * 2;
  if (B < 1 || B > 65535 || T2 < 1 || tab_T2 < T2 || H < 1 || C != H * tc::kAttnDh || pack_bytes > 48 * 1024)
    return fail(SOPRO_ERR_INVALID, "rope pack: unsupported shape (B=%d T2=%d tab_T2=%d C=%d H=%d)", B, T2, tab_T2, C, H);
  const long long T2p = (T2 + 7) / 8 * 8;  // as run_layers pitches v^T
  rope_pack_kernel<tc::kAttnDh><<<dim3((T2 + 31) / 32, B), 256, pack_bytes, reinterpret_cast<cudaStream_t>(stream)>>>(
      qkv, table, static_cast<__nv_bfloat16*>(qh), static_cast<__nv_bfloat16*>(kh), static_cast<__nv_bfloat16*>(vt), T2, T2p, tab_T2, C, H);
  CK(cudaGetLastError());
  return SOPRO_OK;
}

int sopro_debug_mimi_gemm(const float* A, const float* W, const float* bias, const float* R, const float* scale, float* out, int B, int M,
                          int N, int K, int Min, int Cin, int taps, int dil, int pad, int ldc, int bias_mod, int epi, int a_elu,
                          int64_t a_bs, int64_t c_bs, int64_t r_bs, void* stream) {
  if (!A || !W || !out) return fail(SOPRO_ERR_INVALID, "null argument");
  if (B < 1 || B > 65535 || M < 1 || N < 1 || Cin < 4 || Cin % 4 || taps < 1 || dil < 1 || pad < 0 || K != taps * Cin || K % 16 ||
      Min < M || ldc < N || a_bs % 4 || a_bs < 0 || c_bs < 0 || r_bs < 0 || epi < EPI_NONE || epi > EPI_RES ||
      (bias && bias_mod < 1) || (epi >= EPI_RES_SCALE && !R) || (epi == EPI_RES_SCALE && !scale))
    return fail(SOPRO_ERR_INVALID, "igemm: unsupported shape (B=%d M=%d N=%d K=%d Min=%d Cin=%d taps=%d ldc=%d epi=%d)", B, M, N, K, Min,
                Cin, taps, ldc, epi);
  GemmOp g{};
  g.A = A; g.W = W; g.bias = bias; g.R = R; g.scale = scale; g.C = out;
  g.a_bs = a_bs; g.c_bs = c_bs; g.r_bs = r_bs;
  g.M = M; g.N = N; g.K = K; g.Min = Min; g.Cin = Cin; g.taps = taps; g.dil = dil; g.pad = pad; g.ldc = ldc;
  g.bias_mod = bias ? bias_mod : 1; g.epi = epi; g.a_elu = a_elu ? 1 : 0;
  return launch_gemm(g, B, reinterpret_cast<cudaStream_t>(stream));
}

int sopro_debug_mimi_rvq_gather(const int32_t* codes, const float* embed, float* S, int B, int Q, int T, int code_T, int Dc, int vocab,
                                int n_sem, int32_t* bad, void* stream) {
  if (!codes || !embed || !S || !bad) return fail(SOPRO_ERR_INVALID, "null argument");
  if (B < 1 || B > 65535 || Q < 1 || T < 1 || code_T < T || Dc < 1 || vocab < 1 || n_sem < 0 || n_sem > Q)
    return fail(SOPRO_ERR_INVALID, "rvq gather: unsupported shape (B=%d Q=%d T=%d code_T=%d Dc=%d vocab=%d)", B, Q, T, code_T, Dc, vocab);
  rvq_gather_kernel<<<dim3(T, B), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(codes, embed, S, Q, T, code_T, Dc, vocab, n_sem, bad);
  CK(cudaGetLastError());
  return SOPRO_OK;
}

int sopro_debug_mimi_upsample(const float* x, const float* w, float* y, const float* prev, int B, int T, int C, void* stream) {
  if (!x || !w || !y) return fail(SOPRO_ERR_INVALID, "null argument");
  if (B < 1 || B > 65535 || T < 1 || T > 0x3fffffff || C < 1)
    return fail(SOPRO_ERR_INVALID, "upsample: unsupported shape (B=%d T=%d C=%d)", B, T, C);
  upsample_kernel<<<dim3(2 * T, B), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, w, y, T, C, prev);
  CK(cudaGetLastError());
  return SOPRO_OK;
}

int sopro_debug_mimi_layernorm(const float* x, const float* w, const float* b, void* y, int64_t rows, int C, float eps, int out_bf16,
                               void* stream) {
  if (!x || !w || !b || !y) return fail(SOPRO_ERR_INVALID, "null argument");
  if (rows < 1 || (rows + 7) / 8 > 0x7fffffffLL || C < 1) return fail(SOPRO_ERR_INVALID, "layernorm: unsupported shape (rows=%lld C=%d)", (long long)rows, C);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const unsigned grid = (unsigned)((rows + 7) / 8);  // as run_layers launches it
  if (out_bf16) layernorm_kernel<<<grid, 256, 0, st>>>(x, w, b, static_cast<__nv_bfloat16*>(y), rows, C, eps);
  else layernorm_kernel<<<grid, 256, 0, st>>>(x, w, b, static_cast<float*>(y), rows, C, eps);
  CK(cudaGetLastError());
  return SOPRO_OK;
}

int sopro_debug_mimi_attn(float* qkv, const float* table, int tab_T2, void* out, int B, int T2, int C, int H, int window, int pos0,
                          float* kring, float* vring, int R, int out_bf16, void* stream) {
  if (!qkv || !table || !out || !kring != !vring) return fail(SOPRO_ERR_INVALID, "null argument");
  const int Dh = H > 0 ? C / H : 0;
  const size_t asm_bytes = (size_t)8 * (Dh + (size_t)std::max(window, 0)) * 4;
  if (B < 1 || B > 65535 || T2 < 1 || H < 1 || C < 1 || C % H || Dh % 4 || window < 1 || pos0 < 0 || asm_bytes > 48 * 1024 ||
      (long long)pos0 + T2 > tab_T2 || (kring ? (long long)R < (long long)T2 + window - 1 : pos0 != 0))
    return fail(SOPRO_ERR_INVALID, "attention: unsupported shape (B=%d T2=%d C=%d H=%d window=%d pos0=%d R=%d tab_T2=%d)", B, T2, C, H,
                window, pos0, R, tab_T2);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int Rk = kring ? R : 1;
  // as run_layers issues them: RoPE in place (and the ring append), then the attention
  rope_kernel<<<dim3(T2, B), 256, 0, st>>>(qkv, table, T2, tab_T2, C, H, pos0, kring, vring, Rk);
  if (out_bf16)
    attn_kernel<<<dim3((T2 + 7) / 8, H, B), 256, asm_bytes, st>>>(qkv, static_cast<__nv_bfloat16*>(out), T2, C, H, window, pos0, kring, vring, Rk);
  else
    attn_kernel<<<dim3((T2 + 7) / 8, H, B), 256, asm_bytes, st>>>(qkv, static_cast<float*>(out), T2, C, H, window, pos0, kring, vring, Rk);
  CK(cudaGetLastError());
  return SOPRO_OK;
}

int sopro_debug_mimi_final_conv(const void* x, int x_bf16, const float* w, const float* bias, float* y, int B, int64_t Tn, int Cin,
                                int taps, int lo, int64_t x_bs, int64_t y_bs, void* stream) {
  if (!x || !w || !bias || !y) return fail(SOPRO_ERR_INVALID, "null argument");
  const int vec = x_bf16 ? 8 : 4;  // elements per vector load
  const size_t smem = (size_t)(taps * 256 + (size_t)taps * Cin) * 4;
  if (B < 1 || B > 65535 || Tn < 1 || Tn > 0x7fffffffLL || Cin < vec || Cin % vec || taps < 1 || taps > 8 || lo > 0 || lo < -(taps - 1) ||
      x_bs % vec || (B > 1 && (x_bs < (Tn - lo) * Cin || y_bs < Tn)) || (x_bf16 && smem > 48 * 1024))
    return fail(SOPRO_ERR_INVALID, "final conv: unsupported shape (B=%d Tn=%lld Cin=%d taps=%d lo=%d)", B, (long long)Tn, Cin, taps, lo);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (x_bf16) {  // as seanet_tc launches it
    const int per = 256 - (taps - 1);
    final_conv_h_kernel<<<dim3((unsigned)((Tn + per - 1) / per), B), 256, smem, st>>>(static_cast<const __nv_bfloat16*>(x), w, bias, y, Tn,
                                                                                      Cin, taps, lo, x_bs, y_bs);
  } else {
    final_conv_kernel<<<dim3((unsigned)((Tn + 255) / 256), B), 256, 0, st>>>(static_cast<const float*>(x), w, bias, y, Tn, Cin, taps, lo,
                                                                              x_bs, y_bs);
  }
  CK(cudaGetLastError());
  return SOPRO_OK;
}

int sopro_mimi_decode_host(sopro_mimi_t* m, const int32_t* codes_host, int B, int T, float* wav_host, void* stream) {
  if (!m || !codes_host || !wav_host) return fail(SOPRO_ERR_INVALID, "null argument");
  CK(cudaSetDevice(m->device));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (B < 1 || T < 1) return fail(SOPRO_ERR_INVALID, "B and T must be >= 1");
  const size_t nc = (size_t)B * m->cfg.n_q * T;
  const size_t nw = (size_t)B * T * sopro_mimi_samples_per_frame(m);
  for (size_t i = 0; i < nc; ++i)
    if (codes_host[i] < 0 || codes_host[i] >= m->cfg.vocab)
      return fail(SOPRO_ERR_INVALID, "code %d at flat index %zu is outside [0, %d)", codes_host[i], i, m->cfg.vocab);
  if (m->codes_cap < nc * 4 + nw * 4) {
    cudaFree(m->codes_dev);
    m->codes_dev = nullptr;
    m->codes_cap = 0;
    CK(cudaMalloc(&m->codes_dev, nc * 4 + nw * 4));
    m->codes_cap = nc * 4 + nw * 4;
  }
  float* wav_dev = reinterpret_cast<float*>(m->codes_dev + nc);
  CK(cudaMemcpyAsync(m->codes_dev, codes_host, nc * 4, cudaMemcpyHostToDevice, st));
  int rc = sopro_mimi_decode(m, m->codes_dev, B, T, wav_dev, stream);
  if (rc) return rc;
  CK(cudaMemcpyAsync(wav_host, wav_dev, nw * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return SOPRO_OK;
}

}  // extern "C"

// =====================================================================================================================
// ENCODE: waveform -> codes (MimiModel.encode, modeling_mimi.py:1455-1488, 1522-1611; the reference calls it once per
// reference voice, codec/mimi.py:41-63).  fp32 throughout on the kernels above: every conv is the implicit GEMM; a conv
// of kernel 2r and stride r over [L][C] is the 2-tap stride-1 conv over the same memory read as [L/r][r*C] (L padded
// with zero rows to a multiple of r: MimiConv1d's "extra padding", :273-285; its causal left padding of r rows is the
// tap at superrow -1).
// =====================================================================================================================
namespace mimi {
// A batch of clips (sopro_mimi_encode_batch) is right-padded to one length and every kernel runs over all its rows.
// Everything in the encoder is causal, so a clip's valid prefix never reads its padding, except where a kernel below
// takes the clip's own lengths: `info` [B][NS] int, row b = (rows entering stage s for s = 0..n_ratios, the last being
// the transformer positions T2, then the frames T) of clip b.  A single clip passes info = null and B = 1.
constexpr int enc_info_cols(int n_ratios) { return n_ratios + 2; }

// first conv: wav [L] -> y [L][F], kernel k, causal (left zero pad k-1), weight [F][k].  Batch (grid.y = B): clip b's
// samples are wav + b * wav_stride, info[b][0] of them (zero past that), its rows y + b * L * F.
__global__ void enc_conv0_kernel(const float* __restrict__ wav, const float* __restrict__ w, const float* __restrict__ bias,
                                 float* __restrict__ y, long long L, int F, int k, long long wav_stride, const int* __restrict__ info,
                                 int NS) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L * F) return;
  const int b = blockIdx.y;
  const long long n = info ? info[b * NS] : L;
  wav += (long long)b * wav_stride;
  const long long t = i / F;
  const int c = (int)(i - t * F);
  float acc = __ldg(bias + c);
  for (int j = 0; j < k; ++j) {
    const long long ti = t + j - (k - 1);
    if (ti >= 0 && ti < n) acc = fmaf(__ldg(w + c * k + j), __ldg(wav + ti), acc);
  }
  y[(long long)b * L * F + i] = acc;
}

// MimiConv1d's extra padding of clip b (grid.y) before the stride-r conv of stage s: rows [L, roundup(L, r)) of its
// [stride rows][ch] block are zeroed, L = info[b][s]
__global__ void enc_zero_tail_kernel(float* __restrict__ x, long long stride, int ch, int r, const int* __restrict__ info, int NS, int s) {
  const int b = blockIdx.y;
  const long long L = info[b * NS + s], Lp = (L + r - 1) / r * r;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long row = L + i / ch;
  if (row < Lp) x[(long long)b * stride * ch + row * ch + (i % ch)] = 0.f;
}

// replicate padding for the 25 -> 12.5 Hz conv: y rows [0, left) = x[0], [left, left+T) = x, [left+T, rows) = x[T-1].
// Batch (grid.y = B): clip b's x rows are x + b * T * C (T = the padded positions), its y rows y + b * rows * C, and its
// own last position info[b][NS - 2] - 1 is the one replicated.
__global__ void replicate_pad_kernel(const float* __restrict__ x, float* __restrict__ y, int T, int C, int left, int rows,
                                     const int* __restrict__ info, int NS) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)rows * C) return;
  const int b = blockIdx.y;
  const int Tb = info ? info[b * NS + NS - 2] : T;
  const int r = (int)(i / C), c = (int)(i - (long long)r * C);
  int src = r - left;
  src = src < 0 ? 0 : (src >= Tb ? Tb - 1 : src);
  y[(size_t)b * rows * C + i] = x[(size_t)b * T * C + (size_t)src * C + c];
}

// Residual nearest-neighbour search (MimiResidualVectorQuantizer.encode :1262-1280 with MimiEuclideanCodebook.quantize
// :1197-1203): one CTA per frame, the residual (Dc = 32*DPL floats) in registers, lane-sliced; a warp scans every 8th
// code vector, squared distance summed directly (the reference's cdist goes through |x|^2+|e|^2-2xe, same minimiser),
// with torch.argmin's rule: the first NaN distance wins, else the lowest index of the smallest distance, so a frame whose
// every distance is +Inf takes code 0 and every code is in [0, V) whatever the residual holds.  proj [T][2*Dc] =
// [semantic input_proj | acoustic input_proj] of the latent.
// Batch (grid.y = B): clip b's proj rows are proj + b * T * 2Dc and its codes codes + b * n_q * T; frames at or past
// its own info[b][NS - 1] are skipped.
template <int DPL>
__global__ void __launch_bounds__(256) rvq_encode_kernel(const float* __restrict__ proj, const float* __restrict__ embed,
                                                         int* __restrict__ codes, int T, int n_q, int n_sem, int V,
                                                         const int* __restrict__ info, int NS) {
  constexpr int Dc = 32 * DPL;
  __shared__ float best_d[8];
  __shared__ int best_i[8];
  __shared__ int winner;
  const int t = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, b = blockIdx.y;
  if (info && t >= info[b * NS + NS - 1]) return;  // uniform across the CTA
  proj += (size_t)b * T * 2 * Dc;
  codes += (size_t)b * n_q * T;
  float r[DPL];
  for (int q = 0; q < n_q; ++q) {
    if (q == 0 || q == n_sem) {
      const float* p = proj + (size_t)t * 2 * Dc + (q == 0 ? 0 : Dc) + lane * DPL;
#pragma unroll
      for (int i = 0; i < DPL; ++i) r[i] = p[i];
    }
    const float* E = embed + (size_t)q * V * Dc;
    float bd = INFINITY;
    int bi = warp;  // a warp none of whose distances is below +Inf keeps its first index (>= V only when V < 8)
#pragma unroll 4  // four code vectors' loads in flight, as the compiler unrolls the loop without the NaN select
    for (int k = warp; k < V; k += 8) {
      const float* e = E + (size_t)k * Dc + lane * DPL;
      float acc = 0.f;
#pragma unroll
      for (int i = 0; i < DPL; i += 4) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(e + i));
        float d = r[i] - v.x;
        acc = fmaf(d, d, acc);
        d = r[i + 1] - v.y;
        acc = fmaf(d, d, acc);
        d = r[i + 2] - v.z;
        acc = fmaf(d, d, acc);
        d = r[i + 3] - v.w;
        acc = fmaf(d, d, acc);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      acc = acc != acc ? -1.f : acc;  // a NaN distance ranks below every real one (>= 0)
      if (acc < bd) {  // k ascends within a warp: strict < keeps the lowest index (the first NaN)
        bd = acc;
        bi = k;
      }
    }
    if (lane == 0) {
      best_d[warp] = bd;
      best_i[warp] = bi;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      float d = best_d[0];
      int ix = best_i[0];
      for (int w = 1; w < 8; ++w)
        if (best_d[w] < d || (best_d[w] == d && best_i[w] < ix)) {
          d = best_d[w];
          ix = best_i[w];
        }
      winner = ix;
      codes[(size_t)q * T + t] = ix;
    }
    __syncthreads();
    const float* e = E + (size_t)winner * Dc + lane * DPL;
#pragma unroll
    for (int i = 0; i < DPL; ++i) r[i] -= __ldg(e + i);
    // (best_d / best_i / winner are rewritten only after the next __syncthreads pair)
  }
}
}  // namespace mimi

struct sopro_mimi_encoder {
  int device = 0;
  sopro_mimi_config_t cfg{};
  float* dev = nullptr;
  size_t c0w = 0, c0b = 0, lw = 0, lb = 0, down_w = 0, inproj = 0, embed = 0;
  struct Stage {
    size_t r1w, r1b, r2w, r2b, dw, db;
    int ratio, cin;
  };
  std::vector<Stage> stages;
  std::vector<sopro_mimi::Layer> layers;  // fp32 offsets only
  float* rope = nullptr;
  int rope_T2 = 0;
  float* ws = nullptr;
  size_t ws_bytes = 0;
  float* wav_dev = nullptr;   // staging of the *_host entry point
  int* codes_dev = nullptr;
  float* lat_dev = nullptr;
  size_t wav_cap = 0, codes_cap = 0, lat_cap = 0;
  int* info_dev = nullptr;    // the per-clip lengths of a batch (see enc_info_cols)
  size_t info_cap = 0;
};

namespace {
constexpr long long kEncMaxSamples = 24000LL * 600;  // ten minutes of audio; a reference voice is seconds

struct EncPlan {
  long long len[SOPRO_MIMI_MAX_RATIOS + 1];   // rows entering stage s (len[0] = samples), len[n_ratios] = transformer positions
  long long padded[SOPRO_MIMI_MAX_RATIOS];    // len[s] rounded up to the stage's stride
  long long T;                                // frames
  size_t buf, xsz, need;
};

EncPlan enc_plan(const sopro_mimi_config_t& c, long long n) {
  EncPlan p{};
  p.len[0] = n;
  size_t widest = 0;
  int ch = c.num_filters;
  for (int s = 0; s < c.n_ratios; ++s) {
    const int r = c.ratios[c.n_ratios - 1 - s];
    p.padded[s] = (p.len[s] + r - 1) / r * r;
    p.len[s + 1] = p.padded[s] / r;
    widest = std::max(widest, (size_t)p.padded[s] * ch);
    ch *= 2;
  }
  const long long T2 = p.len[c.n_ratios];
  p.T = (T2 + 1) / 2;
  widest = std::max(widest, (size_t)T2 * ch);                                   // last conv input [T2][16F]
  widest = std::max(widest, (size_t)T2 * (size_t)std::max(3 * c.hidden, c.ffn));  // QKV / MLP hidden
  widest = std::max(widest, (size_t)(2 * p.T + 2) * c.hidden);                  // replicate-padded downsample input
  p.buf = (widest + 63) / 64 * 64;
  p.xsz = ((size_t)T2 * c.hidden + 63) / 64 * 64;
  p.need = (3 * p.buf + 2 * p.xsz) * 4;
  return p;
}

// The encode sequence over B clips laid out by plan P (a clip alone: P of its length, B = 1, info = null; a batch: P
// of the padded length, whose every stage length is then a multiple of its stride, and info the clips' own lengths).
// Only enqueues kernels, after the RoPE table and the workspace have been sized.
int encode_run(sopro_mimi_encoder* e, const EncPlan& P, int B, const float* wav, long long wav_stride, const int* info,
               int32_t* codes, float* latent, cudaStream_t st) {
  const sopro_mimi_config_t& c = e->cfg;
  const int C = c.hidden, Dc = c.codebook_dim, NS = enc_info_cols(c.n_ratios);
  const int T2 = (int)P.len[c.n_ratios], T = (int)P.T;
  int rc;
  float* b0 = e->ws;
  float* b1 = b0 + B * P.buf;
  float* b2 = b1 + B * P.buf;
  float* x = b2 + B * P.buf;
  float* ln = x + B * P.xsz;
  const float* Wd = e->dev;
  // ---- SEANet encoder
  float* cur = b0;   // stage input [len][ch]
  float* hid = b1;   // resblock hidden [len][ch/2]
  float* nxt = b2;
  {
    const long long tot = P.len[0] * c.num_filters;
    enc_conv0_kernel<<<dim3((unsigned)((tot + 255) / 256), B), 256, 0, st>>>(wav, Wd + e->c0w, Wd + e->c0b, cur, P.len[0],
                                                                           c.num_filters, c.kernel, wav_stride, info, NS);
    CK(cudaGetLastError());
  }
  int ch = c.num_filters;
  for (int s = 0; s < c.n_ratios; ++s) {
    const sopro_mimi_encoder::Stage& S = e->stages[s];
    const long long Ls = P.len[s], Lp = P.padded[s];
    const int r = S.ratio;
    // ResnetBlock (:412-451): x + conv1(ELU(conv3(ELU(x))))
    if ((rc = gemm_f32({cur, Ls, 0, B}, ch, c.res_kernel, Wd + S.r1w, Wd + S.r1b, ch / 2, ch / 2, EPI_NONE, nullptr, nullptr, hid, 1, st)))
      return rc;
    if ((rc = gemm_f32({hid, Ls, 0, B}, ch / 2, 1, Wd + S.r2w, Wd + S.r2b, ch, ch, EPI_RES, cur, nullptr, cur, 1, st))) return rc;
    // ELU + conv kernel 2r stride r: zero rows up to a multiple of r, then 2 taps over [Lp/r][r*ch]
    if (info && r > 1) {
      enc_zero_tail_kernel<<<dim3((unsigned)(((r - 1) * ch + 255) / 256), B), 256, 0, st>>>(cur, Lp, ch, r, info, NS, s);
      CK(cudaGetLastError());
    } else if (!info && Lp > Ls) {
      CK(cudaMemsetAsync(cur + (size_t)Ls * ch, 0, (size_t)(Lp - Ls) * ch * 4, st));
    }
    if ((rc = gemm_f32({cur, Lp / r, 0, B}, r * ch, 2, Wd + S.dw, Wd + S.db, 2 * ch, 2 * ch, EPI_NONE, nullptr, nullptr, nxt, 1, st)))
      return rc;
    std::swap(cur, nxt);
    ch *= 2;
  }
  // ELU + conv k3 -> residual stream x [T2][C]
  if ((rc = gemm_f32({cur, T2, 0, B}, ch, c.last_kernel, Wd + e->lw, Wd + e->lb, C, C, EPI_NONE, nullptr, nullptr, x, 1, st))) return rc;
  // ---- encoder transformer (MimiTransformerLayer.forward :966-993), fp32 path of the decoder
  LayerBufs lb{};
  lb.ln = ln;
  lb.qkv = b0;
  lb.att = b1;
  lb.hid = b0;
  if ((rc = run_layers(c, e->layers, false, Wd, nullptr, e->rope, e->rope_T2, x, B, T2, lb, nullptr, st))) return rc;
  // ---- 25 -> 12.5 Hz: kernel 4, stride 2, no bias, replicate padding (2 rows left, 0 or 1 right)
  {
    const int rows = 2 * T + 2;
    const long long tot = (long long)rows * C;
    replicate_pad_kernel<<<dim3((unsigned)((tot + 255) / 256), B), 256, 0, st>>>(x, b0, T2, C, 2, rows, info, NS);
    CK(cudaGetLastError());
    float* lat = latent ? latent : b1;
    // 2 taps over the T + 1 row pairs [rows/2][2C]: the first pair (the left padding) is the context of output row 0
    if ((rc = gemm_f32({b0, T, 1, B}, 2 * C, 2, Wd + e->down_w, nullptr, C, C, EPI_NONE, nullptr, nullptr, lat, 0, st))) return rc;
    // ---- quantizer: both input projections in one GEMM, then the residual search
    if ((rc = gemm_f32({lat, T, 0, B}, C, 1, Wd + e->inproj, nullptr, 2 * Dc, 2 * Dc, EPI_NONE, nullptr, nullptr, b2, 0, st))) return rc;
    rvq_encode_kernel<8><<<dim3(T, B), 256, 0, st>>>(b2, Wd + e->embed, codes, T, c.n_q, c.n_sem, c.vocab, info, NS);
    CK(cudaGetLastError());
  }
  return SOPRO_OK;
}

// the RoPE table for T2 positions and a workspace of `need` bytes
int encode_prepare(sopro_mimi_encoder* e, int T2, size_t need, cudaStream_t st) {
  int rc;
  if (e->rope_T2 < T2 && (rc = make_rope(e->cfg, std::max(T2, 256), &e->rope, &e->rope_T2, st))) return rc;
  if (e->ws_bytes < need) {
    cudaFree(e->ws);
    e->ws = nullptr;
    e->ws_bytes = 0;
    cudaError_t ae = cudaMalloc(&e->ws, need);
    if (ae != cudaSuccess) return fail(SOPRO_ERR_CUDA, "Mimi encoder workspace %zu MB: %s", need >> 20, cudaGetErrorString(ae));
    e->ws_bytes = need;
  }
  return SOPRO_OK;
}
}  // namespace

extern "C" {

int sopro_mimi_encoder_create(const sopro_mimi_config_t* cfg, const sopro_mimi_encoder_weights_t* w, int device,
                              sopro_mimi_encoder_t** out) {
  if (!cfg || !w || !out) return fail(SOPRO_ERR_INVALID, "null argument");
  *out = nullptr;
  const int rc = open_device(device, "the Mimi encoder");
  if (rc != SOPRO_OK) return rc;
  const int C = cfg->hidden, Dc = cfg->codebook_dim, Q = cfg->n_q, V = cfg->vocab, NL = cfg->n_layers, FF = cfg->ffn, F0 = cfg->num_filters;
  if (C % 64 || Dc != 256 || C != 2 * Dc || NL < 1 || NL > SOPRO_MIMI_MAX_LAYERS || cfg->n_ratios < 1 || cfg->n_ratios > SOPRO_MIMI_MAX_RATIOS ||
      cfg->n_heads < 1 || C % cfg->n_heads || (C / cfg->n_heads) % 4 || FF % 16 || F0 % 16 || cfg->compress != 2 || Q < 1 || cfg->n_sem < 1 ||
      cfg->n_sem > Q || cfg->kernel < 1 || cfg->kernel > 16)
    return fail(SOPRO_ERR_INVALID, "unsupported Mimi encoder geometry (hidden=%d codebook_dim=%d)", C, Dc);
  sopro_mimi_encoder* e = new sopro_mimi_encoder();
  e->device = device;
  e->cfg = *cfg;
  DevArena A;
  // conv weights [Cout][Cin][k] -> [Cout][(tap, ci)]; a strided conv's taps j = j2*r + rr are ordered (j2, rr, ci), which
  // is the same formula with k = 2r
  auto repack_conv = [&](const float* src, int cout, int cin, int k) {
    std::vector<float> r((size_t)cout * k * cin);
    for (int co = 0; co < cout; ++co)
      for (int ci = 0; ci < cin; ++ci)
        for (int j = 0; j < k; ++j) r[((size_t)co * k + j) * cin + ci] = src[((size_t)co * cin + ci) * k + j];
    return A.add(r.data(), r.size());
  };
  e->c0w = A.add(w->conv0_w, (size_t)F0 * cfg->kernel);
  e->c0b = A.add(w->conv0_b, F0);
  int ch = F0;
  for (int s = 0; s < cfg->n_ratios; ++s) {
    const sopro_mimi_enc_stage_weights_t& S = w->stage[s];
    sopro_mimi_encoder::Stage d;
    d.ratio = cfg->ratios[cfg->n_ratios - 1 - s];
    d.cin = ch;
    d.r1w = repack_conv(S.res1_w, ch / 2, ch, cfg->res_kernel);
    d.r1b = A.add(S.res1_b, ch / 2);
    d.r2w = repack_conv(S.res2_w, ch, ch / 2, 1);
    d.r2b = A.add(S.res2_b, ch);
    d.dw = repack_conv(S.down_w, 2 * ch, ch, 2 * d.ratio);
    d.db = A.add(S.down_b, 2 * ch);
    e->stages.push_back(d);
    ch *= 2;
  }
  e->lw = repack_conv(w->last_w, C, ch, cfg->last_kernel);
  e->lb = A.add(w->last_b, C);
  for (int l = 0; l < NL; ++l) e->layers.push_back(pack_layer(w->layer[l], C, FF, A, nullptr));
  e->down_w = repack_conv(w->downsample_w, C, C, 4);
  {  // [2*Dc][C]: semantic input_proj rows, then acoustic
    std::vector<float> cat((size_t)2 * Dc * C);
    memcpy(cat.data(), w->sem_in_proj, (size_t)Dc * C * 4);
    memcpy(cat.data() + (size_t)Dc * C, w->ac_in_proj, (size_t)Dc * C * 4);
    e->inproj = A.add(cat.data(), cat.size());
  }
  e->embed = A.add(w->embed, (size_t)Q * V * Dc);
  cudaError_t err = cudaMalloc(&e->dev, A.host.size() * 4);
  if (err == cudaSuccess) err = cudaMemcpy(e->dev, A.host.data(), A.host.size() * 4, cudaMemcpyHostToDevice);
  if (err != cudaSuccess) {
    if (e->dev) cudaFree(e->dev);
    delete e;
    return fail(SOPRO_ERR_CUDA, "Mimi encoder weight upload failed: %s", cudaGetErrorString(err));
  }
  *out = e;
  return SOPRO_OK;
}

int sopro_mimi_encoder_destroy(sopro_mimi_encoder_t* e) {
  if (!e) return SOPRO_OK;
  cudaSetDevice(e->device);
  cudaFree(e->dev);
  cudaFree(e->rope);
  cudaFree(e->ws);
  cudaFree(e->wav_dev);
  cudaFree(e->codes_dev);
  cudaFree(e->lat_dev);
  cudaFree(e->info_dev);
  delete e;
  return SOPRO_OK;
}

int64_t sopro_mimi_encoded_frames(const sopro_mimi_encoder_t* e, int64_t n_samples) {
  if (!e || n_samples < 1 || n_samples > kEncMaxSamples) return -1;
  return enc_plan(e->cfg, n_samples).T;
}

int sopro_mimi_encode(sopro_mimi_encoder_t* e, const float* wav, int64_t n_samples, int32_t* codes, float* latent, void* stream) {
  if (!e || !wav || !codes) return fail(SOPRO_ERR_INVALID, "null argument");
  if (n_samples < 1 || n_samples > kEncMaxSamples)
    return fail(SOPRO_ERR_INVALID, "n_samples=%lld outside [1, %lld]", (long long)n_samples, kEncMaxSamples);
  CK(cudaSetDevice(e->device));
  cudaStream_t st = (cudaStream_t)stream;
  const EncPlan P = enc_plan(e->cfg, n_samples);
  const int rc = encode_prepare(e, (int)P.len[e->cfg.n_ratios], P.need, st);
  if (rc) return rc;
  return encode_run(e, P, 1, wav, n_samples, nullptr, codes, latent, st);
}

int sopro_mimi_encode_batch(sopro_mimi_encoder_t* e, const float* wav, int32_t B, int64_t stride, const int64_t* lens_host,
                            int32_t* codes, float* latent, void* stream) {
  if (!e || !wav || !lens_host || !codes) return fail(SOPRO_ERR_INVALID, "null argument");
  if (B < 1) return fail(SOPRO_ERR_INVALID, "B = %d < 1", B);
  long long most = 0;
  for (int b = 0; b < B; ++b) {
    if (lens_host[b] < 1 || lens_host[b] > kEncMaxSamples)
      return fail(SOPRO_ERR_INVALID, "lens[%d] = %lld outside [1, %lld]", b, (long long)lens_host[b], kEncMaxSamples);
    most = std::max(most, (long long)lens_host[b]);
  }
  if (stride < most) return fail(SOPRO_ERR_INVALID, "stride %lld < the longest row's %lld samples", (long long)stride, most);
  const sopro_mimi_config_t& c = e->cfg;
  const int NS = mimi::enc_info_cols(c.n_ratios);
  // pad to a multiple of every stride (2 * prod(ratios)): then no stage of the padded plan pads, and every clip's rows sit
  // at one pitch per stage
  long long unit = 2;
  for (int s = 0; s < c.n_ratios; ++s) unit *= c.ratios[s];
  const long long Lpad = (most + unit - 1) / unit * unit;
  if (Lpad * B > kEncMaxSamples)
    return fail(SOPRO_ERR_INVALID, "B = %d rows padded to %lld samples exceed %lld samples", B, Lpad, kEncMaxSamples);
  const EncPlan P = enc_plan(c, Lpad);
  std::vector<int> info((size_t)B * NS);
  for (int b = 0; b < B; ++b) {
    const EncPlan p = enc_plan(c, lens_host[b]);
    for (int s = 0; s <= c.n_ratios; ++s) info[(size_t)b * NS + s] = (int)p.len[s];
    info[(size_t)b * NS + NS - 1] = (int)p.T;
  }
  CK(cudaSetDevice(e->device));
  cudaStream_t st = (cudaStream_t)stream;
  if (e->info_cap < info.size()) {
    cudaFree(e->info_dev);
    e->info_dev = nullptr;
    e->info_cap = 0;
    CK(cudaMalloc(&e->info_dev, info.size() * sizeof(int)));
    e->info_cap = info.size();
  }
  CK(cudaMemcpyAsync(e->info_dev, info.data(), info.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  const int rc = encode_prepare(e, (int)P.len[c.n_ratios], (size_t)B * P.need, st);
  if (rc) return rc;
  return encode_run(e, P, B, wav, stride, e->info_dev, codes, latent, st);
}

int sopro_debug_mimi_rvq_encode(const float* proj, const float* embed, int32_t* codes, int T, int n_q, int n_sem, int V,
                                const int32_t* frames, int B, void* stream) {
  if (!proj || !embed || !codes) return fail(SOPRO_ERR_INVALID, "null argument");
  if (B < 1 || B > 65535 || T < 1 || n_q < 1 || n_sem < 1 || n_sem > n_q || V < 1)
    return fail(SOPRO_ERR_INVALID, "rvq encode: unsupported shape (B=%d T=%d n_q=%d n_sem=%d V=%d)", B, T, n_q, n_sem, V);
  // as encode_run launches it; frames (one column per clip) stands in for the last column of a batch's info
  rvq_encode_kernel<8><<<dim3(T, B), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(proj, embed, codes, T, n_q, n_sem, V, frames, 1);
  CK(cudaGetLastError());
  return SOPRO_OK;
}

int sopro_mimi_encode_host(sopro_mimi_encoder_t* e, const float* wav_host, int64_t n_samples, int32_t* codes_host,
                           float* latent_host, void* stream) {
  if (!e || !wav_host || !codes_host) return fail(SOPRO_ERR_INVALID, "null argument");
  if (n_samples < 1 || n_samples > kEncMaxSamples)
    return fail(SOPRO_ERR_INVALID, "n_samples=%lld outside [1, %lld]", (long long)n_samples, kEncMaxSamples);
  for (int64_t i = 0; i < n_samples; ++i)
    if (!std::isfinite(wav_host[i])) return fail(SOPRO_ERR_INVALID, "sample %lld is not finite (%g)", (long long)i, (double)wav_host[i]);
  CK(cudaSetDevice(e->device));
  cudaStream_t st = (cudaStream_t)stream;
  const long long T = enc_plan(e->cfg, n_samples).T;
  const size_t nc = (size_t)e->cfg.n_q * T, nl = (size_t)T * e->cfg.hidden;
  if (e->wav_cap < (size_t)n_samples) {
    cudaFree(e->wav_dev);
    e->wav_dev = nullptr;
    e->wav_cap = 0;
    CK(cudaMalloc(&e->wav_dev, (size_t)n_samples * 4));
    e->wav_cap = (size_t)n_samples;
  }
  if (e->codes_cap < nc) {
    cudaFree(e->codes_dev);
    e->codes_dev = nullptr;
    e->codes_cap = 0;
    CK(cudaMalloc(&e->codes_dev, nc * 4));
    e->codes_cap = nc;
  }
  if (latent_host && e->lat_cap < nl) {
    cudaFree(e->lat_dev);
    e->lat_dev = nullptr;
    e->lat_cap = 0;
    CK(cudaMalloc(&e->lat_dev, nl * 4));
    e->lat_cap = nl;
  }
  CK(cudaMemcpyAsync(e->wav_dev, wav_host, (size_t)n_samples * 4, cudaMemcpyHostToDevice, st));
  const int rc = sopro_mimi_encode(e, e->wav_dev, n_samples, e->codes_dev, latent_host ? e->lat_dev : nullptr, st);
  if (rc) return rc;
  CK(cudaMemcpyAsync(codes_host, e->codes_dev, nc * 4, cudaMemcpyDeviceToHost, st));
  if (latent_host) CK(cudaMemcpyAsync(latent_host, e->lat_dev, nl * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return SOPRO_OK;
}

}  // extern "C"
