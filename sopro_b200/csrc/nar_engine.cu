// NAR refiner (reference nn/nar.py:13-116, model.py:307-347) on the device as a handful of fused fp32 kernels:
// per stage  embed-mix + stage adapter (1 launch)  ->  6 x SSMLiteBlock (RMSNorm+GLU GEMM | dwconv+residual |
// RMSNorm+FFN1+GELU GEMM | FFN2+residual GEMM)  ->  RMSNorm+pre GEMM  ->  all heads of the stage in ONE grouped GEMM launch
// with an argmax epilogue (the logits never reach memory)  ->  argmax finish.  28 launches per stage instead of ~150
// ATen ops.  The ids must equal the reference's, so every contraction is fp32 (dense_f32.cuh).
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/sopro_b200.h"
#include "common.cuh"
#include "dense_f32.cuh"
#include "mimi_tc.cuh"  // tc::launch: the wgmma / TMA implicit-GEMM kernel, reused for the exact split products

namespace pstage {

struct FArena {
  std::vector<float> host;
  size_t add(const float* p, size_t n) {
    const size_t off = (host.size() + 63) / 64 * 64;
    host.resize(off + n);
    if (p) memcpy(host.data() + off, p, n * 4);
    return off;
  }
};

struct BlockOff {
  size_t norm_w, glu_w, glu_b, dw_w, dw_b, ffn_norm_w, w1, b1, w2, b2;
};

void add_block(FArena& A, const sopro_ssm_block_weights_t& L, int D, int k, BlockOff* o) {
  o->norm_w = A.add(L.norm_w, D);
  o->glu_w = A.add(L.glu_w, (size_t)2 * D * D);
  o->glu_b = A.add(L.glu_b, 2 * D);
  o->dw_w = A.add(L.dw_w, (size_t)D * k);
  o->dw_b = A.add(L.dw_b, D);
  o->ffn_norm_w = A.add(L.ffn_norm_w, D);
  o->w1 = A.add(L.ffn_w1, (size_t)4 * D * D);
  o->b1 = A.add(L.ffn_b1, 4 * D);
  o->w2 = A.add(L.ffn_w2, (size_t)4 * D * D);
  o->b2 = A.add(L.ffn_b2, D);
}

bool block_ok(const sopro_ssm_block_weights_t& L) {
  return L.norm_w && L.glu_w && L.glu_b && L.dw_w && L.dw_b && L.ffn_norm_w && L.ffn_w1 && L.ffn_b1 && L.ffn_w2 && L.ffn_b2;
}

// Tile edge of the tile kernel for an [M x N] output in `groups` groups: the largest of 128 / 64 / 32 that still gives
// (about) every SM a CTA -- a streaming window of ~190 rows would otherwise run on a handful of SMs.  The result does
// not depend on the choice (one fma chain over k per output, dense_f32.cuh).  GLU pairs value / gate columns inside a
// thread, which the 32-wide tile cannot: 64 is its smallest.
int tile_edge(int M, int N, int groups, int epi) {
  const int target = 120;
  for (int e : {128, 64}) {
    const long long ctas = (long long)((M + e - 1) / e) * ((N + e - 1) / e) * groups;
    if (ctas >= target) return e;
  }
  return epi == dense::EPI_GLU ? 64 : 32;
}

// C = epi(prologue(A) . W^T): picks the skinny kernel for M <= 16 rows, a tile kernel otherwise.
// groups > 1 (argmax heads): blockIdx.z = group.  edge: 0 = that choice, 16 = the skinny kernel (more than 16 rows in
// blocks of 16, each row with the reduction order of a launch of <= 16 rows), 32 / 64 / 128 = that tile edge (tests).
// parts_out: the argmax partial slots per row the launch writes.
int launch_dense(dense::DenseOp op, int groups, cudaStream_t st, int edge = 0, int* parts_out = nullptr) {
  if (op.K % 16 || op.M < 1 || op.N < 1) return fail(SOPRO_ERR_INVALID, "dense: bad shape M=%d N=%d K=%d", op.M, op.N, op.K);
  if (edge == 0) edge = op.M <= dense::kSkinnyRows ? 16 : tile_edge(op.M, op.N, groups, op.epi);
  if (edge == 16) {
    const int row_blocks = (op.M + dense::kSkinnyRows - 1) / dense::kSkinnyRows;
    if ((row_blocks > 1 && op.epi == dense::EPI_ARGMAX) || row_blocks > 65535)
      return fail(SOPRO_ERR_INVALID, "dense: M=%d too many rows for the skinny kernel", op.M);
    const int ncol = op.epi == dense::EPI_GLU ? op.N / 2 : op.N;
    // about two waves of CTAs over the GPU, at least one column per warp
    int cols = std::max(8, (ncol * groups + 295) / 296);
    cols = (cols + 7) / 8 * 8;
    const int parts = (ncol + cols - 1) / cols;
    if (op.epi == dense::EPI_ARGMAX) op.parts = parts;
    const size_t smem = (size_t)dense::kSkinnyRows * op.K * 4;
    if (smem > (size_t)16 * 2048 * 4) return fail(SOPRO_ERR_INVALID, "dense: K=%d too large for the skinny kernel", op.K);
    // a function attribute belongs to the current device's context: set once per device
    static unsigned long long attr_done = 0;
    if (tc::attr_needed(attr_done))
      CK(cudaFuncSetAttribute(dense::dense_skinny_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 16 * 2048 * 4));
    if (parts_out) *parts_out = parts;
    dense::dense_skinny_kernel<<<dim3(parts, row_blocks, groups), dense::kSkinnyThreads, smem, st>>>(op, cols);
  } else {
    const int e = edge;
    if ((e != 32 && e != 64 && e != 128) || (e == 32 && op.epi == dense::EPI_GLU))
      return fail(SOPRO_ERR_INVALID, "dense: no %d-wide tile for epilogue %d", e, op.epi);
    const dim3 grid((op.M + e - 1) / e, (op.N + e - 1) / e, groups);
    if (op.epi == dense::EPI_ARGMAX) op.parts = (int)grid.y;
    if (parts_out) *parts_out = (int)grid.y;
    if (e == 128) dense::dense_tile_kernel<128, 128><<<grid, dense::kTileThreads, 0, st>>>(op);
    else if (e == 64) dense::dense_tile_kernel<64, 64><<<grid, dense::kTileThreads, 0, st>>>(op);
    else dense::dense_tile_kernel<32, 32><<<grid, dense::kTileThreads, 0, st>>>(op);
  }
  CK(cudaGetLastError());
  return SOPRO_OK;
}

// argmax partial slots per row the launch above will write (must match launch_dense)
int argmax_parts(int M, int N, int groups) {
  if (M <= dense::kSkinnyRows) {
    int cols = std::max(8, (N * groups + 295) / 296);
    cols = (cols + 7) / 8 * 8;
    return (N + cols - 1) / cols;
  }
  const int e = tile_edge(M, N, groups, dense::EPI_ARGMAX);
  return (N + e - 1) / e;
}

// =================================================================================================
// Exact fp32 products on the tensor cores (row counts above the skinny kernel's).  Every fp32 operand is the exact sum
// of three bf16 terms (h + m + l: 3 x 8 mantissa bits), a product of two bf16 numbers is exact in fp32, so
//   x . w = sum over the six term pairs whose magnitude reaches fp32's last bit (mm, lh, hl, mh, hm, hh; the pairs ml, lm,
//   ll are below 2^-26 of the product)
// accumulated in fp32 by the tensor cores: the same quantity the fp32 FMA kernels compute, up to the order of the fp32
// additions.  One GEMM launch does all six: the weights are stored as W6 [N][6K] (K blocks = the w term of each pair,
// built once on the host), the activations as A3 [M][3K] = [h | m | l] written by split3_rows_kernel (fused with the
// RMSNorm of the rows), and the GEMM kernel's "tap" j (mimi_tc.cuh: K block j of W against A columns tap_col[j] + ...)
// selects the x term.  M = batch x frames rows fill 128-row tiles, which is what the tensor cores need (the AR step's
// 22..86 rows per CTA do not, DESIGN.md §3).
// =================================================================================================
constexpr int kPairs = 6;
constexpr int kPairX[kPairs] = {1, 2, 0, 1, 0, 0};  // x term of pair j (0 = h, 1 = m, 2 = l), smallest products first
constexpr int kPairW[kPairs] = {1, 0, 2, 0, 1, 0};  // w term of pair j

inline uint16_t bf16_rne(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);
  u += 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}
inline float bf16_f32(uint16_t h) {
  const uint32_t u = (uint32_t)h << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}
// W [N][K] fp32 -> W6 [N][6K] bf16 appended to `dst`; returns the element offset
size_t pack_w6(std::vector<uint16_t>& dst, const float* W, size_t N, size_t K) {
  const size_t off = (dst.size() + 63) / 64 * 64;
  dst.resize(off + N * kPairs * K);
  for (size_t n = 0; n < N; ++n)
    for (size_t k = 0; k < K; ++k) {
      const float w = W[n * K + k];
      uint16_t t[3];
      t[0] = bf16_rne(w);
      const float r1 = w - bf16_f32(t[0]);
      t[1] = bf16_rne(r1);
      t[2] = bf16_rne(r1 - bf16_f32(t[1]));
      for (int j = 0; j < kPairs; ++j) dst[off + (n * kPairs + j) * K + k] = t[kPairW[j]];
    }
  return off;
}

// rows [M][K] fp32 (optionally RMS-normalised, nn/blocks.py:32-37) -> A3 [M][3K] bf16 = [h | m | l], one warp per row
__global__ void __launch_bounds__(256) split3_rows_kernel(const float* __restrict__ x, const float* __restrict__ norm_w,
                                                          __nv_bfloat16* __restrict__ out, long long rows, int K) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* xr = x + row * K;
  float inv = 1.f;
  if (norm_w) {
    float ss = 0.f;
    for (int k = lane * 4; k < K; k += 128) {
      const float4 v = *reinterpret_cast<const float4*>(xr + k);
      ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    inv = 1.0f / sqrtf(ss / (float)K + 1e-6f);
  }
  __nv_bfloat16* o = out + row * 3 * K;
  for (int k = lane * 4; k < K; k += 128) {
    float4 v = *reinterpret_cast<const float4*>(xr + k);
    if (norm_w) {
      const float4 w = __ldg(reinterpret_cast<const float4*>(norm_w + k));
      v.x = (v.x * inv) * w.x;
      v.y = (v.y * inv) * w.y;
      v.z = (v.z * inv) * w.z;
      v.w = (v.w * inv) * w.w;
    }
    const __nv_bfloat162 h0 = __floats2bfloat162_rn(v.x, v.y), h1 = __floats2bfloat162_rn(v.z, v.w);
    const float rx = v.x - __low2float(h0), ry = v.y - __high2float(h0), rz = v.z - __low2float(h1), rw = v.w - __high2float(h1);
    const __nv_bfloat162 m0 = __floats2bfloat162_rn(rx, ry), m1 = __floats2bfloat162_rn(rz, rw);
    const __nv_bfloat162 l0 = __floats2bfloat162_rn(rx - __low2float(m0), ry - __high2float(m0));
    const __nv_bfloat162 l1 = __floats2bfloat162_rn(rz - __low2float(m1), rw - __high2float(m1));
    uint2 ph, pm, pl;
    ph.x = *reinterpret_cast<const unsigned*>(&h0), ph.y = *reinterpret_cast<const unsigned*>(&h1);
    pm.x = *reinterpret_cast<const unsigned*>(&m0), pm.y = *reinterpret_cast<const unsigned*>(&m1);
    pl.x = *reinterpret_cast<const unsigned*>(&l0), pl.y = *reinterpret_cast<const unsigned*>(&l1);
    *reinterpret_cast<uint2*>(o + k) = ph;
    *reinterpret_cast<uint2*>(o + K + k) = pm;
    *reinterpret_cast<uint2*>(o + 2 * K + k) = pl;
  }
}

// GLU (nn/blocks.py:16-23) on the GEMM's [M][2D] output (bias included): h = value * sigmoid(gate)
__global__ void __launch_bounds__(256) glu_rows_kernel(const float* __restrict__ v, float* __restrict__ h, long long rows, int D) {
  const long long i = ((long long)blockIdx.x * 256 + threadIdx.x) * 4;
  if (i >= rows * D) return;
  const long long r = i / D;
  const int c = (int)(i - r * D);
  const float4 a = *reinterpret_cast<const float4*>(v + r * 2 * D + c);
  const float4 g = *reinterpret_cast<const float4*>(v + r * 2 * D + D + c);
  float4 o;
  o.x = a.x * dense::sigmoid_ref(g.x);
  o.y = a.y * dense::sigmoid_ref(g.y);
  o.z = a.z * dense::sigmoid_ref(g.z);
  o.w = a.w * dense::sigmoid_ref(g.w);
  *reinterpret_cast<float4*>(h + i) = o;
}

// first maximum (torch.argmax) of each head's V logits: one warp per (row, head)
__global__ void __launch_bounds__(256) argmax_heads_kernel(const float* __restrict__ logits, long long rows, int heads, int V,
                                                           int* __restrict__ codes, int Q) {
  const long long w = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (w >= rows * heads) return;
  const long long r = w / heads;
  const int hd = (int)(w - r * heads);
  const float* lg = logits + (r * heads + hd) * V;
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int c = lane * 4; c < V; c += 128) {
    const float4 q = *reinterpret_cast<const float4*>(lg + c);
    const float vv[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int e = 0; e < 4; ++e)
      if (dense::before(vv[e], c + e, bv, bi)) bv = vv[e], bi = c + e;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (dense::before(ov, oi, bv, bi)) bv = ov, bi = oi;
  }
  if (lane == 0) codes[r * Q + hd] = bi;
}

// C [M][N] = epi(A . W^T + bias): A3 [M][3K] bf16 (split3_rows_kernel), W6 [N][6K] bf16 (pack_w6)
int launch_tc6(const __nv_bfloat16* A3, const uint16_t* W6, const float* bias, const float* R, float* C, long long M, int N, int K, int epi,
               cudaStream_t st) {
  tc::TcOp o{};
  o.bias = bias;
  o.R = R;
  o.out_f32 = C;
  o.c_bs = M * N;
  o.M = (int)M;
  o.N = N;
  o.K = kPairs * K;
  o.Cin = K;
  o.dil = 0;
  o.pad = 0;
  o.bias_mod = N;
  o.epi = epi;
  for (int j = 0; j < kPairs; ++j) o.tap_col[j] = kPairX[j] * K;
  if (!tc::supported(N, o.K, K)) return fail(SOPRO_ERR_INVALID, "tensor-core NAR GEMM: unsupported shape N=%d K=%d", N, K);
  const cudaError_t e = tc::launch(A3, M, W6, o, 1, st, 3 * K);
  if (e != cudaSuccess) return fail(SOPRO_ERR_CUDA, "tensor-core NAR GEMM (N=%d K=%d M=%lld): %s", N, K, M, cudaGetErrorString(e));
  return SOPRO_OK;
}

struct BlockTc {
  size_t glu, w1, w2;  // W6 element offsets
};

// one SSMLiteBlock with the three contractions on the tensor cores; a3 [M][3*4D] bf16 and v [M][4D] fp32 are scratch
int ssm_block_tc(const float* W, const BlockOff& o, const uint16_t* T, const BlockTc& t, float* x, float* h, float* v, __nv_bfloat16* a3,
                 const int* lens, int B, int Tmax, int D, int k, int dil, cudaStream_t st) {
  const long long M = (long long)B * Tmax;
  const unsigned rb = (unsigned)((M + 7) / 8);
  split3_rows_kernel<<<rb, 256, 0, st>>>(x, W + o.norm_w, a3, M, D);
  int rc = launch_tc6(a3, T + t.glu, W + o.glu_b, nullptr, v, M, 2 * D, D, tc::EPI_NONE, st);
  if (rc) return rc;
  glu_rows_kernel<<<(unsigned)((M * D / 4 + 255) / 256), 256, 0, st>>>(v, h, M, D);
  const int total = (k - 1) * dil;
  dense::dwconv_res_kernel<<<dim3(Tmax, B), 128, 0, st>>>(h, x, W + o.dw_w, W + o.dw_b, x, lens, Tmax, D, k, dil, total / 2);
  split3_rows_kernel<<<rb, 256, 0, st>>>(x, W + o.ffn_norm_w, a3, M, D);
  if ((rc = launch_tc6(a3, T + t.w1, W + o.b1, nullptr, v, M, 4 * D, D, tc::EPI_GELU, st))) return rc;
  split3_rows_kernel<<<rb, 256, 0, st>>>(v, nullptr, a3, M, 4 * D);
  if ((rc = launch_tc6(a3, T + t.w2, W + o.b2, x, x, M, D, 4 * D, tc::EPI_RES, st))) return rc;
  CK(cudaGetLastError());
  return SOPRO_OK;
}

// one SSMLiteBlock (nn/blocks.py:143-148) over rows [B][Tmax][D], in place on x; h [M][D] and hid [M][4D] are scratch
int ssm_block(const float* W, const BlockOff& o, float* x, float* h, float* hid, const int* lens, int B, int Tmax, int D, int k, int dil,
              bool causal, cudaStream_t st) {
  const int M = B * Tmax;
  dense::DenseOp g{};
  g.A = x; g.W = W + o.glu_w; g.bias = W + o.glu_b; g.norm_w = W + o.norm_w; g.C = h; g.M = M; g.N = 2 * D; g.K = D; g.ldc = D;
  g.epi = dense::EPI_GLU;
  int rc = launch_dense(g, 1, st);
  if (rc) return rc;
  const int total = (k - 1) * dil, left = causal ? total : total / 2;
  dense::dwconv_res_kernel<<<dim3(Tmax, B), 128, 0, st>>>(h, x, W + o.dw_w, W + o.dw_b, x, lens, Tmax, D, k, dil, left);
  CK(cudaGetLastError());
  g = dense::DenseOp{};
  g.A = x; g.W = W + o.w1; g.bias = W + o.b1; g.norm_w = W + o.ffn_norm_w; g.C = hid; g.M = M; g.N = 4 * D; g.K = D; g.ldc = 4 * D;
  g.epi = dense::EPI_GELU;
  if ((rc = launch_dense(g, 1, st))) return rc;
  g = dense::DenseOp{};
  g.A = hid; g.W = W + o.w2; g.bias = W + o.b2; g.R = x; g.C = x; g.M = M; g.N = D; g.K = 4 * D; g.ldc = D; g.epi = dense::EPI_RES;
  return launch_dense(g, 1, st);
}

// ---- NAR stage input (model.py:318-341 + nn/embeddings.py:77-112 + nn/nar.py:28-32), one warp per (b, t) row:
//   prev = sum_j w[j] * cb_embed[cb[j]*V + tok[j]]      (the codebooks decided so far, softmax weights)
//   x    = mix0 * cond + mix1 * prev
//   out  = RMSNorm(x) * (1 + tanh(g)) + tanh(b)         (stage adapter; g, b depend on the stage only)
struct EmbedMix {
  const float* cond;      // [B][cond_bs] rows of D
  long long cond_bs;
  const int* codes;       // [B][Tmax][Q] (codebooks < n_prev already decided)
  const float* emb;       // [Q*V + 1][D]
  const float* w_prev;    // [n_prev]
  const float* norm_w;    // adapter RMSNorm
  const float* mul;       // [D] 1 + tanh(g)
  const float* add;       // [D] tanh(b)
  float* out;             // [B][Tmax][D]
  float mix0, mix1;
  int Tmax, D, Q, V, n_prev;
};

__global__ void __launch_bounds__(256) nar_embed_mix_kernel(const EmbedMix p, long long rows) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const long long b = row / p.Tmax, t = row - b * p.Tmax;
  const float* c = p.cond + b * p.cond_bs + t * p.D;
  const int* tk = p.codes + row * p.Q;
  constexpr int kMaxPer = 16;  // D <= 512
  float x[kMaxPer];
  float ss = 0.f;
  int n = 0;
  for (int k = lane; k < p.D; k += 32, ++n) {
    float prev = 0.f;
    for (int j = 0; j < p.n_prev; ++j) {
      const int tok = min(max(tk[j], 0), p.V - 1);
      prev += __ldg(p.w_prev + j) * __ldg(p.emb + ((size_t)j * p.V + tok) * p.D + k);
    }
    const float v = p.mix0 * c[k] + p.mix1 * prev;
    x[n] = v;
    ss += v * v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float inv = 1.0f / sqrtf(ss / (float)p.D + 1e-6f);
  n = 0;
  for (int k = lane; k < p.D; k += 32, ++n)
    p.out[row * p.D + k] = ((x[n] * inv) * __ldg(p.norm_w + k)) * __ldg(p.mul + k) + __ldg(p.add + k);
}

// codes[b][t][0] = rvq1[b][t]
__global__ void set_first_codebook_kernel(const int* __restrict__ rvq1, int* __restrict__ codes, long long rows, int Q) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < rows) codes[i * Q] = rvq1[i];
}

}  // namespace pstage

using namespace pstage;

struct sopro_nar {
  int device = 0;
  sopro_nar_config_t cfg{};
  float* dev = nullptr;
  size_t n_floats = 0;
  BlockOff blk[SOPRO_MAX_SSM_LAYERS]{};
  size_t norm_w = 0, pre_w = 0, pre_b = 0, adapter_norm_w = 0, emb = 0;
  struct Stage {
    int first, count, n_prev;
    size_t w_prev, mul, add, head_w, head_b, head_id;
    float mix0, mix1;
    size_t tc_heads = 0, head_b_folded = 0;  // tensor-core path: W6 of the stage's heads; bias + W . id_embedding
  };
  // tensor-core path (exact six-product split): W6 images of every contraction, bf16
  uint16_t* tcw = nullptr;
  BlockTc tblk[SOPRO_MAX_SSM_LAYERS]{};
  size_t tc_pre = 0;
  bool tc_ok = false;
  std::vector<Stage> stages;
  // workspace
  float* ws = nullptr;
  size_t ws_bytes = 0;
  const int32_t* forced = nullptr;  // test hook: the previous codebooks every stage conditions on
  float* trace_z = nullptr;         // test hook: every stage's pre-head activation z, [n_stages][B][Tmax][Hn]
  int tc_mode = -1;                 // -1 automatic (tensor cores above the skinny kernel's row count), 0 fp32 FMA kernels only
  // launch-bound streaming windows (one utterance, <= kNarGraphRows frames: 113..217 launches each) are replayed from
  // CUDA graphs captured over static buffers; every graph dies when the workspace is reallocated
  struct Replay {
    int T, tc;
    cudaGraphExec_t exec;
  };
  std::vector<Replay> replays;
  float* g_cond = nullptr;
  int32_t* g_rvq1 = nullptr;
  int32_t* g_codes = nullptr;
  bool graphs = true;
  cudaStream_t cap_stream = nullptr;
  cudaEvent_t g_done = nullptr;     // last replay's completion: the static buffers are reused across caller streams
  size_t reserve_bytes = 0;         // workspace floor (so that no graph-sized call reallocates)
};

constexpr int kNarGraphRows = 256;

static void nar_drop_replays(sopro_nar* n) {
  for (auto& r : n->replays) cudaGraphExecDestroy(r.exec);
  n->replays.clear();
}

extern "C" {

int sopro_nar_create(const sopro_nar_config_t* cfg, const sopro_nar_weights_t* w, int device, sopro_nar_t** out) {
  if (!cfg || !w || !out) return fail(SOPRO_ERR_INVALID, "null argument");
  *out = nullptr;
  const int rc = open_device(device, "the NAR refiner");
  if (rc != SOPRO_OK) return rc;
  const int D = cfg->d_model, NL = cfg->n_layers, k = cfg->kernel, Q = cfg->n_codebooks, V = cfg->codebook_size, Hn = cfg->head_dim,
            AH = cfg->adapter_hidden, NS = cfg->n_stages;
  if (D < 32 || D > 512 || D % 16 || Hn % 16 || NL < 1 || NL > SOPRO_MAX_SSM_LAYERS || k < 1 || k > 64 || Q < 2 || Q > SOPRO_NAR_MAX_CODEBOOKS ||
      NS < 1 || NS > SOPRO_NAR_MAX_STAGES || V < 2 || AH < 1)
    return fail(SOPRO_ERR_INVALID, "unsupported NAR geometry (d_model=%d head_dim=%d layers=%d codebooks=%d stages=%d)", D, Hn, NL, Q, NS);
  for (int i = 0; i < NL; ++i)
    if (!block_ok(w->block[i]) || cfg->dilation[i] < 1) return fail(SOPRO_ERR_INVALID, "NAR block %d: null weight or bad dilation", i);
  if (!w->norm_w || !w->pre_w || !w->pre_b || !w->stage_emb || !w->adapter_norm_w || !w->adapter_w0 || !w->adapter_b0 || !w->adapter_w2 ||
      !w->adapter_b2 || !w->prev_cb_weights || !w->cb_embed)
    return fail(SOPRO_ERR_INVALID, "NAR: null weight pointer");
  int covered = 1;
  for (int s = 0; s < NS; ++s) {
    if (cfg->stage_first[s] != covered || cfg->stage_count[s] < 1 || !w->head_id_emb[s] || !w->mix[s])
      return fail(SOPRO_ERR_INVALID, "NAR stage %d: codebooks must be consecutive from 1 (first=%d count=%d)", s, cfg->stage_first[s],
                  cfg->stage_count[s]);
    for (int j = 0; j < cfg->stage_count[s]; ++j)
      if (covered + j >= Q || !w->head_w[covered + j] || !w->head_b[covered + j])
        return fail(SOPRO_ERR_INVALID, "NAR stage %d head %d: null weight or codebook out of range", s, j);
    covered += cfg->stage_count[s];
  }
  sopro_nar* n = new sopro_nar();
  n->device = device;
  n->cfg = *cfg;
  FArena A;
  for (int i = 0; i < NL; ++i) add_block(A, w->block[i], D, k, &n->blk[i]);
  n->norm_w = A.add(w->norm_w, D);
  n->pre_w = A.add(w->pre_w, (size_t)Hn * D);
  n->pre_b = A.add(w->pre_b, Hn);
  n->adapter_norm_w = A.add(w->adapter_norm_w, D);
  n->emb = A.add(w->cb_embed, ((size_t)Q * V + 1) * D);
  for (int s = 0; s < NS; ++s) {
    sopro_nar::Stage S{};
    S.first = cfg->stage_first[s];
    S.count = cfg->stage_count[s];
    S.n_prev = S.first;  // codebooks 0 .. first-1 are decided when the stage runs
    // softmax over the previous codebooks' weights (model.py:332, nn/embeddings.py:94-108), in double
    {
      std::vector<double> e(S.n_prev);
      double mx = -1e300, sum = 0;
      for (int j = 0; j < S.n_prev; ++j) mx = std::max(mx, (double)w->prev_cb_weights[j]);
      for (int j = 0; j < S.n_prev; ++j) sum += (e[j] = exp((double)w->prev_cb_weights[j] - mx));
      std::vector<float> wp(S.n_prev);
      for (int j = 0; j < S.n_prev; ++j) wp[j] = (float)(e[j] / sum);
      S.w_prev = A.add(wp.data(), wp.size());
    }
    {
      const double a = w->mix[s][0], b = w->mix[s][1], mx = std::max(a, b);
      const double ea = exp(a - mx), eb = exp(b - mx);
      S.mix0 = (float)(ea / (ea + eb));
      S.mix1 = (float)(eb / (ea + eb));
    }
    // stage adapter MLP on the stage embedding (nn/nar.py:20-31): g, b = Linear(GELU(Linear(e))).chunk(2); constants
    {
      std::vector<double> hmid(AH);
      const float* e = w->stage_emb + (size_t)s * D;
      for (int i = 0; i < AH; ++i) {
        double acc = w->adapter_b0[i];
        for (int c = 0; c < D; ++c) acc += (double)w->adapter_w0[(size_t)i * D + c] * e[c];
        const double x = acc;
        hmid[i] = 0.5 * x * (1.0 + erf(x * 0.70710678118654752440));
      }
      std::vector<float> mul(D), add(D);
      for (int c = 0; c < 2 * D; ++c) {
        double acc = w->adapter_b2[c];
        for (int i = 0; i < AH; ++i) acc += (double)w->adapter_w2[(size_t)c * AH + i] * hmid[i];
        if (c < D) mul[c] = (float)(1.0 + tanh(acc));
        else add[c - D] = (float)tanh(acc);
      }
      S.mul = A.add(mul.data(), D);
      S.add = A.add(add.data(), D);
    }
    // the stage's heads, contiguous: W [count][V][Hn], bias [count][V], id embedding [count][Hn]
    S.head_w = A.add(nullptr, (size_t)S.count * V * Hn);
    S.head_b = A.add(nullptr, (size_t)S.count * V);
    for (int j = 0; j < S.count; ++j) {
      memcpy(A.host.data() + S.head_w + (size_t)j * V * Hn, w->head_w[S.first + j], (size_t)V * Hn * 4);
      memcpy(A.host.data() + S.head_b + (size_t)j * V, w->head_b[S.first + j], (size_t)V * 4);
    }
    S.head_id = A.add(w->head_id_emb[s], (size_t)S.count * Hn);
    {  // (z + e_h) . W_h^T + b_h = z . W_h^T + (b_h + W_h e_h): the head's id embedding folded into its bias
      std::vector<float> fb((size_t)S.count * V);
      for (int j = 0; j < S.count; ++j) {
        const float* Wh = w->head_w[S.first + j];
        const float* e = w->head_id_emb[s] + (size_t)j * Hn;
        for (int v = 0; v < V; ++v) {
          double acc = w->head_b[S.first + j][v];
          for (int c = 0; c < Hn; ++c) acc += (double)Wh[(size_t)v * Hn + c] * (double)e[c];
          fb[(size_t)j * V + v] = (float)acc;
        }
      }
      S.head_b_folded = A.add(fb.data(), fb.size());
    }
    n->stages.push_back(S);
  }
  // tensor-core images (W6) of every contraction; geometry the implicit-GEMM kernel takes: K blocks of 64, N tiles of 32+
  std::vector<uint16_t> T;
  const bool tc_ok = D % 64 == 0 && Hn % 64 == 0 && V % 32 == 0 && (2 * D) % 32 == 0;
  if (tc_ok) {
    for (int i = 0; i < NL; ++i) {
      n->tblk[i].glu = pack_w6(T, w->block[i].glu_w, (size_t)2 * D, D);
      n->tblk[i].w1 = pack_w6(T, w->block[i].ffn_w1, (size_t)4 * D, D);
      n->tblk[i].w2 = pack_w6(T, w->block[i].ffn_w2, D, (size_t)4 * D);
    }
    n->tc_pre = pack_w6(T, w->pre_w, Hn, D);
    for (auto& S : n->stages) {
      std::vector<float> hw((size_t)S.count * V * Hn);
      for (int j = 0; j < S.count; ++j) memcpy(hw.data() + (size_t)j * V * Hn, w->head_w[S.first + j], (size_t)V * Hn * 4);
      S.tc_heads = pack_w6(T, hw.data(), (size_t)S.count * V, Hn);
    }
  }
  n->n_floats = A.host.size();
  cudaError_t err = cudaMalloc(&n->dev, n->n_floats * 4);
  if (err == cudaSuccess) err = cudaMemcpy(n->dev, A.host.data(), n->n_floats * 4, cudaMemcpyHostToDevice);
  if (err == cudaSuccess && tc_ok) {
    err = cudaMalloc(&n->tcw, T.size() * 2);
    if (err == cudaSuccess) err = cudaMemcpy(n->tcw, T.data(), T.size() * 2, cudaMemcpyHostToDevice);
    n->tc_ok = err == cudaSuccess;
  }
  if (err != cudaSuccess) {
    if (n->dev) cudaFree(n->dev);
    if (n->tcw) cudaFree(n->tcw);
    delete n;
    return fail(SOPRO_ERR_CUDA, "NAR weight upload (%zu MB) failed: %s", (A.host.size() * 4 + T.size() * 2) >> 20, cudaGetErrorString(err));
  }
  *out = n;
  return SOPRO_OK;
}

int sopro_nar_destroy(sopro_nar_t* n) {
  if (!n) return SOPRO_OK;
  cudaSetDevice(n->device);
  nar_drop_replays(n);
  if (n->cap_stream) cudaStreamDestroy(n->cap_stream);
  if (n->g_done) cudaEventDestroy(n->g_done);
  cudaFree(n->g_cond);
  cudaFree(n->g_rvq1);
  cudaFree(n->g_codes);
  cudaFree(n->dev);
  cudaFree(n->tcw);
  cudaFree(n->ws);
  delete n;
  return SOPRO_OK;
}

// test hook (host only): the W6 image pack_w6 builds for W [N][K] -> out [N][6K] bf16 bit patterns
int sopro_debug_pack_w6(const float* W, int N, int K, uint16_t* out) {
  if (!W || !out || N < 1 || K < 1) return fail(SOPRO_ERR_INVALID, "bad argument");
  std::vector<uint16_t> T;
  const size_t off = pack_w6(T, W, (size_t)N, (size_t)K);
  memcpy(out, T.data() + off, (size_t)N * kPairs * K * 2);
  return SOPRO_OK;
}

int sopro_debug_dense(const float* A, const float* W, const float* bias, const float* norm_w, const float* a_add, const float* R, float* C,
                      float gate, int M, int N, int K, int ldc, int epi, int groups, int64_t zW, int64_t zBias, int64_t zAdd, int kernel,
                      int32_t* ids, void* ws, int64_t ws_bytes, void* stream) {
  if (!A || !W) return fail(SOPRO_ERR_INVALID, "null argument");
  const bool glu = epi == dense::EPI_GLU, amax = epi == dense::EPI_ARGMAX;
  if (epi < dense::EPI_BIAS || epi > dense::EPI_RES_GATE || groups < 1 || groups > 65535 || M < 1 || M > 0x3fffffff || N < 1 || K < 16 ||
      K % 16 || zW < 0 || zBias < 0 || zAdd < 0 || (glu && (N % 2 || !bias)) ||
      ((epi == dense::EPI_RES || epi == dense::EPI_RES_GATE) && !R) || (!amax && (!C || ldc < (glu ? N / 2 : N))))
    return fail(SOPRO_ERR_INVALID, "debug dense: bad arguments (M=%d N=%d K=%d epi=%d groups=%d ldc=%d)", M, N, K, epi, groups, ldc);
  if ((kernel != 0 && kernel != 16 && kernel != 32 && kernel != 64 && kernel != 128) || (kernel == 16 && M > dense::kSkinnyRows) ||
      (kernel == 32 && glu) || (kernel == 16 && K > 2048))
    return fail(SOPRO_ERR_INVALID, "debug dense: kernel %d does not take M=%d K=%d epi=%d", kernel, M, K, epi);
  const long long slots = (long long)groups * M * ((N + 7) / 8);  // >= groups * M * parts of any kernel choice
  if (amax && (!ids || !ws || ws_bytes < 8 * slots)) return fail(SOPRO_ERR_INVALID, "debug dense: argmax needs ids and %lld workspace bytes", 8 * slots);
  if (!amax && groups > 1) return fail(SOPRO_ERR_INVALID, "debug dense: grouped launches are argmax only");
  dense::DenseOp op{};
  op.A = A; op.W = W; op.bias = bias; op.norm_w = norm_w; op.a_add = a_add; op.R = R; op.C = C; op.gate = gate;
  op.M = M; op.N = N; op.K = K; op.ldc = ldc; op.epi = epi; op.zW = (size_t)zW; op.zBias = (size_t)zBias; op.zAdd = (size_t)zAdd;
  if (amax) {
    op.amax_val = static_cast<float*>(ws);
    op.amax_idx = reinterpret_cast<int*>(static_cast<float*>(ws) + slots);
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int parts = 0;
  int rc = launch_dense(op, groups, st, kernel, &parts);
  if (rc || !amax) return rc;
  dense::argmax_finish_kernel<<<dim3((unsigned)((M + 127) / 128), groups), 128, 0, st>>>(op.amax_val, op.amax_idx, M, parts, ids, groups);
  CK(cudaGetLastError());
  return SOPRO_OK;
}

int sopro_debug_tc6(const float* X, const float* norm_w, const uint16_t* W6, const float* bias, const float* R, float* C, void* A3, int64_t M,
                    int N, int K, int epi, void* stream) {
  if (!X || !W6 || !C || !A3 || (epi == tc::EPI_RES && !R)) return fail(SOPRO_ERR_INVALID, "null argument");
  if (M < 1 || M > 0x3fffffffLL || K < 4 || K % 4 || N < 1 || (epi != tc::EPI_NONE && epi != tc::EPI_GELU && epi != tc::EPI_RES) ||
      !tc::supported(N, kPairs * K, K))
    return fail(SOPRO_ERR_INVALID, "debug tc6: unsupported shape M=%lld N=%d K=%d epi=%d", (long long)M, N, K, epi);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  __nv_bfloat16* a3 = static_cast<__nv_bfloat16*>(A3);
  split3_rows_kernel<<<(unsigned)((M + 7) / 8), 256, 0, st>>>(X, norm_w, a3, M, K);
  CK(cudaGetLastError());
  return launch_tc6(a3, W6, bias, R, C, M, N, K, epi, st);
}

int sopro_debug_dwconv_res(const float* h, const float* x, const float* w, const float* bias, float* out, const int32_t* lens, int B, int Tmax,
                           int D, int k, int dil, int left, void* stream) {
  if (!h || !x || !w || !bias || !out) return fail(SOPRO_ERR_INVALID, "null argument");
  if (B < 1 || B > 65535 || Tmax < 1 || D < 1 || k < 1 || k > 64 || dil < 1 || left < 0 || left > (k - 1) * dil)
    return fail(SOPRO_ERR_INVALID, "debug dwconv: bad shape B=%d Tmax=%d D=%d k=%d dil=%d left=%d", B, Tmax, D, k, dil, left);
  dense::dwconv_res_kernel<<<dim3(Tmax, B), 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(h, x, w, bias, out, lens, Tmax, D, k, dil, left);
  CK(cudaGetLastError());
  return SOPRO_OK;
}

int sopro_debug_argmax_heads(const float* logits, int64_t rows, int heads, int V, int32_t* codes, int Q, void* stream) {
  if (!logits || !codes) return fail(SOPRO_ERR_INVALID, "null argument");
  if (rows < 1 || rows > 0x3fffffffLL || heads < 1 || V < 4 || V % 4 || Q < heads)
    return fail(SOPRO_ERR_INVALID, "debug argmax heads: bad shape rows=%lld heads=%d V=%d Q=%d", (long long)rows, heads, V, Q);
  argmax_heads_kernel<<<(unsigned)((rows * heads + 7) / 8), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(logits, rows, heads, V, codes, Q);
  CK(cudaGetLastError());
  return SOPRO_OK;
}

int sopro_nar_set_contraction(sopro_nar_t* n, int mode) {
  if (!n || mode < -1 || mode > 1) return fail(SOPRO_ERR_INVALID, "bad argument");
  if (mode == 1 && !n->tc_ok) return fail(SOPRO_ERR_INVALID, "this NAR geometry has no tensor-core images");
  n->tc_mode = mode;
  return SOPRO_OK;
}

int sopro_nar_set_forced(sopro_nar_t* n, const int32_t* forced_codes) {
  if (!n) return fail(SOPRO_ERR_INVALID, "null argument");
  n->forced = forced_codes;
  return SOPRO_OK;
}

int sopro_nar_set_trace(sopro_nar_t* n, float* z) {
  if (!n) return fail(SOPRO_ERR_INVALID, "null argument");
  n->trace_z = z;
  return SOPRO_OK;
}

}  // extern "C"

// the refiner's launches on `st`; reserve_only: size (and grow) the workspace for this shape, launch nothing
static int nar_refine_impl(sopro_nar_t* n, const float* cond, int64_t cond_batch_stride, const int32_t* rvq1, const int32_t* lens, int B,
                           int Tmax, int32_t* codes, void* stream, bool reserve_only = false) {
  if (!n || (!reserve_only && (!cond || !rvq1 || !codes))) return fail(SOPRO_ERR_INVALID, "null argument");
  if (B < 1 || Tmax < 1 || (long long)B * Tmax > 0x3fffffffLL) return fail(SOPRO_ERR_INVALID, "bad B=%d Tmax=%d", B, Tmax);
  const sopro_nar_config_t& c = n->cfg;
  const int D = c.d_model, Q = c.n_codebooks, V = c.codebook_size, Hn = c.head_dim;
  if (cond_batch_stride < (int64_t)Tmax * D) return fail(SOPRO_ERR_INVALID, "cond_batch_stride smaller than Tmax*d_model");
  CK(cudaSetDevice(n->device));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long M = (long long)B * Tmax;
  int max_heads = 1;
  for (const auto& S : n->stages) max_heads = std::max(max_heads, S.count);
  const size_t parts_max = (size_t)std::max(argmax_parts((int)M, V, 1), argmax_parts((int)M, V, max_heads));
  // Tensor cores (exact six-product split) for every row count the skinny fp32 kernel does not take; SOPRO_NAR_TC=0 keeps
  // the fp32 FMA tile kernels (the reference for tests/test_nar_gpu.py::test_tensor_core_path_equals_the_fp32_path)
  static const bool tc_env_off = getenv("SOPRO_NAR_TC") && atoi(getenv("SOPRO_NAR_TC")) == 0;
  const bool use_tc = n->tc_ok && !tc_env_off && n->tc_mode != 0 && M > dense::kSkinnyRows;
  // rows per head-logits chunk of the tensor-core path (logits [chunk][heads * V] fp32 reach memory there, <= 256 MB)
  long long mc = ((256ll << 20) / ((long long)max_heads * V * 4)) / 128 * 128;
  mc = std::max<long long>(128, std::min<long long>(mc, (M + 127) / 128 * 128));
  const size_t fx = (size_t)M * D, fh = (size_t)M * D, fhid = (size_t)M * 4 * D, fz = (size_t)M * Hn,
               famax = use_tc ? 0 : (size_t)max_heads * M * parts_max;
  auto al = [](size_t x) { return (x + 63) / 64 * 64; };
  const size_t fa3 = use_tc ? ((size_t)M * 3 * 4 * D + 1) / 2 : 0;          // bf16 [M][3 * 4D], in floats
  const size_t flog = use_tc ? (size_t)mc * max_heads * V : 0;
  const size_t need = std::max(n->reserve_bytes, (al(fx) + al(fh) + al(fhid) + al(fz) + 2 * al(famax) + al(fa3) + al(flog)) * 4);
  if (n->ws_bytes < need) {
    CK(cudaStreamSynchronize(st));
    nar_drop_replays(n);  // the graphs hold pointers into the old workspace
    cudaFree(n->ws);
    n->ws = nullptr;
    n->ws_bytes = 0;
    cudaError_t e = cudaMalloc(&n->ws, need);
    if (e != cudaSuccess) return fail(SOPRO_ERR_CUDA, "NAR workspace %zu MB: %s", need >> 20, cudaGetErrorString(e));
    n->ws_bytes = need;
  }
  if (reserve_only) {
    n->reserve_bytes = std::max(n->reserve_bytes, need);
    return SOPRO_OK;
  }
  float* x = n->ws;
  float* h = x + al(fx);
  float* hid = h + al(fh);
  float* z = hid + al(fhid);
  float* amax_v = z + al(fz);
  int* amax_i = reinterpret_cast<int*>(amax_v + al(famax));
  __nv_bfloat16* a3 = reinterpret_cast<__nv_bfloat16*>(amax_v + 2 * al(famax));
  float* logits = amax_v + 2 * al(famax) + al(fa3);
  const float* W = n->dev;
  set_first_codebook_kernel<<<(unsigned)((M + 255) / 256), 256, 0, st>>>(rvq1, codes, M, Q);
  CK(cudaGetLastError());
  float* trace = n->trace_z;
  for (const auto& S : n->stages) {
    EmbedMix em{};
    em.cond = cond; em.cond_bs = cond_batch_stride; em.codes = n->forced ? n->forced : codes; em.emb = W + n->emb; em.w_prev = W + S.w_prev;
    em.norm_w = W + n->adapter_norm_w; em.mul = W + S.mul; em.add = W + S.add; em.out = x; em.mix0 = S.mix0; em.mix1 = S.mix1;
    em.Tmax = Tmax; em.D = D; em.Q = Q; em.V = V; em.n_prev = S.n_prev;
    nar_embed_mix_kernel<<<(unsigned)((M + 7) / 8), 256, 0, st>>>(em, M);
    CK(cudaGetLastError());
    int rc;
    if (use_tc) {
      for (int i = 0; i < c.n_layers; ++i)
        if ((rc = ssm_block_tc(W, n->blk[i], n->tcw, n->tblk[i], x, h, hid, a3, lens, B, Tmax, D, c.kernel, c.dilation[i], st))) return rc;
      const unsigned rb = (unsigned)((M + 7) / 8);
      split3_rows_kernel<<<rb, 256, 0, st>>>(x, W + n->norm_w, a3, M, D);
      if ((rc = launch_tc6(a3, n->tcw + n->tc_pre, W + n->pre_b, nullptr, z, M, Hn, D, tc::EPI_NONE, st))) return rc;
      if (trace) {
        CK(cudaMemcpyAsync(trace, z, (size_t)M * Hn * 4, cudaMemcpyDeviceToDevice, st));
        trace += (size_t)M * Hn;
      }
      split3_rows_kernel<<<rb, 256, 0, st>>>(z, nullptr, a3, M, Hn);
      for (long long m0 = 0; m0 < M; m0 += mc) {
        const long long rows = std::min<long long>(mc, M - m0);
        if ((rc = launch_tc6(a3 + m0 * 3 * Hn, n->tcw + S.tc_heads, W + S.head_b_folded, nullptr, logits, rows, S.count * V, Hn, tc::EPI_NONE, st)))
          return rc;
        argmax_heads_kernel<<<(unsigned)((rows * S.count + 7) / 8), 256, 0, st>>>(logits, rows, S.count, V, codes + m0 * Q + S.first, Q);
      }
      CK(cudaGetLastError());
      continue;
    }
    for (int i = 0; i < c.n_layers; ++i)
      if ((rc = ssm_block(W, n->blk[i], x, h, hid, lens, B, Tmax, D, c.kernel, c.dilation[i], false, st))) return rc;
    dense::DenseOp g{};
    g.A = x; g.W = W + n->pre_w; g.bias = W + n->pre_b; g.norm_w = W + n->norm_w; g.C = z; g.M = (int)M; g.N = Hn; g.K = D; g.ldc = Hn;
    g.epi = dense::EPI_BIAS;
    if ((rc = launch_dense(g, 1, st))) return rc;
    if (trace) {
      CK(cudaMemcpyAsync(trace, z, (size_t)M * Hn * 4, cudaMemcpyDeviceToDevice, st));
      trace += (size_t)M * Hn;
    }
    g = dense::DenseOp{};
    g.A = z; g.W = W + S.head_w; g.bias = W + S.head_b; g.a_add = W + S.head_id; g.M = (int)M; g.N = V; g.K = Hn; g.epi = dense::EPI_ARGMAX;
    g.amax_val = amax_v; g.amax_idx = amax_i; g.zW = (size_t)V * Hn; g.zBias = V; g.zAdd = Hn;
    const int parts = argmax_parts((int)M, V, S.count);
    if ((rc = launch_dense(g, S.count, st))) return rc;
    dense::argmax_finish_kernel<<<dim3((unsigned)((M + 127) / 128), S.count), 128, 0, st>>>(amax_v, amax_i, (int)M, parts, codes + S.first, Q);
    CK(cudaGetLastError());
  }
  return SOPRO_OK;
}

extern "C" {

int sopro_nar_set_graphs(sopro_nar_t* n, int enabled) {
  if (!n) return fail(SOPRO_ERR_INVALID, "null argument");
  n->graphs = enabled != 0;
  return SOPRO_OK;
}

int sopro_nar_refine(sopro_nar_t* n, const float* cond, int64_t cond_batch_stride, const int32_t* rvq1, const int32_t* lens, int B,
                     int Tmax, int32_t* codes, void* stream) {
  if (!n || !cond || !rvq1 || !codes) return fail(SOPRO_ERR_INVALID, "null argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  CK(cudaSetDevice(n->device));
  CK(cudaStreamIsCapturing(st, &cap));
  // one utterance's streaming window: replay the whole pass (113..217 launches) from a graph over static buffers
  if (!n->graphs || B != 1 || Tmax < 1 || Tmax > kNarGraphRows || lens || n->forced || n->trace_z || cap != cudaStreamCaptureStatusNone)
    return nar_refine_impl(n, cond, cond_batch_stride, rvq1, lens, B, Tmax, codes, stream);
  const sopro_nar_config_t& c = n->cfg;
  const int D = c.d_model, Q = c.n_codebooks;
  if (!n->g_cond) {
    CK(cudaMalloc(&n->g_cond, (size_t)kNarGraphRows * D * 4));
    CK(cudaMalloc(&n->g_rvq1, (size_t)kNarGraphRows * 4));
    CK(cudaMalloc(&n->g_codes, (size_t)kNarGraphRows * Q * 4));
  }
  // no graph-sized call may reallocate the workspace: reserve the largest graph shape of either arithmetic path once
  if (n->reserve_bytes == 0) {
    int rc = nar_refine_impl(n, nullptr, (int64_t)kNarGraphRows * D, nullptr, nullptr, 1, kNarGraphRows, nullptr, stream, true);
    if (!rc) rc = nar_refine_impl(n, nullptr, (int64_t)dense::kSkinnyRows * D, nullptr, nullptr, 1, dense::kSkinnyRows, nullptr, stream, true);
    if (rc) return rc;
  }
  const int tc = n->tc_mode;
  cudaGraphExec_t exec = nullptr;
  for (auto& r : n->replays)
    if (r.T == Tmax && r.tc == tc) exec = r.exec;
  if (!exec) {
    if (n->replays.size() >= 96) nar_drop_replays(n);
    // warm-up outside the capture (first use of a kernel sets function attributes), then capture on a private stream
    int rc = nar_refine_impl(n, cond, cond_batch_stride, rvq1, nullptr, 1, Tmax, codes, stream);
    if (rc) return rc;
    if (!n->cap_stream) CK(cudaStreamCreateWithFlags(&n->cap_stream, cudaStreamNonBlocking));
    CK(cudaStreamBeginCapture(n->cap_stream, cudaStreamCaptureModeThreadLocal));
    rc = nar_refine_impl(n, n->g_cond, (int64_t)Tmax * D, n->g_rvq1, nullptr, 1, Tmax, n->g_codes, n->cap_stream);
    cudaGraph_t graph = nullptr;
    cudaError_t ce = cudaStreamEndCapture(n->cap_stream, &graph);
    if (rc || ce != cudaSuccess) {  // this call already ran eagerly; just do not cache
      if (graph) cudaGraphDestroy(graph);
      cudaGetLastError();
      return SOPRO_OK;
    }
    ce = cudaGraphInstantiate(&exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ce == cudaSuccess) n->replays.push_back({Tmax, tc, exec});
    else cudaGetLastError();
    return SOPRO_OK;  // the eager warm-up produced this call's result
  }
  // replays from different caller streams share the static buffers: each waits for the previous one to finish
  if (!n->g_done) CK(cudaEventCreateWithFlags(&n->g_done, cudaEventDisableTiming));
  else CK(cudaStreamWaitEvent(st, n->g_done, 0));
  CK(cudaMemcpyAsync(n->g_cond, cond, (size_t)Tmax * D * 4, cudaMemcpyDeviceToDevice, st));
  CK(cudaMemcpyAsync(n->g_rvq1, rvq1, (size_t)Tmax * 4, cudaMemcpyDeviceToDevice, st));
  CK(cudaGraphLaunch(exec, st));
  CK(cudaMemcpyAsync(codes, n->g_codes, (size_t)Tmax * Q * 4, cudaMemcpyDeviceToDevice, st));
  CK(cudaEventRecord(n->g_done, st));
  return SOPRO_OK;
}

}  // extern "C"

// =================================================================================================
// Prefill: SoproTTSModel.prepare_conditioning (reference model.py:172-216) batched over utterances that share one
// prepared reference voice:
//   TextEncoder (nn/text.py:29-44): embedding + sinusoid -> mask -> n SSMLiteBlocks (non-causal) -> RMSNorm -> masked mean
//   base[t] = txt_pool + frame_pos[t]                                 (model.py:200-202)
//   SpeakerFiLM (nn/speaker.py:76-85): LayerNorm(base) * (1 + s*tanh(gamma)) + s*tanh(beta)
//   3 x RefXAttnBlock with cached K/V (nn/ref.py:57-108): q = Wq RMSNorm(x); softmax(q K^T / sqrt(dh)) V; nan_to_num;
//       a *= clamp(rms(x) / rms(a), 0, 10); x += gmax*tanh(gate) * Wo a
//   cond_ar = RMSNorm(x)                                              (model.py:208)
// cond_ar and txt_seq are INPUTS of the id-exact AR kernel, hence fp32 everywhere.
// =================================================================================================
namespace pstage {

// x[b][l] = (emb[id] + pos[l]) * (l < len[b])      (nn/text.py:31-35)
__global__ void __launch_bounds__(128) text_embed_kernel(const int* __restrict__ ids, const int* __restrict__ len,
                                                         const float* __restrict__ emb, const float* __restrict__ pos,
                                                         float* __restrict__ x, int Lmax, int D, int vocab) {
  const int l = blockIdx.x, b = blockIdx.y;
  const bool live = l < len[b];
  const int id = min(max(ids[(size_t)b * Lmax + l], 0), vocab - 1);
  for (int c = threadIdx.x; c < D; c += blockDim.x)
    x[((size_t)b * Lmax + l) * D + c] = live ? __ldg(emb + (size_t)id * D + c) + __ldg(pos + (size_t)l * D + c) : 0.f;
}

// pool[b][c] = sum_{l < len} x[b][l][c] / (len + 1e-6)      (nn/text.py:41-43)
__global__ void __launch_bounds__(128) mean_pool_kernel(const float* __restrict__ x, const int* __restrict__ len,
                                                        float* __restrict__ pool, int Lmax, int D) {
  const int b = blockIdx.x;
  const int L = len[b];
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    float s = 0.f;
    for (int l = 0; l < L; ++l) s += x[((size_t)b * Lmax + l) * D + c];
    pool[(size_t)b * D + c] = s / ((float)L + 1e-6f);
  }
}

// one warp per (b, t) row: base = pool[b] + frame_pos[t]; LayerNorm (eps 1e-5, biased variance) * w + bias;
// y = ln * (1 + s*tanh(gamma[v])) + s*tanh(beta[v]), v = voice_of[b]      (film rows [n_voices][2D])
__global__ void __launch_bounds__(256) film_rows_kernel(const float* __restrict__ pool, const float* __restrict__ fpos,
                                                        const float* __restrict__ ln_w, const float* __restrict__ ln_b,
                                                        const float* __restrict__ film, const int* __restrict__ voice_of, float strength,
                                                        float* __restrict__ y, long long rows, int T, int D) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const long long b = row / T, t = row - b * T;
  constexpr int kMaxPer = 16;
  float v[kMaxPer];
  float s = 0.f;
  int n = 0;
  for (int k = lane; k < D; k += 32, ++n) {
    v[n] = pool[b * D + k] + __ldg(fpos + t * D + k);
    s += v[n];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / (float)D;
  float var = 0.f;
  n = 0;
  for (int k = lane; k < D; k += 32, ++n) {
    const float d = v[n] - mean;
    var += d * d;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) var += __shfl_xor_sync(0xffffffffu, var, o);
  const float inv = 1.0f / sqrtf(var / (float)D + 1e-5f);
  const float* f = film + (size_t)voice_of[b] * 2 * D;
  n = 0;
  for (int k = lane; k < D; k += 32, ++n) {
    const float ln = (v[n] - mean) * inv * __ldg(ln_w + k) + __ldg(ln_b + k);
    y[row * D + k] = ln * (1.0f + strength * tanhf(f[k])) + strength * tanhf(f[D + k]);
  }
}

// Cached reference cross-attention core + RMS matching, one warp per query row (nn/ref.py:84-101):
//   per head: s_j = q.K_j / sqrt(dh); p = softmax(s); a = sum_j p_j V_j; nan_to_num
//   a *= clamp(rms(x) / rms(a), 0, 10) over the full row (both heads)
// Row `row` belongs to utterance b = row / T, which speaks voice v = voice_of[b]: K = Kv[v], V = Vv[v], both [H][Tr][dh]
// with Tr = tr_of[v].  A row's arithmetic depends on its voice alone (the loops run to that voice's Tr), so it equals
// the row of a launch with that one voice.  Shared memory per warp: q [D] | p [Tr_max] | a [D].
// kBlend: voice v is a blend whose K / V are its segments seg_first[v] .. seg_first[v + 1] - 1 one after another along
// the frame axis, segment s seg_len[s] frames with weight seg_w[s].  Each head runs the pass above over each segment
// alone (its own max, sum and nan_to_num) and accumulates a = sum_s seg_w[s] a_s in segment order; the RMS match runs
// once on that mix.  A voice of one segment with weight 1 gives the rows of kBlend = false bit for bit (a = 1 * a_0, and
// ssa sums the same squares in the same order).
template <bool kBlend>
__global__ void __launch_bounds__(256) ref_attn_kernel(const float* __restrict__ q, const float* __restrict__ x,
                                                       const int* __restrict__ voice_of, const int* __restrict__ tr_of,
                                                       const float* const* __restrict__ Kv, const float* const* __restrict__ Vv,
                                                       const int* __restrict__ seg_first, const int* __restrict__ seg_len,
                                                       const float* __restrict__ seg_w, float* __restrict__ out, long long rows,
                                                       int T, int D, int H, int Tr_max) {
  extern __shared__ float rsm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * 8 + warp;
  if (row >= rows) return;
  const int v = voice_of[row / T], Tr = tr_of[v];
  const float* __restrict__ Kc = Kv[v];
  const float* __restrict__ Vc = Vv[v];
  const int dh = D / H, Trp = (Tr_max + 3) & ~3;  // padded: the per-warp regions stay 16-byte aligned
  float* qs = rsm + (size_t)warp * (2 * D + Trp);
  float* ps = qs + D;
  float* as = ps + Trp;
  for (int k = lane; k < D; k += 32) qs[k] = q[row * D + k];
  __syncwarp();
  const float scale = 1.0f / sqrtf((float)dh);
  int s0 = 0, s1 = 1;
  if constexpr (kBlend) {
    s0 = seg_first[v];
    s1 = seg_first[v + 1];
  }
  float ssa = 0.f;
  for (int h = 0; h < H; ++h) {
    int off = 0;
    for (int g = s0; g < s1; ++g) {
      const int n = kBlend ? seg_len[g] : Tr;
      const float* Kh = Kc + ((size_t)h * Tr + off) * dh;
      const float* Vh = Vc + ((size_t)h * Tr + off) * dh;
      float mx = -INFINITY;
      for (int j = lane; j < n; j += 32) {
        const float* kr = Kh + (size_t)j * dh;
        float s = 0.f;
        for (int d = 0; d < dh; d += 4) {
          const float4 kk = __ldg(reinterpret_cast<const float4*>(kr + d));
          const float4 qq = *reinterpret_cast<const float4*>(qs + h * dh + d);
          s += kk.x * qq.x + kk.y * qq.y + kk.z * qq.z + kk.w * qq.w;
        }
        s *= scale;
        ps[j] = s;
        mx = fmaxf(mx, s);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      float sum = 0.f;
      for (int j = lane; j < n; j += 32) {
        const float e = expf(ps[j] - mx);
        ps[j] = e;
        sum += e;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      __syncwarp();
      const float inv = 1.0f / sum;
      for (int d = lane; d < dh; d += 32) {
        float o = 0.f;
        for (int j = 0; j < n; ++j) o += (ps[j] * inv) * __ldg(Vh + (size_t)j * dh + d);
        if (!isfinite(o)) o = 0.f;
        if constexpr (kBlend) {
          const float w = seg_w[g];
          as[h * dh + d] = g == s0 ? w * o : as[h * dh + d] + w * o;
        } else {
          as[h * dh + d] = o;
          ssa += o * o;
        }
      }
      __syncwarp();
      off += n;
    }
    if constexpr (kBlend) {
      for (int d = lane; d < dh; d += 32) {
        const float o = as[h * dh + d];
        ssa += o * o;
      }
    }
  }
  float ssx = 0.f;
  for (int k = lane; k < D; k += 32) {
    const float xv = x[row * D + k];
    ssx += xv * xv;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ssa += __shfl_xor_sync(0xffffffffu, ssa, o);
    ssx += __shfl_xor_sync(0xffffffffu, ssx, o);
  }
  const float rx = sqrtf(ssx / (float)D + 1e-6f), ra = sqrtf(ssa / (float)D + 1e-6f);
  const float sc = fminf(fmaxf(rx / ra, 0.0f), 10.0f);
  for (int k = lane; k < D; k += 32) out[row * D + k] = as[k] * sc;
}

}  // namespace pstage

struct sopro_prefill {
  int device = 0;
  sopro_prefill_config_t cfg{};
  float* dev = nullptr;
  size_t n_floats = 0;
  size_t text_emb = 0, text_pos = 0, frame_pos = 0, text_norm_w = 0, film_w0 = 0, film_b0 = 0, film_w2 = 0, film_b2 = 0, film_ln_w = 0,
         film_ln_b = 0, cond_norm_w = 0;
  BlockOff blk[SOPRO_MAX_SSM_LAYERS]{};
  struct Ref {
    size_t nq_w, q_w, o_w;
    float gate_eff;
  } ref[SOPRO_PREFILL_MAX_REF_LAYERS]{};
  float* ws = nullptr;
  size_t ws_bytes = 0;
};

extern "C" {

int sopro_prefill_create(const sopro_prefill_config_t* cfg, const sopro_prefill_weights_t* w, int device, sopro_prefill_t** out) {
  if (!cfg || !w || !out) return fail(SOPRO_ERR_INVALID, "null argument");
  *out = nullptr;
  const int rc = open_device(device, "the prefill");
  if (rc != SOPRO_OK) return rc;
  const int D = cfg->d_model, NL = cfg->n_layers_text, k = cfg->text_kernel, SV = cfg->sv_dim, RL = cfg->ref_layers, H = cfg->ref_heads;
  if (D < 32 || D > 512 || D % 16 || NL < 0 || NL > SOPRO_MAX_SSM_LAYERS || k < 1 || k > 64 || SV < 16 || SV % 16 || RL < 0 ||
      RL > SOPRO_PREFILL_MAX_REF_LAYERS || H < 1 || D % H || (D / H) % 4 || cfg->text_vocab < 1 || cfg->max_text_len < 1 || cfg->max_frames_pos < 1)
    return fail(SOPRO_ERR_INVALID, "unsupported prefill geometry");
  for (int i = 0; i < NL; ++i)
    if (!block_ok(w->text_block[i])) return fail(SOPRO_ERR_INVALID, "text block %d: null weight", i);
  if (!w->text_emb || !w->text_pos || !w->frame_pos || !w->text_norm_w || !w->film_w0 || !w->film_b0 || !w->film_w2 || !w->film_b2 ||
      !w->film_norm_w || !w->film_norm_b || !w->cond_norm_w)
    return fail(SOPRO_ERR_INVALID, "prefill: null weight pointer");
  for (int i = 0; i < RL; ++i)
    if (!w->ref_layer[i].nq_w || !w->ref_layer[i].q_w || !w->ref_layer[i].o_w) return fail(SOPRO_ERR_INVALID, "ref layer %d: null weight", i);
  sopro_prefill* p = new sopro_prefill();
  p->device = device;
  p->cfg = *cfg;
  FArena A;
  p->text_emb = A.add(w->text_emb, (size_t)cfg->text_vocab * D);
  p->text_pos = A.add(w->text_pos, (size_t)cfg->max_text_len * D);
  p->frame_pos = A.add(w->frame_pos, (size_t)cfg->max_frames_pos * D);
  for (int i = 0; i < NL; ++i) add_block(A, w->text_block[i], D, k, &p->blk[i]);
  p->text_norm_w = A.add(w->text_norm_w, D);
  p->film_w0 = A.add(w->film_w0, (size_t)D * SV);
  p->film_b0 = A.add(w->film_b0, D);
  p->film_w2 = A.add(w->film_w2, (size_t)2 * D * D);
  p->film_b2 = A.add(w->film_b2, 2 * D);
  p->film_ln_w = A.add(w->film_norm_w, D);
  p->film_ln_b = A.add(w->film_norm_b, D);
  for (int i = 0; i < RL; ++i) {
    p->ref[i].nq_w = A.add(w->ref_layer[i].nq_w, D);
    p->ref[i].q_w = A.add(w->ref_layer[i].q_w, (size_t)D * D);
    p->ref[i].o_w = A.add(w->ref_layer[i].o_w, (size_t)D * D);
    p->ref[i].gate_eff = cfg->ref_gmax * tanhf(w->ref_layer[i].gate);
  }
  p->cond_norm_w = A.add(w->cond_norm_w, D);
  p->n_floats = A.host.size();
  cudaError_t err = cudaMalloc(&p->dev, p->n_floats * 4);
  if (err == cudaSuccess) err = cudaMemcpy(p->dev, A.host.data(), p->n_floats * 4, cudaMemcpyHostToDevice);
  if (err != cudaSuccess) {
    if (p->dev) cudaFree(p->dev);
    delete p;
    return fail(SOPRO_ERR_CUDA, "prefill weight upload failed: %s", cudaGetErrorString(err));
  }
  *out = p;
  return SOPRO_OK;
}

int sopro_prefill_destroy(sopro_prefill_t* p) {
  if (!p) return SOPRO_OK;
  cudaSetDevice(p->device);
  cudaFree(p->dev);
  cudaFree(p->ws);
  delete p;
  return SOPRO_OK;
}

}  // extern "C"

namespace pstage {

// The prefill of B texts over a table of n_voices voices: text b speaks voice voice_of[b] (host), voice v has speaker
// vector sv[v] (device [n_voices][SV]), tr[v] reference frames (host) and, for reference layer i, cached K / V at
// ref_k[i * n_voices + v] / ref_v[...] (host arrays of device pointers).  The one-voice call is n_voices = 1.
// n_seg != nullptr (sopro_prefill_run_blends, checked there): voice v is a blend of n_seg[v] segments, whose frames and
// weights follow those of voices 0 .. v-1 in seg_frames / seg_w (host); the reference attention runs the blend kernel.
int prefill_core(sopro_prefill* p, const int32_t* text_ids, const int32_t* text_len, int B, int Lmax, int n_voices,
                 const int32_t* voice_of, const float* sv, const int32_t* tr, const float* const* ref_k, const float* const* ref_v,
                 float style_strength, int n_frames, float* txt_seq, float* txt_pool, float* cond_ar, cudaStream_t st,
                 const int32_t* n_seg = nullptr, const int32_t* seg_frames = nullptr, const float* seg_w = nullptr) {
  if (!p || !text_ids || !text_len || !sv || !txt_seq || !txt_pool || !cond_ar || !voice_of) return fail(SOPRO_ERR_INVALID, "null argument");
  const sopro_prefill_config_t& c = p->cfg;
  const int D = c.d_model, SV = c.sv_dim, H = c.ref_heads, RL = c.ref_layers;
  if (B < 1 || Lmax < 1 || Lmax > c.max_text_len || n_frames < 1 || n_frames > c.max_frames_pos || (long long)B * n_frames > 0x3fffffffLL)
    return fail(SOPRO_ERR_INVALID, "bad B=%d Lmax=%d (max %d) n_frames=%d (max %d)", B, Lmax, c.max_text_len, n_frames, c.max_frames_pos);
  if (n_voices < 1 || n_voices > B) return fail(SOPRO_ERR_INVALID, "n_voices=%d outside [1, B=%d]", n_voices, B);
  for (int b = 0; b < B; ++b)
    if (voice_of[b] < 0 || voice_of[b] >= n_voices) return fail(SOPRO_ERR_INVALID, "voice_of[%d]=%d outside [0, %d)", b, voice_of[b], n_voices);
  int Tr_max = 1;
  if (RL > 0) {
    if (!ref_k || !ref_v || !tr) return fail(SOPRO_ERR_INVALID, "reference K/V missing");
    for (int v = 0; v < n_voices; ++v) {
      if (tr[v] < 1 || tr[v] > 4096) return fail(SOPRO_ERR_INVALID, "reference K/V missing or Tr=%d out of range", tr[v]);
      Tr_max = std::max(Tr_max, (int)tr[v]);
      for (int i = 0; i < RL; ++i)
        if (!ref_k[(size_t)i * n_voices + v] || !ref_v[(size_t)i * n_voices + v])
          return fail(SOPRO_ERR_INVALID, "reference K/V of layer %d, voice %d is null", i, v);
    }
  }
  CK(cudaSetDevice(p->device));
  const long long Mt = (long long)B * Lmax, Mc = (long long)B * n_frames;
  auto al = [](size_t x) { return (x + 63) / 64 * 64; };
  const size_t rows = (size_t)std::max(Mt, Mc);
  // the voice table: K pointers [RL][n_voices] | V pointers [RL][n_voices] | tr [n_voices] | voice_of [B], and for a
  // blend launch | seg_first [n_voices + 1] | seg_len [S] | seg_w [S] (float)
  size_t n_segs = 0;
  for (int v = 0; n_seg && v < n_voices; ++v) n_segs += (size_t)n_seg[v];
  const size_t seg_bytes = n_seg ? ((size_t)n_voices + 1 + 2 * n_segs) * sizeof(int) : 0;
  const size_t n_ptr = (size_t)RL * n_voices,
               tab_bytes = 2 * n_ptr * sizeof(void*) + ((size_t)n_voices + B) * sizeof(int) + seg_bytes;
  const size_t need = (al(rows * D) * 3 + al(rows * 4 * D) + al((size_t)B * D) + al((size_t)B * 2 * D) + al((tab_bytes + 3) / 4)) * 4;
  if (p->ws_bytes < need) {
    CK(cudaStreamSynchronize(st));
    cudaFree(p->ws);
    p->ws = nullptr;
    p->ws_bytes = 0;
    cudaError_t e = cudaMalloc(&p->ws, need);
    if (e != cudaSuccess) return fail(SOPRO_ERR_CUDA, "prefill workspace %zu MB: %s", need >> 20, cudaGetErrorString(e));
    p->ws_bytes = need;
  }
  float* x = p->ws;
  float* h = x + al(rows * D);
  float* q = h + al(rows * D);
  float* hid = q + al(rows * D);
  float* fmid = hid + al(rows * 4 * D);           // [n_voices][D] FiLM hidden
  float* film = fmid + al((size_t)B * D);         // [n_voices][2D]
  char* tab = reinterpret_cast<char*>(film + al((size_t)B * 2 * D));
  const float* const* kv_dev = reinterpret_cast<const float* const*>(tab);
  const int* tr_dev = reinterpret_cast<const int*>(tab + 2 * n_ptr * sizeof(void*));
  const int* voice_dev = tr_dev + n_voices;
  const int* seg_first_dev = voice_dev + B;
  const int* seg_len_dev = seg_first_dev + n_voices + 1;
  const float* seg_w_dev = reinterpret_cast<const float*>(seg_len_dev + n_segs);
  {
    // one copy from pageable memory: cudaMemcpyAsync has staged the bytes when it returns, so `host` may go
    std::vector<char> host(tab_bytes);
    if (n_ptr) {
      memcpy(host.data(), ref_k, n_ptr * sizeof(void*));
      memcpy(host.data() + n_ptr * sizeof(void*), ref_v, n_ptr * sizeof(void*));
    }
    std::vector<int> tr_h(n_voices, 1);
    if (RL > 0) std::copy(tr, tr + n_voices, tr_h.begin());
    memcpy(host.data() + 2 * n_ptr * sizeof(void*), tr_h.data(), (size_t)n_voices * sizeof(int));
    memcpy(host.data() + 2 * n_ptr * sizeof(void*) + (size_t)n_voices * sizeof(int), voice_of, (size_t)B * sizeof(int));
    if (n_seg) {
      int* first = reinterpret_cast<int*>(host.data() + 2 * n_ptr * sizeof(void*) + ((size_t)n_voices + B) * sizeof(int));
      first[0] = 0;
      for (int v = 0; v < n_voices; ++v) first[v + 1] = first[v] + n_seg[v];
      memcpy(first + n_voices + 1, seg_frames, n_segs * sizeof(int));
      memcpy(first + n_voices + 1 + n_segs, seg_w, n_segs * sizeof(float));
    }
    CK(cudaMemcpyAsync(tab, host.data(), tab_bytes, cudaMemcpyHostToDevice, st));
  }
  const float* W = p->dev;
  int rc;
  // ---- text encoder
  text_embed_kernel<<<dim3(Lmax, B), 128, 0, st>>>(text_ids, text_len, W + p->text_emb, W + p->text_pos, x, Lmax, D, c.text_vocab);
  CK(cudaGetLastError());
  for (int i = 0; i < c.n_layers_text; ++i)
    if ((rc = ssm_block(W, p->blk[i], x, h, hid, text_len, B, Lmax, D, c.text_kernel, 1, false, st))) return rc;
  dense::rmsnorm_rows_kernel<<<(unsigned)((Mt + 7) / 8), 256, 0, st>>>(x, W + p->text_norm_w, nullptr, nullptr, txt_seq, Mt, D);
  CK(cudaGetLastError());
  mean_pool_kernel<<<B, 128, 0, st>>>(txt_seq, text_len, txt_pool, Lmax, D);
  CK(cudaGetLastError());
  // ---- FiLM parameters of every voice, on the skinny kernel whatever n_voices is: each voice's row then has the
  // reduction order of a one-voice (M = 1) launch (the tile kernel, taken above 16 rows by default, sums in another)
  dense::DenseOp g{};
  g.A = sv; g.W = W + p->film_w0; g.bias = W + p->film_b0; g.C = fmid; g.M = n_voices; g.N = D; g.K = SV; g.ldc = D; g.epi = dense::EPI_GELU;
  if ((rc = launch_dense(g, 1, st, 16))) return rc;
  g = dense::DenseOp{};
  g.A = fmid; g.W = W + p->film_w2; g.bias = W + p->film_b2; g.C = film; g.M = n_voices; g.N = 2 * D; g.K = D; g.ldc = 2 * D; g.epi = dense::EPI_BIAS;
  if ((rc = launch_dense(g, 1, st, 16))) return rc;
  film_rows_kernel<<<(unsigned)((Mc + 7) / 8), 256, 0, st>>>(txt_pool, W + p->frame_pos, W + p->film_ln_w, W + p->film_ln_b, film, voice_dev,
                                                            style_strength, x, Mc, n_frames, D);
  CK(cudaGetLastError());
  // ---- reference cross-attention stack
  const size_t rsmem = (size_t)8 * (2 * D + ((Tr_max + 3) & ~3)) * 4;
  if (RL > 0 && rsmem > 48 * 1024) {
    static unsigned long long attr_done = 0, attr_blend_done = 0;  // per device, like every function attribute
    if (!n_seg && tc::attr_needed(attr_done))
      CK(cudaFuncSetAttribute(ref_attn_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    if (n_seg && tc::attr_needed(attr_blend_done))
      CK(cudaFuncSetAttribute(ref_attn_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  }
  for (int i = 0; i < RL; ++i) {
    g = dense::DenseOp{};
    g.A = x; g.W = W + p->ref[i].q_w; g.norm_w = W + p->ref[i].nq_w; g.C = q; g.M = (int)Mc; g.N = D; g.K = D; g.ldc = D; g.epi = dense::EPI_BIAS;
    if ((rc = launch_dense(g, 1, st))) return rc;
    const float* const* Ki = kv_dev + (size_t)i * n_voices;
    const float* const* Vi = kv_dev + n_ptr + (size_t)i * n_voices;
    if (n_seg)
      ref_attn_kernel<true><<<(unsigned)((Mc + 7) / 8), 256, rsmem, st>>>(q, x, voice_dev, tr_dev, Ki, Vi, seg_first_dev, seg_len_dev,
                                                                          seg_w_dev, h, Mc, n_frames, D, H, Tr_max);
    else
      ref_attn_kernel<false><<<(unsigned)((Mc + 7) / 8), 256, rsmem, st>>>(q, x, voice_dev, tr_dev, Ki, Vi, nullptr, nullptr, nullptr,
                                                                           h, Mc, n_frames, D, H, Tr_max);
    CK(cudaGetLastError());
    g = dense::DenseOp{};
    g.A = h; g.W = W + p->ref[i].o_w; g.R = x; g.C = x; g.M = (int)Mc; g.N = D; g.K = D; g.ldc = D; g.epi = dense::EPI_RES_GATE;
    g.gate = p->ref[i].gate_eff;
    if ((rc = launch_dense(g, 1, st))) return rc;
  }
  dense::rmsnorm_rows_kernel<<<(unsigned)((Mc + 7) / 8), 256, 0, st>>>(x, W + p->cond_norm_w, nullptr, nullptr, cond_ar, Mc, D);
  CK(cudaGetLastError());
  return SOPRO_OK;
}

}  // namespace pstage

extern "C" {

int sopro_prefill_run(sopro_prefill_t* p, const int32_t* text_ids, const int32_t* text_len, int B, int Lmax, const float* sv,
                      int sv_shared, const float* const* ref_k, const float* const* ref_v, int Tr, float style_strength, int n_frames,
                      float* txt_seq, float* txt_pool, float* cond_ar, void* stream) {
  if (!p || !text_ids || !text_len || !sv || !txt_seq || !txt_pool || !cond_ar) return fail(SOPRO_ERR_INVALID, "null argument");
  // one voice (sv_shared), or one speaker vector per text over the same K / V: a table of B voices that differ in sv only
  const int nb = std::max(B, 1), nv = sv_shared ? 1 : nb, RL = p->cfg.ref_layers;
  std::vector<int32_t> voice_of(nb), tr(nv, Tr);
  for (int b = 0; b < nb; ++b) voice_of[b] = sv_shared ? 0 : b;
  std::vector<const float*> kp((size_t)RL * nv), vp((size_t)RL * nv);
  const bool kv = ref_k && ref_v;
  for (int i = 0; kv && i < RL; ++i)
    for (int v = 0; v < nv; ++v) {
      kp[(size_t)i * nv + v] = ref_k[i];
      vp[(size_t)i * nv + v] = ref_v[i];
    }
  return pstage::prefill_core(p, text_ids, text_len, B, Lmax, nv, voice_of.data(), sv, tr.data(), kv ? kp.data() : nullptr,
                              kv ? vp.data() : nullptr, style_strength, n_frames, txt_seq, txt_pool, cond_ar,
                              reinterpret_cast<cudaStream_t>(stream));
}

int sopro_prefill_run_voices(sopro_prefill_t* p, const int32_t* text_ids, const int32_t* text_len, int B, int Lmax, int n_voices,
                             const int32_t* voice_of, const float* sv, const int32_t* tr, const float* const* ref_k,
                             const float* const* ref_v, float style_strength, int n_frames, float* txt_seq, float* txt_pool,
                             float* cond_ar, void* stream) {
  return pstage::prefill_core(p, text_ids, text_len, B, Lmax, n_voices, voice_of, sv, tr, ref_k, ref_v, style_strength, n_frames, txt_seq,
                              txt_pool, cond_ar, reinterpret_cast<cudaStream_t>(stream));
}

int sopro_prefill_run_blends(sopro_prefill_t* p, const int32_t* text_ids, const int32_t* text_len, int B, int Lmax, int n_voices,
                             const int32_t* voice_of, const float* sv, const int32_t* tr, const float* const* ref_k,
                             const float* const* ref_v, const int32_t* n_seg, const int32_t* seg_frames, const float* seg_w,
                             float style_strength, int n_frames, float* txt_seq, float* txt_pool, float* cond_ar, void* stream) {
  if (!p || !n_seg || !seg_frames || !seg_w || !tr) return fail(SOPRO_ERR_INVALID, "null argument");
  if (n_voices < 1 || n_voices > B) return fail(SOPRO_ERR_INVALID, "n_voices=%d outside [1, B=%d]", n_voices, B);
  size_t s = 0;
  for (int v = 0; v < n_voices; ++v) {
    if (n_seg[v] < 1 || n_seg[v] > SOPRO_PREFILL_MAX_BLEND_SEGMENTS)
      return fail(SOPRO_ERR_INVALID, "n_seg[%d]=%d outside [1, %d]", v, n_seg[v], SOPRO_PREFILL_MAX_BLEND_SEGMENTS);
    long long frames = 0;
    for (int k = 0; k < n_seg[v]; ++k, ++s) {
      if (seg_frames[s] < 1) return fail(SOPRO_ERR_INVALID, "voice %d, segment %d: %d frames", v, k, seg_frames[s]);
      if (!std::isfinite(seg_w[s]) || !(seg_w[s] > 0.f)) return fail(SOPRO_ERR_INVALID, "voice %d, segment %d: weight %g", v, k, seg_w[s]);
      frames += seg_frames[s];
    }
    if (frames != tr[v]) return fail(SOPRO_ERR_INVALID, "voice %d: segments of %lld frames, tr=%d", v, frames, tr[v]);
  }
  return pstage::prefill_core(p, text_ids, text_len, B, Lmax, n_voices, voice_of, sv, tr, ref_k, ref_v, style_strength, n_frames, txt_seq,
                              txt_pool, cond_ar, reinterpret_cast<cudaStream_t>(stream), n_seg, seg_frames, seg_w);
}

}  // extern "C"

// =================================================================================================
// Reference preparation: SoproTTSModel.prepare_reference (reference model.py:152-170), once per voice, from the voice's
// codes [Tr][Q]:
//   Token2SV (nn/speaker.py:12-61): softmax(cb_weights)-weighted sum of per-codebook embeddings -> 2 x (depthwise conv k7,
//       non-causal, GELU) -> AttentiveStatsPool (nn/blocks.py:165-188: softmax_t(w2 . tanh(W0 h + b0) + b2), weighted mean
//       and std) -> Linear -> L2 normalise                                               -> sv_ref [sv_dim]
//   _encode_reference_seq (model.py:136-150): softmax(ref_cb_weights)-weighted sum of cb_embed rows -> SSMLiteBlocks
//       (non-causal) -> RMSNorm                                                           -> ref_seq [Tr][D]
//   RefXAttnStack.build_kv_caches (nn/ref.py): per layer K = Wk RMSNorm_kv(ref_seq), V = Wv RMSNorm_kv(ref_seq), stored
//       [H][Tr][D/H]                                                                      -> the prefill engine's ref_k / ref_v
// fp32 (everything here feeds cond_ar, an input of the id-exact AR kernel).
// =================================================================================================
namespace pstage {

// Token2SV's batch of B sequences is PACKED: rows[2b] = the first row of sequence b in the [frames][d] buffers,
// rows[2b+1] = its length.  Every kernel then runs over valid frames only, and the pooling projection is one dense
// launch over them (a padded layout would compute every padding frame of a ragged batch: one 4096-frame take beside
// fifteen 40-frame ones would be 16 x 4096 rows instead of 4696).

// out[r][c] = sum_q w[q] * emb[(q*V + tok[b][t][q]) * dim + c], q ascending (the reference's loop order); a code outside
// [0, V) is clamped and flagged.  Frame t = blockIdx.x of sequence b = blockIdx.y, tok [B][T][Q]; rows null: r = t
// (one sequence), otherwise r = rows[2b] + t and frames past rows[2b+1] are skipped
__global__ void __launch_bounds__(128) codes_mix_kernel(const int* __restrict__ tok, const float* __restrict__ emb,
                                                        const float* __restrict__ w, float* __restrict__ out, int Q, int V, int dim,
                                                        int* __restrict__ bad, const int* __restrict__ rows = nullptr, int T = 0) {
  const int t = blockIdx.x, b = blockIdx.y;
  size_t r = t;
  if (rows) {
    if (t >= rows[2 * b + 1]) return;
    r = (size_t)rows[2 * b] + t;
    tok += (size_t)b * T * Q;
  }
  out += r * dim;
  extern __shared__ int ids[];
  for (int q = threadIdx.x; q < Q; q += blockDim.x) {
    int id = tok[(size_t)t * Q + q];
    if (id < 0 || id >= V) {
      atomicExch(bad, 1);
      id = min(max(id, 0), V - 1);
    }
    ids[q] = id;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < dim; c += blockDim.x) {
    float acc = 0.f;
    for (int q = 0; q < Q; ++q) acc = __fadd_rn(acc, __fmul_rn(__ldg(w + q), __ldg(emb + ((size_t)q * V + ids[q]) * dim + c)));
    out[c] = acc;
  }
}

// y[t][c] = gelu(bias[c] + sum_j x[t + j - left][c] * w[c][j])   (DepthwiseConv1d non-causal + GELU, zero padding at
// both ends of each sequence): frame t = blockIdx.x of packed sequence b = blockIdx.y
__global__ void __launch_bounds__(128) dwconv_gelu_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                          const float* __restrict__ bias, float* __restrict__ y,
                                                          const int* __restrict__ rows, int D, int k, int left) {
  const int t = blockIdx.x, b = blockIdx.y, T = rows[2 * b + 1];
  if (t >= T) return;
  const size_t base = rows[2 * b];
  x += base * D;
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    float acc = 0.f;
    for (int j = 0; j < k; ++j) {
      const int r = t + j - left;
      if (r >= 0 && r < T) acc = fmaf(x[(size_t)r * D + c], __ldg(w + c * k + j), acc);
    }
    y[(base + t) * D + c] = dense::gelu_erf(acc + __ldg(bias + c));
  }
}

// AttentiveStatsPool tail: u [T][D] = W0 h + b0 (from the dense kernel); logits[t] = w2 . tanh(u[t]) + b2; a = softmax_t;
// mu = sum_t a h; std = sqrt(max(sum_t a (h - mu)^2, 1e-6)); out = [mu | std]  (one CTA per packed sequence
// b = blockIdx.x, out [B][2D]; T floats of shared memory)
__global__ void __launch_bounds__(256) attn_stats_pool_kernel(const float* __restrict__ u, const float* __restrict__ h,
                                                              const float* __restrict__ w2, float b2, float* __restrict__ out,
                                                              const int* __restrict__ rows, int D) {
  extern __shared__ float a[];
  __shared__ float red[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x, T = rows[2 * b + 1];
  u += (size_t)rows[2 * b] * D;
  h += (size_t)rows[2 * b] * D;
  out += (size_t)b * 2 * D;
  for (int t = warp; t < T; t += 8) {
    float s = 0.f;
    for (int c = lane; c < D; c += 32) s = fmaf(__ldg(w2 + c), tanhf(u[(size_t)t * D + c]), s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) a[t] = s + b2;
  }
  __syncthreads();
  float mx = -INFINITY;
  for (int t = threadIdx.x; t < T; t += 256) mx = fmaxf(mx, a[t]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  mx = red[0];
  for (int i = 1; i < 8; ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int t = threadIdx.x; t < T; t += 256) {
    const float e = expf(a[t] - mx);
    a[t] = e;
    sum += e;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if (lane == 0) red[warp] = sum;
  __syncthreads();
  sum = 0.f;
  for (int i = 0; i < 8; ++i) sum += red[i];
  const float inv = 1.0f / sum;
  for (int c = threadIdx.x; c < D; c += 256) {
    float mu = 0.f;
    for (int t = 0; t < T; ++t) mu = fmaf(h[(size_t)t * D + c], a[t] * inv, mu);
    float var = 0.f;
    for (int t = 0; t < T; ++t) {
      const float d = h[(size_t)t * D + c] - mu;
      var = fmaf(a[t] * inv, d * d, var);
    }
    out[c] = mu;
    out[D + c] = sqrtf(fmaxf(var, 1e-6f));
  }
}

// F.normalize(e, eps): e / max(||e||, eps), one warp per row b = blockIdx.x of e / out [B][n]; with ref, also
// cos[b] = out[b] . ref[b * ref_stride .. + n) (the rows and ref are unit vectors, so this is their cosine; ref_stride 0:
// every row against the one vector ref [n])
__global__ void l2_normalize_kernel(const float* __restrict__ e, float* __restrict__ out, int n, float eps,
                                    const float* __restrict__ ref, int ref_stride, float* __restrict__ cos) {
  const int lane = threadIdx.x;
  e += (size_t)blockIdx.x * n;
  out += (size_t)blockIdx.x * n;
  if (ref) ref += (size_t)blockIdx.x * ref_stride;
  float s = 0.f;
  for (int i = lane; i < n; i += 32) s = fmaf(e[i], e[i], s);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float d = fmaxf(sqrtf(s), eps);
  float c = 0.f;
  for (int i = lane; i < n; i += 32) {
    const float v = e[i] / d;
    out[i] = v;
    if (ref) c = fmaf(v, __ldg(ref + i), c);
  }
  if (!ref) return;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if (lane == 0) cos[blockIdx.x] = c;
}

// [T][H*Dh] -> [H][T][Dh]
__global__ void heads_major_kernel(const float* __restrict__ x, float* __restrict__ y, int T, int H, int Dh) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)T * H * Dh) return;
  const int d = (int)(i % Dh), t = (int)((i / Dh) % T), h = (int)(i / ((long long)Dh * T));
  y[i] = x[(size_t)t * H * Dh + h * Dh + d];
}

}  // namespace pstage

struct sopro_refprep {
  int device = 0;
  sopro_refprep_config_t cfg{};
  float* dev = nullptr;
  size_t sv_emb = 0, sv_w = 0, dw0_w = 0, dw0_b = 0, dw1_w = 0, dw1_b = 0, pool_w0 = 0, pool_b0 = 0, pool_w2 = 0, proj_w = 0, proj_b = 0,
         cb_embed = 0, ref_w = 0, ref_norm_w = 0;
  float pool_b2 = 0.f;
  BlockOff blk[SOPRO_MAX_SSM_LAYERS]{};
  struct Layer {
    size_t nkv_w, k_w, v_w;
  } layer[SOPRO_PREFILL_MAX_REF_LAYERS]{};
  float* ws = nullptr;
  size_t ws_bytes = 0;
  int* bad = nullptr;
};

namespace pstage {

size_t al64(size_t x) { return (x + 63) / 64 * 64; }

// the workspace holds at least `need` bytes (a grown one replaces the old once the stream is done with it)
int grow_ws(sopro_refprep* p, size_t need, cudaStream_t st) {
  if (p->ws_bytes >= need) return SOPRO_OK;
  CK(cudaStreamSynchronize(st));
  cudaFree(p->ws);
  p->ws = nullptr;
  p->ws_bytes = 0;
  cudaError_t e = cudaMalloc(&p->ws, need);
  if (e != cudaSuccess) return fail(SOPRO_ERR_CUDA, "reference-preparation workspace: %s", cudaGetErrorString(e));
  p->ws_bytes = need;
  return SOPRO_OK;
}

// Token2SV of B code sequences, tokens [B][Tmax][Q], lens[b] (host) frames each -> sv [B][SV], and cos [B] when ref_sv
// is given (row b against ref_sv + b * ref_stride).  x / h / q: [sum lens][d] each, stats [B][2d], e [B][SV], rows: 2B ints (device).  A row's result does not
// depend on the batch: the convolutions and the pooling stay inside each sequence, and both matmuls run each row in the
// reduction order it gets alone -- a sequence of <= 16 frames (and the B-row projection) on the skinny kernel in blocks
// of 16 rows, longer sequences on the tile kernel, whose order does not depend on M.  So the long sequences are packed
// first, the short ones after them, and the pooling matmul is one launch per kind.
int token2sv(sopro_refprep* p, const int32_t* tokens, int B, int Tmax, const int32_t* lens, float* sv, const float* ref_sv, int ref_stride,
             float* cos, float* x, float* h, float* q, float* stats, float* e, int* rows, cudaStream_t st) {
  const sopro_refprep_config_t& c = p->cfg;
  const int d = c.sv_embed_dim, SV = c.sv_dim, Q = c.n_codebooks, V = c.codebook_size;
  std::vector<int> host(2 * (size_t)B);
  int n_long = 0, total = 0;
  for (int pass = 0; pass < 2; ++pass) {
    for (int b = 0; b < B; ++b) {
      if ((lens[b] > dense::kSkinnyRows) != (pass == 0)) continue;
      host[2 * b] = total;
      host[2 * b + 1] = lens[b];
      total += lens[b];
    }
    if (pass == 0) n_long = total;
  }
  CK(cudaMemcpyAsync(rows, host.data(), host.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  const float* W = p->dev;
  const dim3 frames(Tmax, B);
  codes_mix_kernel<<<frames, 128, Q * sizeof(int), st>>>(tokens, W + p->sv_emb, W + p->sv_w, x, Q, V, d, p->bad, rows, Tmax);
  CK(cudaGetLastError());
  const int left = (c.sv_kernel - 1) / 2;
  dwconv_gelu_kernel<<<frames, 128, 0, st>>>(x, W + p->dw0_w, W + p->dw0_b, h, rows, d, c.sv_kernel, left);
  dwconv_gelu_kernel<<<frames, 128, 0, st>>>(h, W + p->dw1_w, W + p->dw1_b, x, rows, d, c.sv_kernel, left);
  CK(cudaGetLastError());
  int rc;
  dense::DenseOp g{};
  g.W = W + p->pool_w0; g.bias = W + p->pool_b0; g.N = d; g.K = d; g.ldc = d; g.epi = dense::EPI_BIAS;
  if (n_long > 0) {  // > 16 rows: the tile kernel
    g.A = x; g.C = q; g.M = n_long;
    if ((rc = launch_dense(g, 1, st))) return rc;
  }
  if (total > n_long) {
    g.A = x + (size_t)n_long * d; g.C = q + (size_t)n_long * d; g.M = total - n_long;
    if ((rc = launch_dense(g, 1, st, 16))) return rc;
  }
  attn_stats_pool_kernel<<<B, 256, (size_t)Tmax * 4, st>>>(q, x, W + p->pool_w2, p->pool_b2, stats, rows, d);
  CK(cudaGetLastError());
  g = dense::DenseOp{};
  g.A = stats; g.W = W + p->proj_w; g.bias = W + p->proj_b; g.C = e; g.M = B; g.N = SV; g.K = 2 * d; g.ldc = SV; g.epi = dense::EPI_BIAS;
  if ((rc = launch_dense(g, 1, st, 16))) return rc;
  l2_normalize_kernel<<<B, 32, 0, st>>>(e, sv, SV, 1e-6f, ref_sv, ref_stride, cos);
  CK(cudaGetLastError());
  return SOPRO_OK;
}

}  // namespace pstage

extern "C" {

int sopro_refprep_create(const sopro_refprep_config_t* cfg, const sopro_refprep_weights_t* w, int device, sopro_refprep_t** out) {
  if (!cfg || !w || !out) return fail(SOPRO_ERR_INVALID, "null argument");
  *out = nullptr;
  const int rc = open_device(device, "the reference preparation");
  if (rc != SOPRO_OK) return rc;
  const int D = cfg->d_model, d = cfg->sv_embed_dim, SV = cfg->sv_dim, Q = cfg->n_codebooks, V = cfg->codebook_size, NL = cfg->ref_enc_layers,
            RL = cfg->ref_layers, H = cfg->ref_heads;
  if (D < 32 || D > 512 || D % 16 || d < 16 || d % 16 || SV < 16 || SV % 16 || Q < 1 || Q > 64 || V < 1 || NL < 0 || NL > SOPRO_MAX_SSM_LAYERS ||
      RL < 0 || RL > SOPRO_PREFILL_MAX_REF_LAYERS || H < 1 || D % H || cfg->sv_kernel < 1 || cfg->sv_kernel > 64 || cfg->ref_enc_kernel < 1 ||
      cfg->ref_enc_kernel > 64)
    return fail(SOPRO_ERR_INVALID, "unsupported reference-preparation geometry");
  if (!w->sv_emb || !w->sv_cb_weights || !w->sv_dw0_w || !w->sv_dw0_b || !w->sv_dw1_w || !w->sv_dw1_b || !w->pool_w0 || !w->pool_b0 || !w->pool_w2 ||
      !w->proj_w || !w->proj_b || !w->cb_embed || !w->ref_cb_weights || !w->ref_norm_w)
    return fail(SOPRO_ERR_INVALID, "reference preparation: null weight pointer");
  for (int i = 0; i < NL; ++i)
    if (!block_ok(w->ref_block[i])) return fail(SOPRO_ERR_INVALID, "reference encoder block %d: null weight", i);
  for (int i = 0; i < RL; ++i)
    if (!w->layer[i].nkv_w || !w->layer[i].k_w || !w->layer[i].v_w) return fail(SOPRO_ERR_INVALID, "ref layer %d: null weight", i);
  sopro_refprep* p = new sopro_refprep();
  p->device = device;
  p->cfg = *cfg;
  FArena A;
  auto softmax = [&](const float* x) {  // F.softmax(cb_weights, dim=0), fp32
    std::vector<float> s(Q);
    float mx = x[0];
    for (int q = 1; q < Q; ++q) mx = std::max(mx, x[q]);
    float sum = 0.f;
    for (int q = 0; q < Q; ++q) sum += (s[q] = expf(x[q] - mx));
    for (int q = 0; q < Q; ++q) s[q] /= sum;
    return A.add(s.data(), Q);
  };
  p->sv_emb = A.add(w->sv_emb, (size_t)Q * V * d);
  p->sv_w = softmax(w->sv_cb_weights);
  p->dw0_w = A.add(w->sv_dw0_w, (size_t)d * cfg->sv_kernel);
  p->dw0_b = A.add(w->sv_dw0_b, d);
  p->dw1_w = A.add(w->sv_dw1_w, (size_t)d * cfg->sv_kernel);
  p->dw1_b = A.add(w->sv_dw1_b, d);
  p->pool_w0 = A.add(w->pool_w0, (size_t)d * d);
  p->pool_b0 = A.add(w->pool_b0, d);
  p->pool_w2 = A.add(w->pool_w2, d);
  p->pool_b2 = w->pool_b2;
  p->proj_w = A.add(w->proj_w, (size_t)SV * 2 * d);
  p->proj_b = A.add(w->proj_b, SV);
  p->cb_embed = A.add(w->cb_embed, (size_t)Q * V * D);
  p->ref_w = softmax(w->ref_cb_weights);
  for (int i = 0; i < NL; ++i) add_block(A, w->ref_block[i], D, cfg->ref_enc_kernel, &p->blk[i]);
  p->ref_norm_w = A.add(w->ref_norm_w, D);
  for (int i = 0; i < RL; ++i) {
    p->layer[i].nkv_w = A.add(w->layer[i].nkv_w, D);
    p->layer[i].k_w = A.add(w->layer[i].k_w, (size_t)D * D);
    p->layer[i].v_w = A.add(w->layer[i].v_w, (size_t)D * D);
  }
  cudaError_t err = cudaMalloc(&p->dev, A.host.size() * 4);
  if (err == cudaSuccess) err = cudaMemcpy(p->dev, A.host.data(), A.host.size() * 4, cudaMemcpyHostToDevice);
  if (err == cudaSuccess) err = cudaMalloc(&p->bad, 256);
  if (err == cudaSuccess) err = cudaMemset(p->bad, 0, 256);
  if (err != cudaSuccess) {
    if (p->dev) cudaFree(p->dev);
    if (p->bad) cudaFree(p->bad);
    delete p;
    return fail(SOPRO_ERR_CUDA, "reference-preparation weight upload failed: %s", cudaGetErrorString(err));
  }
  *out = p;
  return SOPRO_OK;
}

int sopro_refprep_destroy(sopro_refprep_t* p) {
  if (!p) return SOPRO_OK;
  cudaSetDevice(p->device);
  cudaFree(p->dev);
  cudaFree(p->ws);
  cudaFree(p->bad);
  delete p;
  return SOPRO_OK;
}

int sopro_refprep_run(sopro_refprep_t* p, const int32_t* tokens, int Tr, float* sv, float* ref_seq, float* const* ref_k, float* const* ref_v,
                      void* stream) {
  if (!p || !tokens || !sv || !ref_seq) return fail(SOPRO_ERR_INVALID, "null argument");
  const sopro_refprep_config_t& c = p->cfg;
  if (Tr < 1 || Tr > 4096) return fail(SOPRO_ERR_INVALID, "Tr=%d outside [1, 4096]", Tr);
  if (c.ref_layers > 0 && (!ref_k || !ref_v)) return fail(SOPRO_ERR_INVALID, "ref_k / ref_v missing");
  for (int i = 0; i < c.ref_layers; ++i)
    if (!ref_k[i] || !ref_v[i]) return fail(SOPRO_ERR_INVALID, "ref_k[%d] / ref_v[%d] is null", i, i);
  CK(cudaSetDevice(p->device));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int D = c.d_model, d = c.sv_embed_dim, SV = c.sv_dim, Q = c.n_codebooks, V = c.codebook_size, H = c.ref_heads;
  const auto al = al64;
  const size_t rows = (size_t)Tr;
  const size_t need = (al(rows * D) * 3 + al(rows * 4 * D) + al(2 * (size_t)d) + al((size_t)SV) + al(2)) * 4;
  int rc;
  if ((rc = grow_ws(p, need, st))) return rc;
  float* x = p->ws;
  float* h = x + al(rows * D);
  float* q = h + al(rows * D);
  float* hid = q + al(rows * D);
  float* stats = hid + al(rows * 4 * D);  // [2d]
  float* e = stats + al(2 * (size_t)d);   // [SV]
  int* seq_rows = reinterpret_cast<int*>(e + al((size_t)SV));
  const float* W = p->dev;
  dense::DenseOp g{};
  // ---- Token2SV: the batched path with B = 1 (d <= D: the [Tr][d] buffers live in x / h / q)
  const int32_t len = Tr;
  if ((rc = token2sv(p, tokens, 1, Tr, &len, sv, nullptr, 0, nullptr, x, h, q, stats, e, seq_rows, st))) return rc;
  // ---- reference encoder
  codes_mix_kernel<<<Tr, 128, Q * sizeof(int), st>>>(tokens, W + p->cb_embed, W + p->ref_w, x, Q, V, D, p->bad, nullptr, 0);
  CK(cudaGetLastError());
  for (int i = 0; i < c.ref_enc_layers; ++i)
    if ((rc = ssm_block(W, p->blk[i], x, h, hid, nullptr, 1, Tr, D, c.ref_enc_kernel, 1, false, st))) return rc;
  dense::rmsnorm_rows_kernel<<<(unsigned)((Tr + 7) / 8), 256, 0, st>>>(x, W + p->ref_norm_w, nullptr, nullptr, ref_seq, (long long)Tr, D);
  CK(cudaGetLastError());
  // ---- cached K / V of every reference cross-attention layer, heads-major
  const long long tot = (long long)Tr * D;
  for (int i = 0; i < c.ref_layers; ++i) {
    for (int kv = 0; kv < 2; ++kv) {
      g = dense::DenseOp{};
      g.A = ref_seq; g.W = W + (kv ? p->layer[i].v_w : p->layer[i].k_w); g.norm_w = W + p->layer[i].nkv_w; g.C = h; g.M = Tr; g.N = D; g.K = D;
      g.ldc = D; g.epi = dense::EPI_BIAS;
      if ((rc = launch_dense(g, 1, st))) return rc;
      heads_major_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(h, kv ? ref_v[i] : ref_k[i], Tr, H, D / H);
      CK(cudaGetLastError());
    }
  }
  return SOPRO_OK;
}

}  // extern "C"

namespace pstage {

// sopro_refprep_speaker_vectors with row b scored against ref_sv + b * ref_stride (0: one vector for every row)
int speaker_vectors(sopro_refprep* p, const int32_t* tokens, int32_t B, int32_t Tmax, const int32_t* lens_host, float* sv,
                    const float* ref_sv, int ref_stride, float* cos, cudaStream_t st) {
  if (!p || !tokens || !lens_host || !sv) return fail(SOPRO_ERR_INVALID, "null argument");
  if (B < 1 || B > 65535) return fail(SOPRO_ERR_INVALID, "B=%d outside [1, 65535]", B);
  if (Tmax < 1 || Tmax > 4096) return fail(SOPRO_ERR_INVALID, "Tmax=%d outside [1, 4096]", Tmax);
  if (ref_sv && !cos) return fail(SOPRO_ERR_INVALID, "ref_sv given without cos");
  size_t total = 0;
  for (int b = 0; b < B; ++b) {
    if (lens_host[b] < 1 || lens_host[b] > Tmax) return fail(SOPRO_ERR_INVALID, "lens[%d]=%d outside [1, %d]", b, lens_host[b], Tmax);
    total += (size_t)lens_host[b];
  }
  CK(cudaSetDevice(p->device));
  const size_t d = p->cfg.sv_embed_dim, SV = p->cfg.sv_dim, nb = (size_t)B;
  const auto al = al64;
  const size_t need = (al(total * d) * 3 + al(nb * 2 * d) + al(nb * SV) + al(2 * nb)) * 4;
  int rc;
  if ((rc = grow_ws(p, need, st))) return rc;
  float* x = p->ws;
  float* h = x + al(total * d);
  float* q = h + al(total * d);
  float* stats = q + al(total * d);
  float* e = stats + al(nb * 2 * d);
  int* rows = reinterpret_cast<int*>(e + al(nb * SV));
  return token2sv(p, tokens, B, Tmax, lens_host, sv, ref_sv, ref_stride, cos, x, h, q, stats, e, rows, st);
}

}  // namespace pstage

extern "C" {

int sopro_refprep_speaker_vectors(sopro_refprep_t* p, const int32_t* tokens, int32_t B, int32_t Tmax, const int32_t* lens_host,
                                  float* sv, const float* ref_sv, float* cos, void* stream) {
  return pstage::speaker_vectors(p, tokens, B, Tmax, lens_host, sv, ref_sv, 0, cos, reinterpret_cast<cudaStream_t>(stream));
}

int sopro_refprep_speaker_vectors_per_row(sopro_refprep_t* p, const int32_t* tokens, int32_t B, int32_t Tmax, const int32_t* lens_host,
                                          float* sv, const float* ref_sv, float* cos, void* stream) {
  if (!ref_sv || !cos) return fail(SOPRO_ERR_INVALID, "ref_sv and cos are required");
  return pstage::speaker_vectors(p, tokens, B, Tmax, lens_host, sv, ref_sv, p ? p->cfg.sv_dim : 0, cos,
                                 reinterpret_cast<cudaStream_t>(stream));
}

/* Synchronises `stream`; SOPRO_ERR_INVALID if a run since the last check met a code outside [0, codebook_size). */
int sopro_refprep_check(sopro_refprep_t* p, void* stream) {
  if (!p) return fail(SOPRO_ERR_INVALID, "null argument");
  CK(cudaSetDevice(p->device));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int bad = 0;
  CK(cudaMemcpyAsync(&bad, p->bad, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (bad) {
    CK(cudaMemsetAsync(p->bad, 0, 4, st));
    return fail(SOPRO_ERR_INVALID, "reference codes outside [0, %d)", p->cfg.codebook_size);
  }
  return SOPRO_OK;
}

}  // extern "C"
