// Watermark: a keyed spread-spectrum mark on the 24 kHz output, its streaming form, and a batched detector.  The
// definition is in include/sopro_b200.h and, in float64, in oracle/watermark_oracle.py:
//   pattern p: P = 8192 samples, the real-DFT bins in [1000, 3500] Hz at unit magnitude and splitmix64 phases, unit RMS;
//   embed:  r_j = the RMS of 240-sample block j (a trailing partial block over its own samples), g_j = a min(r_{j-1}, r_j)
//           with r_{-1} = 0 and a = 10^(-30/20), y[n] = x[n] + g_{j(n)} p[n mod P] (one fma; g = 0 leaves x bit-equal);
//   detect: w_j = 1 / r_j where r_j > max(10^(-40/20) max r, 1e-6), else 0; F[k] = sum over n = k mod P of w x[n];
//           c[l] = sum_k F[k] p[(k + l) mod P]; score = max c / sqrt(mean c^2), offset = argmax.
//
// block_rms() is the only place a block's RMS is computed: one warp sums the block's squares in double in a fixed
// order that depends only on the block's own samples, so a row's marks are the same alone, in any ragged batch and in
// any chunking of a stream.  The one-shot and stream kernels call it and gain() / mark() on the same values.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <vector>

#include "../../include/sopro_b200.h"
#include "chunk_stream.cuh"

namespace {

constexpr int kP = SOPRO_WATERMARK_PERIOD, kBlk = SOPRO_WATERMARK_BLOCK;
constexpr int kT = 256, kWarps = kT / 32;
constexpr int kRowsPerLaunch = 128;  // rows of a ragged batch per launch (their lengths travel as a kernel parameter)
constexpr long long kMaxLen = 1LL << 40;
constexpr int kRate = 24000;
constexpr int kLoBin = (SOPRO_WATERMARK_LO_HZ * kP + kRate - 1) / kRate, kHiBin = SOPRO_WATERMARK_HI_HZ * kP / kRate;
// correlation: thread t scores the kR consecutive lags l0 + kR t + [0, kR) (register-blocked sliding dot product; kR
// odd, so the lanes' window loads hit 32 distinct banks), over k in tiles of kKT staged in shared memory
constexpr int kR = 9, kLags = kR * kT, kKT = 1024, kLagCtas = (kP + kLags - 1) / kLags;
constexpr int kScoreT = 1024;
constexpr double kPi = 3.141592653589793;
static_assert((kP & (kP - 1)) == 0 && kP % kT == 0 && kP % kKT == 0, "geometry");
static_assert(kLoBin == 342 && kHiBin == 1194, "the band's bins");

double level() { return std::pow(10.0, SOPRO_WATERMARK_LEVEL_DB / 20.0); }
double floor_ratio() { return std::pow(10.0, SOPRO_WATERMARK_FLOOR_DB / 20.0); }

// logical sample i of an utterance: [0, split) from a, the rest from b (the one-shot path has a single source, a stream
// its carried partial block and the new chunk)
struct Src {
  const float* a;
  const float* b;
  long long split;
};

__device__ __forceinline__ float src_at(const Src& s, long long i) { return i < s.split ? s.a[i] : s.b[i - s.split]; }

// sqrt(sum x^2 / count) over samples [start, start + count) in double; one warp, every lane returns the same value
// (lane l adds samples l, l + 32, ... in order, then a butterfly whose partners add the same two values)
__device__ __forceinline__ double block_rms(const Src& s, long long start, int count) {
  const int lane = threadIdx.x & 31;
  double acc = 0.0;
  for (int i = lane; i < count; i += 32) {
    const double v = src_at(s, start + i);
    acc = fma(v, v, acc);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  return sqrt(acc / (double)count);
}

__device__ __forceinline__ float gain(double a, double r_prev, double r) { return __double2float_rn(a * fmin(r_prev, r)); }

__device__ __forceinline__ float mark(float x, float g, float p) { return g == 0.0f ? x : __fmaf_rn(g, p, x); }

// one-shot: grid (ceil(blocks / 8), rows); warp w -> r of block 8 blockIdx.x + w of the row
__global__ void __launch_bounds__(kT) wm_rms_kernel(const float* __restrict__ x, long long x_stride, RowLens<kRowsPerLaunch> lens,
                                                    double* __restrict__ r, long long r_stride) {
  const int b = blockIdx.y;
  const long long n = lens.v[b], j = (long long)blockIdx.x * kWarps + (threadIdx.x >> 5), start = j * kBlk;
  if (start >= n) return;  // whole warps leave together
  const Src s{x + (long long)b * x_stride, nullptr, n};
  const double v = block_rms(s, start, (int)std::min<long long>(kBlk, n - start));
  if ((threadIdx.x & 31) == 0) r[(long long)b * r_stride + j] = v;
}

// one-shot: y = x + g_j p[n mod P] over [0, lens[b])
__global__ void __launch_bounds__(kT) wm_apply_kernel(const float* __restrict__ x, long long x_stride, RowLens<kRowsPerLaunch> lens,
                                                      const double* __restrict__ r, long long r_stride, const float* __restrict__ p,
                                                      double a, float* __restrict__ y, long long y_stride) {
  const int b = blockIdx.y;
  const long long n = lens.v[b];
  const float* xb = x + (long long)b * x_stride;
  const double* rb = r + (long long)b * r_stride;
  float* yb = y + (long long)b * y_stride;
  for (long long i = (long long)blockIdx.x * kT + threadIdx.x; i < n; i += (long long)gridDim.x * kT) {
    const long long j = i / kBlk;
    yb[i] = mark(xb[i], gain(a, j ? rb[j - 1] : 0.0, rb[j]), p[i & (kP - 1)]);
  }
}

// stream: the RMS of the nb blocks of the span s (the last one `last_count` samples when nonzero) -> r[1 ..], and
// r[0] = the block before the span's (0 before the utterance's first block)
__global__ void __launch_bounds__(kT) wm_stream_rms_kernel(Src s, int nb, int last_count, const double* __restrict__ r_last,
                                                           int have_prev, double* __restrict__ r) {
  const int q = blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (blockIdx.x == 0 && threadIdx.x == 0) r[0] = have_prev ? *r_last : 0.0;
  if (q >= nb) return;
  const double v = block_rms(s, (long long)q * kBlk, (q == nb - 1 && last_count) ? last_count : kBlk);
  if ((threadIdx.x & 31) == 0) r[1 + q] = v;
}

// stream: the span's first `count` samples marked; `base` is the utterance index of the span's first sample.  The
// last block's r is carried to the next push in r_last (the rms kernel of this push has read it already).
__global__ void __launch_bounds__(kT) wm_stream_apply_kernel(Src s, long long count, long long base, int nb, const double* __restrict__ r,
                                                             const float* __restrict__ p, double a, float* __restrict__ y,
                                                             double* __restrict__ r_last) {
  for (long long i = (long long)blockIdx.x * kT + threadIdx.x; i < count; i += (long long)gridDim.x * kT) {
    const long long q = i / kBlk;
    y[i] = mark(src_at(s, i), gain(a, r[q], r[q + 1]), p[(base + i) & (kP - 1)]);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *r_last = r[nb];
}

// detect: grid (P / kT, rows); thread k: F[k] = sum over m ascending of w_{j(n)} x[n], n = k + m P < lens[b], in double
__global__ void __launch_bounds__(kT) wm_fold_kernel(const float* __restrict__ x, long long x_stride, RowLens<kRowsPerLaunch> lens,
                                                     const double* __restrict__ r, long long r_stride, double floor_ratio,
                                                     float* __restrict__ F) {
  __shared__ double red[kT];
  const int b = blockIdx.y, tid = threadIdx.x;
  const long long n = lens.v[b], nblk = (n + kBlk - 1) / kBlk;
  const double* rb = r + (long long)b * r_stride;
  double m = 0.0;
  for (long long j = tid; j < nblk; j += kT) m = fmax(m, rb[j]);
  red[tid] = m;
  __syncthreads();
  for (int h = kT / 2; h > 0; h >>= 1) {
    if (tid < h) red[tid] = fmax(red[tid], red[tid + h]);
    __syncthreads();
  }
  const double thr = fmax(floor_ratio * red[0], 1e-6);
  const float* xb = x + (long long)b * x_stride;
  const long long k = (long long)blockIdx.x * kT + tid;
  double acc = 0.0;
  for (long long i = k; i < n; i += kP) {
    const double rj = rb[i / kBlk];
    if (rj > thr) acc = fma(1.0 / rj, (double)xb[i], acc);
  }
  F[(long long)b * kP + k] = (float)acc;
}

// detect: grid (kLagCtas, rows); c[l] = sum_k F[k] p[(k + l) mod P], k ascending, fp32
__global__ void __launch_bounds__(kT) wm_corr_kernel(const float* __restrict__ F, const float* __restrict__ p, float* __restrict__ c) {
  __shared__ float fs[kKT];
  __shared__ float ps[kKT + kLags];
  const int b = blockIdx.y, tid = threadIdx.x, l0 = blockIdx.x * kLags;
  const float* Fb = F + (long long)b * kP;
  float acc[kR];
#pragma unroll
  for (int j = 0; j < kR; ++j) acc[j] = 0.0f;
  for (int k0 = 0; k0 < kP; k0 += kKT) {
    __syncthreads();  // the previous tile is consumed
    for (int i = tid; i < kKT; i += kT) fs[i] = Fb[k0 + i];
    for (int i = tid; i < kKT + kLags; i += kT) ps[i] = p[(k0 + l0 + i) & (kP - 1)];  // ps[i] = p[(k0 + l0 + i) mod P]
    __syncthreads();
    const float* w = ps + kR * tid;  // lag l0 + kR tid + j at k0 + kk reads w[kk + j]
    float xr[kR];
#pragma unroll
    for (int j = 0; j < kR; ++j) xr[j] = w[j];
#pragma unroll kR
    for (int kk = 0; kk < kKT; ++kk) {
      const float f = fs[kk];
#pragma unroll
      for (int j = 0; j < kR; ++j) acc[j] = __fmaf_rn(f, xr[j], acc[j]);
#pragma unroll
      for (int j = 0; j + 1 < kR; ++j) xr[j] = xr[j + 1];
      xr[kR - 1] = w[kk + kR];
    }
  }
#pragma unroll
  for (int j = 0; j < kR; ++j) {
    const int l = l0 + kR * tid + j;
    if (l < kP) c[(long long)b * kP + l] = acc[j];
  }
}

// detect: one CTA per row; the peak (ties to the smaller lag), sum c^2 in double by a fixed tree, score and decision
__global__ void __launch_bounds__(kScoreT) wm_score_kernel(const float* __restrict__ c, float* __restrict__ score,
                                                           int64_t* __restrict__ offset, uint8_t* __restrict__ detected) {
  __shared__ float bm[kScoreT];
  __shared__ int bl[kScoreT];
  __shared__ double bs[kScoreT];
  const int b = blockIdx.x, tid = threadIdx.x;
  const float* cb = c + (long long)b * kP;
  float m = -INFINITY;
  int at = 0;
  double ss = 0.0;
  for (int l = tid; l < kP; l += kScoreT) {
    const float v = cb[l];
    ss = fma((double)v, (double)v, ss);
    if (v > m) {
      m = v;
      at = l;
    }
  }
  bm[tid] = m;
  bl[tid] = at;
  bs[tid] = ss;
  __syncthreads();
  for (int h = kScoreT / 2; h > 0; h >>= 1) {
    if (tid < h) {
      const float m2 = bm[tid + h];
      const int l2 = bl[tid + h];
      if (m2 > bm[tid] || (m2 == bm[tid] && l2 < bl[tid])) {
        bm[tid] = m2;
        bl[tid] = l2;
      }
      bs[tid] += bs[tid + h];
    }
    __syncthreads();
  }
  if (tid == 0) {
    const double mean = bs[0] / kP;
    const double s = mean > 0.0 ? (double)bm[0] / sqrt(mean) : 0.0;
    score[b] = (float)s;
    offset[b] = mean > 0.0 ? bl[0] : 0;
    detected[b] = s >= SOPRO_WATERMARK_THRESHOLD ? 1 : 0;
  }
}

// the workspaces: r [B][blocks] (embed and detect), then F [B][P] and c [B][P] (detect)
struct Layout {
  long long nblk = 0;
  size_t r = 0, F = 0, c = 0, embed = 0, detect = 0;
};

Layout layout(int B, long long max_len) {
  Layout l;
  l.nblk = (max_len + kBlk - 1) / kBlk;
  auto up = [](size_t v) { return (v + 255) & ~(size_t)255; };
  l.r = 0;
  l.embed = up((size_t)B * l.nblk * sizeof(double));
  l.F = l.embed;
  l.c = l.F + up((size_t)B * kP * sizeof(float));
  l.detect = l.c + up((size_t)B * kP * sizeof(float));
  return l;
}

// carried partial block: fewer than kBlk samples
constexpr long long kCarryCap = kBlk;

}  // namespace

// the tail holds the held partial block: samples [done, n_seen) of the utterance
struct sopro_watermark_stream : chunk::ChunkStream {
  const float* pattern = nullptr;  // the key's table (device)
  double* r = nullptr;             // [max_chunk / kBlk + 2]: one push's blocks, after the one before them
  double* r_last = nullptr;        // the last complete block's r

  cudaError_t alloc_own() {
    const cudaError_t e = cudaMalloc(&r, (size_t)(max_chunk / kBlk + 2) * sizeof(double));
    return e == cudaSuccess ? cudaMalloc(&r_last, sizeof(double)) : e;
  }
  void free_own() {
    cudaFree(r);
    cudaFree(r_last);
  }
};

namespace {
// the tail followed by x: the span [done, done + count) marked -> y, its nb blocks' RMS first (the last one over
// last_count samples)
int stream_launch(sopro_watermark_stream* s, const float* x, int nb, int last_count, long long count, float* y, cudaStream_t st) {
  if (nb == 0) return SOPRO_OK;
  const long long done = s->tail.base;
  const Src src{s->tail.data(), x, s->tail.held()};
  wm_stream_rms_kernel<<<(nb + kWarps - 1) / kWarps, kT, 0, st>>>(src, nb, last_count, s->r_last, done > 0 ? 1 : 0, s->r);
  CK(cudaGetLastError());
  const long long gx = std::min<long long>((count + kT - 1) / kT, 4096);
  wm_stream_apply_kernel<<<(unsigned)gx, kT, 0, st>>>(src, count, done, nb, s->r, s->pattern, level(), y, s->r_last);
  CK(cudaGetLastError());
  return SOPRO_OK;
}
}  // namespace

extern "C" {

int sopro_watermark_pattern(int64_t key, float* out) {
  if (!out) return fail(SOPRO_ERR_INVALID, "null argument");
  if (key < 0 || key > 0xFFFFFFFFLL) return fail(SOPRO_ERR_INVALID, "watermark key must be an integer in [0, 2^32) (got %lld)", (long long)key);
  std::vector<double> cs(kP), sn(kP), acc(kP, 0.0);
  for (int m = 0; m < kP; ++m) {
    cs[m] = std::cos(2.0 * kPi * m / kP);
    sn[m] = std::sin(2.0 * kPi * m / kP);
  }
  uint64_t state = (uint64_t)key;
  for (int k = kLoBin; k <= kHiBin; ++k) {  // splitmix64, one draw per bin in bin order
    state += 0x9E3779B97F4A7C15ULL;
    uint64_t z = state;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    z ^= z >> 31;
    const double phi = 2.0 * kPi * ((double)(z >> 11) * 0x1.0p-53);
    const double c = std::cos(phi), s = std::sin(phi);
    // cos(2 pi k n / P + phi) = cos(2 pi m / P) cos(phi) - sin(2 pi m / P) sin(phi), m = k n mod P
    for (int n = 0; n < kP; ++n) {
      const int m = (int)(((long long)k * n) & (kP - 1));
      acc[n] += cs[m] * c - sn[m] * s;
    }
  }
  double e = 0.0;
  for (int n = 0; n < kP; ++n) e += acc[n] * acc[n];
  const double inv = 1.0 / std::sqrt(e / kP);
  for (int n = 0; n < kP; ++n) out[n] = (float)(acc[n] * inv);
  return SOPRO_OK;
}

int sopro_watermark_sizes(int32_t B, int64_t max_len, int64_t* embed_ws, int64_t* detect_ws) {
  if (B < 1 || max_len < 0 || max_len > kMaxLen) return fail(SOPRO_ERR_INVALID, "bad geometry (B=%d, max_len=%lld)", B, (long long)max_len);
  const Layout l = layout(B, max_len);
  if (embed_ws) *embed_ws = (int64_t)l.embed;
  if (detect_ws) *detect_ws = (int64_t)l.detect;
  return SOPRO_OK;
}

int sopro_watermark_embed(const float* x, int32_t B, int64_t x_stride, const int64_t* lens_host, const float* pattern, float* y,
                          int64_t y_stride, void* ws, void* stream) {
  if (!pattern || !ws) return fail(SOPRO_ERR_INVALID, "null argument");
  long long most = 0;
  int rc = check_rows(x, B, x_stride, lens_host, kMaxLen, &most);
  if (rc == SOPRO_OK) rc = check_out_rows(y, B, y_stride, most);
  if (rc != SOPRO_OK) return rc;
  if (most == 0) return SOPRO_OK;
  const Layout l = layout(B, most);
  double* r = reinterpret_cast<double*>(static_cast<char*>(ws) + l.r);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const double a = level();
  const long long gx = std::min<long long>((most + kT - 1) / kT, 4096);
  for (int b0 = 0; b0 < B; b0 += kRowsPerLaunch) {
    const int rows = std::min(kRowsPerLaunch, B - b0);
    const RowLens<kRowsPerLaunch> L = row_lens<kRowsPerLaunch>(lens_host, x_stride, b0, rows);
    double* rb = r + (long long)b0 * l.nblk;
    wm_rms_kernel<<<dim3((unsigned)((l.nblk + kWarps - 1) / kWarps), rows), kT, 0, st>>>(x + (long long)b0 * x_stride, x_stride, L,
                                                                                          rb, l.nblk);
    CK(cudaGetLastError());
    wm_apply_kernel<<<dim3((unsigned)gx, rows), kT, 0, st>>>(x + (long long)b0 * x_stride, x_stride, L, rb, l.nblk, pattern, a,
                                                              y + (long long)b0 * y_stride, y_stride);
    CK(cudaGetLastError());
  }
  return SOPRO_OK;
}

int sopro_watermark_detect(const float* x, int32_t B, int64_t x_stride, const int64_t* lens_host, const float* pattern, void* ws,
                           float* score, int64_t* offset, uint8_t* detected, void* stream) {
  if (!pattern || !ws) return fail(SOPRO_ERR_INVALID, "null argument");
  long long most = 0;
  const int rc = check_rows(x, B, x_stride, lens_host, kMaxLen, &most);
  if (rc != SOPRO_OK) return rc;
  if (!score || !offset || !detected) return fail(SOPRO_ERR_INVALID, "null argument");
  const Layout l = layout(B, most);
  char* w = static_cast<char*>(ws);
  double* r = reinterpret_cast<double*>(w + l.r);
  float* F = reinterpret_cast<float*>(w + l.F);
  float* c = reinterpret_cast<float*>(w + l.c);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const double fr = floor_ratio();
  for (int b0 = 0; b0 < B; b0 += kRowsPerLaunch) {
    const int rows = std::min(kRowsPerLaunch, B - b0);
    const RowLens<kRowsPerLaunch> L = row_lens<kRowsPerLaunch>(lens_host, x_stride, b0, rows);
    const float* xb = x + (long long)b0 * x_stride;
    double* rb = r + (long long)b0 * l.nblk;
    float* Fb = F + (long long)b0 * kP;
    float* cb = c + (long long)b0 * kP;
    if (l.nblk > 0) {
      wm_rms_kernel<<<dim3((unsigned)((l.nblk + kWarps - 1) / kWarps), rows), kT, 0, st>>>(xb, x_stride, L, rb, l.nblk);
      CK(cudaGetLastError());
    }
    wm_fold_kernel<<<dim3(kP / kT, rows), kT, 0, st>>>(xb, x_stride, L, rb, l.nblk, fr, Fb);
    CK(cudaGetLastError());
    wm_corr_kernel<<<dim3(kLagCtas, rows), kT, 0, st>>>(Fb, pattern, cb);
    CK(cudaGetLastError());
    wm_score_kernel<<<rows, kScoreT, 0, st>>>(cb, score + b0, offset + b0, detected + b0);
    CK(cudaGetLastError());
  }
  return SOPRO_OK;
}

int sopro_watermark_stream_create(int64_t max_chunk, int device, sopro_watermark_stream_t** out) {
  int rc = chunk::check_create(max_chunk, out);
  if (rc == SOPRO_OK) rc = open_device(device, "the watermark");
  if (rc != SOPRO_OK) return rc;
  sopro_watermark_stream* s = new sopro_watermark_stream();
  s->unset = "key";
  return chunk::create(s, max_chunk, kCarryCap, "watermark", out);
}

int sopro_watermark_stream_destroy(sopro_watermark_stream_t* s) { return chunk::destroy(s); }

int sopro_watermark_stream_reset(sopro_watermark_stream_t* s, const float* pattern) {
  if (!s || !pattern) return fail(SOPRO_ERR_INVALID, "null argument");
  s->pattern = pattern;
  s->restart(0);
  return SOPRO_OK;
}

int64_t sopro_watermark_stream_ready(const sopro_watermark_stream_t* s, int64_t n_more, int final) {
  if (!chunk::can_run(s, n_more)) return -1;
  const long long n = s->tail.held() + n_more;
  return final ? n : n / kBlk * kBlk;
}

int sopro_watermark_push(sopro_watermark_stream_t* s, const float* x, int64_t n, float* y, void* stream) {
  int rc = chunk::check_push(s, n);
  if (rc != SOPRO_OK || n == 0) return rc;
  const long long count = (s->tail.held() + n) / kBlk * kBlk;
  if ((rc = chunk::check_io(x, n, y, count)) != SOPRO_OK) return rc;
  CK(cudaSetDevice(s->tail.device));
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  rc = stream_launch(s, x, (int)(count / kBlk), 0, count, y, st);
  if (rc == SOPRO_OK) rc = s->tail.keep(s->tail.base + count, x, n, st);  // the new partial block
  return rc;
}

int sopro_watermark_finish(sopro_watermark_stream_t* s, float* y, void* stream) {
  int rc = chunk::check_finish(s);
  if (rc != SOPRO_OK) return rc;
  const long long held = s->tail.held();
  if ((rc = chunk::check_io(nullptr, 0, y, held)) != SOPRO_OK) return rc;
  if (held > 0) {
    CK(cudaSetDevice(s->tail.device));
    rc = stream_launch(s, nullptr, 1, (int)held, held, y, reinterpret_cast<cudaStream_t>(stream));
    if (rc != SOPRO_OK) return rc;
  }
  s->finished = true;
  return SOPRO_OK;
}

}  // extern "C"
