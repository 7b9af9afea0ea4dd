// Long-form synthesis: the speech extent of each segment's decoded row, and the join of those extents into one waveform.
// The definition (include/sopro_b200.h, oracle/longform_oracle.py in float64), at the codec's 24 kHz:
//   extents: the energy trim of sopro_b200.audio.trim_silence_energy.  Frames of 600 samples every 240,
//     K = floor((n - 600) / 240) + 1; e_k = sum x^2 / 600, dB_k = 10 log10(e_k + 1e-10) in fp64; thr = max(max dB - 40,
//     -40); frame k is voiced when dB_k > thr; start = max(0, first 240 - 720), end = min(n, last 240 + 600 + 720).
//     The row is left whole, (0, n), when n < 2400, nothing is voiced, or end - start < 12000.
//   join: for each non-empty extent in order, x[start, end) with a raised-cosine fade over its first and last
//     F = min(240, floor(span / 2)) samples, f[i] = 0.5 - 0.5 cos(pi (i + 0.5) / F) (double on the host, fp32 once; one
//     fp32 multiply per faded sample), and P zero samples between consecutive spans.
//
// extents_kernel: one CTA per row.  A warp computes a frame: lane l sums x^2 over the frame's samples l, l + 32, ... in
// order (each product is exact in fp64), then a butterfly; every frame's dB therefore has one fixed value whatever the
// batch.  Pass 1 takes the maximum; pass 2 looks for the first voiced frame in rounds of one frame per warp from the
// start, and the last from the end, stopping at the first round that finds one.
// join_kernel: grid (pieces, segments); the segments of one launch share their F, and their fade table travels in the
// kernel parameters with the source pointers, so nothing is copied to the device first.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../include/sopro_b200.h"
#include "common.cuh"

namespace {

constexpr int kFrame = 600, kHop = 240, kPad = 720, kMinRow = 2400, kMinKeep = 12000;  // 25 ms, 10 ms, 30 ms, 0.1 s, 0.5 s
constexpr int kFadeMax = 240;                // 10 ms
constexpr long long kMaxPause = 48000;       // 2 s
constexpr int kExtThreads = 512, kExtWarps = kExtThreads / 32;
constexpr int kJoinThreads = 256;
constexpr int kRowsPerLaunch = 128;          // rows of one extents launch (their lengths travel as a kernel parameter)
constexpr int kSegsPerLaunch = 64;           // segments of one join launch
constexpr long long kMaxLen = 1LL << 40;
constexpr double kPi = 3.141592653589793;

// frame k's dB, the same value in every lane
__device__ __forceinline__ double frame_db(const float* __restrict__ x, long long k, int lane) {
  const float* f = x + k * kHop;
  double s = 0.0;
#pragma unroll
  for (int j = 0; j < (kFrame + 31) / 32; ++j) {
    const int i = lane + 32 * j;
    if (i < kFrame) {
      const double v = (double)__ldg(f + i);
      s = fma(v, v, s);  // v * v is exact: the fma rounds exactly as the separate add would
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return 10.0 * log10(s / (double)kFrame + 1e-10);
}

__global__ void __launch_bounds__(kExtThreads) extents_kernel(const float* __restrict__ x, long long x_stride, RowLens<kRowsPerLaunch> lens,
                                                              long long* __restrict__ ext) {
  __shared__ double wmax[kExtWarps];
  __shared__ long long s_first, s_last;
  const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long n = lens.v[b];
  const float* xb = x + (long long)b * x_stride;
  long long* out = ext + 2LL * b;
  if (n < kMinRow) {  // (kMinRow > kFrame: every row that gets here has at least 8 frames)
    if (threadIdx.x == 0) {
      out[0] = 0;
      out[1] = n;
    }
    return;
  }
  const long long K = (n - kFrame) / kHop + 1;
  double m = -INFINITY;
  for (long long k = warp; k < K; k += kExtWarps) m = fmax(m, frame_db(xb, k, lane));
  if (lane == 0) wmax[warp] = m;
  if (threadIdx.x == 0) {
    s_first = K;
    s_last = -1;
  }
  __syncthreads();
  double mx = wmax[0];
  for (int w = 1; w < kExtWarps; ++w) mx = fmax(mx, wmax[w]);
  const double thr = fmax(mx - 40.0, -40.0);
  if (mx > thr) {  // the loudest frame is voiced (uniform across the CTA)
    for (long long k0 = 0; k0 < K; k0 += kExtWarps) {
      const long long k = k0 + warp;
      const bool v = k < K && frame_db(xb, k, lane) > thr;
      if (v && lane == 0) atomicMin(&s_first, k);
      if (__syncthreads_or(v)) break;
    }
    for (long long k0 = 0; k0 < K; k0 += kExtWarps) {
      const long long k = K - 1 - (k0 + warp);
      const bool v = k >= 0 && frame_db(xb, k, lane) > thr;
      if (v && lane == 0) atomicMax(&s_last, k);
      if (__syncthreads_or(v)) break;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    long long start = 0, end = n;
    if (s_last >= 0) {
      start = std::max(0LL, s_first * kHop - kPad);
      end = std::min(n, s_last * kHop + kFrame + kPad);
      if (end - start < kMinKeep) start = 0, end = n;
    }
    out[0] = start;
    out[1] = end;
  }
}

struct JoinSeg {
  const float* src;  // x + start
  long long span, off;
  long long pause;   // zero samples written after the span
};

struct JoinArgs {
  float f[kFadeMax];
  int F, nseg;
  JoinSeg s[kSegsPerLaunch];
};
static_assert(sizeof(JoinArgs) <= 4000, "the join's arguments fit the kernel parameter space");

__global__ void __launch_bounds__(kJoinThreads) join_kernel(const JoinArgs a, float* __restrict__ y) {
  const JoinSeg s = a.s[blockIdx.y];
  const long long total = s.span + s.pause;
  float* yo = y + s.off;
  for (long long j = (long long)blockIdx.x * kJoinThreads + threadIdx.x; j < total; j += (long long)gridDim.x * kJoinThreads) {
    float v = 0.0f;
    if (j < s.span) {
      v = __ldg(s.src + j);
      if (j < a.F)
        v = __fmul_rn(v, a.f[j]);
      else if (j >= s.span - a.F)
        v = __fmul_rn(v, a.f[s.span - 1 - j]);
    }
    yo[j] = v;
  }
}

void fade(int F, float* f) {
  for (int i = 0; i < F; ++i) f[i] = (float)(0.5 - 0.5 * std::cos(kPi * (i + 0.5) / F));
}

int fade_len(long long span) { return (int)std::min<long long>(kFadeMax, span / 2); }

}  // namespace

extern "C" {

int sopro_longform_fade(int32_t F, float* f) {
  if (F < 0 || F > kFadeMax) return fail(SOPRO_ERR_INVALID, "fade length %d not in [0, %d]", F, kFadeMax);
  if (F > 0 && !f) return fail(SOPRO_ERR_INVALID, "null argument");
  fade(F, f);
  return SOPRO_OK;
}

int sopro_longform_extents(const float* x, int32_t B, int64_t x_stride, const int64_t* lens_host, int64_t* ext, void* stream) {
  if (!ext) return fail(SOPRO_ERR_INVALID, "null argument");
  long long most = 0;
  const int rc = check_rows(x, B, x_stride, lens_host, kMaxLen, &most);
  if (rc != SOPRO_OK) return rc;
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  for (int b0 = 0; b0 < B; b0 += kRowsPerLaunch) {
    const int rows = std::min(kRowsPerLaunch, B - b0);
    extents_kernel<<<rows, kExtThreads, 0, st>>>(x + (long long)b0 * x_stride, x_stride,
                                                 row_lens<kRowsPerLaunch>(lens_host, x_stride, b0, rows),
                                                 reinterpret_cast<long long*>(ext) + 2LL * b0);
    CK(cudaGetLastError());
  }
  return SOPRO_OK;
}

int sopro_longform_join(const float* const* src, int32_t n_seg, const int64_t* lens_host, const int64_t* ext_host, int64_t pause,
                        float* y, int64_t y_len, void* stream) {
  if (!src || !lens_host || !ext_host) return fail(SOPRO_ERR_INVALID, "null argument");
  if (n_seg < 1) return fail(SOPRO_ERR_INVALID, "n_seg = %d < 1", n_seg);
  if (pause < 0 || pause > kMaxPause) return fail(SOPRO_ERR_INVALID, "pause of %lld samples not in [0, %lld]", (long long)pause, kMaxPause);
  long long total = 0, last = -1;
  for (int i = 0; i < n_seg; ++i) {
    const long long len = lens_host[i], s = ext_host[2 * i], e = ext_host[2 * i + 1];
    if (len < 0 || len > kMaxLen) return fail(SOPRO_ERR_INVALID, "lens[%d] = %lld not in [0, 2^40]", i, len);
    if (s < 0 || s > e || e > len)
      return fail(SOPRO_ERR_INVALID, "extent [%lld, %lld) of segment %d is not inside its %lld samples", s, e, i, len);
    if (e > s && !src[i]) return fail(SOPRO_ERR_INVALID, "null source for segment %d", i);
    if (e > s) {
      total += (last >= 0 ? pause : 0) + (e - s);
      last = i;
    }
  }
  if (y_len != total) return fail(SOPRO_ERR_INVALID, "y_len = %lld, the joined length is %lld", (long long)y_len, total);
  if (total == 0) return SOPRO_OK;
  if (!y) return fail(SOPRO_ERR_INVALID, "null argument");
  // each span's place in y, then one launch per (fade length, run of at most kSegsPerLaunch segments)
  std::vector<long long> off(n_seg, 0);
  std::vector<char> done(n_seg, 1);
  for (long long i = 0, o = 0; i < n_seg; ++i) {
    const long long span = ext_host[2 * i + 1] - ext_host[2 * i];
    if (span == 0) continue;
    off[i] = o;
    o += span + pause;
    done[i] = 0;
  }
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  JoinArgs a{};
  long long most = 0;  // the longest span + pause of the pending launch
  auto launch = [&]() -> int {
    const unsigned gx = (unsigned)std::min<long long>((most + kJoinThreads - 1) / kJoinThreads, 1024);
    join_kernel<<<dim3(gx, a.nseg), kJoinThreads, 0, st>>>(a, y);
    CK(cudaGetLastError());
    a.nseg = 0;
    most = 0;
    return SOPRO_OK;
  };
  for (int i = 0; i < n_seg; ++i) {
    if (done[i]) continue;
    const int F = fade_len(ext_host[2 * i + 1] - ext_host[2 * i]);
    std::memset(&a, 0, sizeof(a));
    fade(F, a.f);
    a.F = F;
    for (int j = i; j < n_seg; ++j) {
      const long long span = ext_host[2 * j + 1] - ext_host[2 * j];
      if (done[j] || fade_len(span) != F) continue;
      JoinSeg& s = a.s[a.nseg++];
      s.src = src[j] + ext_host[2 * j];
      s.span = span;
      s.off = off[j];
      s.pause = j == last ? 0 : pause;
      most = std::max(most, span + s.pause);
      done[j] = 1;
      if (a.nseg == kSegsPerLaunch) {
        const int r = launch();
        if (r != SOPRO_OK) return r;
      }
    }
    if (a.nseg > 0) {
      const int r = launch();
      if (r != SOPRO_OK) return r;
    }
  }
  return SOPRO_OK;
}

}  // extern "C"
