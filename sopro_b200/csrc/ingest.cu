// Voice ingestion: the host-side preparation of MimiCodec.encode_file (energy trim, then the rows the resampler and the
// encoder read) for a ragged batch of clips, each at its own sample rate.  The definitions are in include/sopro_b200.h;
// oracle/ingest_oracle.py restates the trim in float64.
//
// trim_kernel: one CTA per row, the longform extents kernel (longform.cu) with the frame geometry of the row's rate.  A
// warp computes a frame: lane l sums x^2 over the frame's samples l, l + 32, ... in order (each product is exact in
// fp64), then a butterfly; every frame's dB therefore has one fixed value whatever the batch.  Pass 1 takes the maximum;
// pass 2 looks for the first voiced frame in rounds of one frame per warp from the start, and the last from the end,
// stopping at the first round that finds one.
// pack_kernel: grid (pieces, rows); the rows' source pointers and lengths travel in the kernel parameters.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>

#include "../../include/sopro_b200.h"
#include "common.cuh"

namespace {

constexpr int kMinRate = 4000, kMaxRate = 192000;
constexpr long long kMaxLen = 1LL << 40;
constexpr int kTrimThreads = 512, kTrimWarps = kTrimThreads / 32;
constexpr int kTrimRows = 64;   // rows of one trim launch
constexpr int kPackThreads = 256;
constexpr int kPackRows = 128;  // rows of one pack launch

// one row of a trim launch: its samples and the frame geometry of its rate
struct TrimRow {
  const float* x;
  long long n;
  int flen, hop, pad, min_row, min_keep;
};

struct TrimArgs {
  TrimRow r[kTrimRows];
};
static_assert(sizeof(TrimArgs) <= 4000, "the trim's rows fit the kernel parameter space");

struct PackArgs {
  const float* src[kPackRows];
  long long len[kPackRows];
};
static_assert(sizeof(PackArgs) <= 4000, "the pack's rows fit the kernel parameter space");

// The reference's frame geometry, in its double arithmetic (int() truncates the positive products)
TrimRow trim_row(const float* x, long long n, int sr) {
  TrimRow r{};
  r.x = x;
  r.n = n;
  r.flen = std::max(1, (int)(sr * 25.0 / 1000.0));
  r.hop = std::max(1, (int)(sr * 10.0 / 1000.0));
  r.pad = (int)(sr * 30.0 / 1000.0);
  r.min_row = (int)(sr * 0.1);
  r.min_keep = (int)(0.5 * sr);
  return r;
}

// frame k's dB, the same value in every lane
__device__ __forceinline__ double frame_db(const TrimRow& r, long long k, int lane) {
  const float* f = r.x + k * r.hop;
  double s = 0.0;
  for (int i = lane; i < r.flen; i += 32) {
    const double v = (double)__ldg(f + i);
    s = fma(v, v, s);  // v * v is exact: the fma rounds exactly as the separate add would
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return 10.0 * log10(s / (double)r.flen + 1e-10);
}

__global__ void __launch_bounds__(kTrimThreads) trim_kernel(const TrimArgs a, long long* __restrict__ ext) {
  __shared__ double wmax[kTrimWarps];
  __shared__ long long s_first, s_last;
  const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const TrimRow& r = a.r[b];
  const long long n = r.n;
  long long* out = ext + 2LL * b;
  if (n < r.min_row || n < r.flen) {
    if (threadIdx.x == 0) {
      out[0] = 0;
      out[1] = n;
    }
    return;
  }
  const long long K = (n - r.flen) / r.hop + 1;
  double m = -INFINITY;
  for (long long k = warp; k < K; k += kTrimWarps) m = fmax(m, frame_db(r, k, lane));
  if (lane == 0) wmax[warp] = m;
  if (threadIdx.x == 0) {
    s_first = K;
    s_last = -1;
  }
  __syncthreads();
  double mx = wmax[0];
  for (int w = 1; w < kTrimWarps; ++w) mx = fmax(mx, wmax[w]);
  const double thr = fmax(mx - 40.0, -40.0);
  if (mx > thr) {  // the loudest frame is voiced (uniform across the CTA)
    for (long long k0 = 0; k0 < K; k0 += kTrimWarps) {
      const long long k = k0 + warp;
      const bool v = k < K && frame_db(r, k, lane) > thr;
      if (v && lane == 0) atomicMin(&s_first, k);
      if (__syncthreads_or(v)) break;
    }
    for (long long k0 = 0; k0 < K; k0 += kTrimWarps) {
      const long long k = K - 1 - (k0 + warp);
      const bool v = k >= 0 && frame_db(r, k, lane) > thr;
      if (v && lane == 0) atomicMax(&s_last, k);
      if (__syncthreads_or(v)) break;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    long long start = 0, end = n;
    if (s_last >= 0) {
      start = std::max(0LL, s_first * r.hop - r.pad);
      end = std::min(n, s_last * r.hop + r.flen + r.pad);
      if (end - start < r.min_keep) start = 0, end = n;
    }
    out[0] = start;
    out[1] = end;
  }
}

__global__ void __launch_bounds__(kPackThreads) pack_kernel(const PackArgs a, float* __restrict__ dst, long long dst_stride) {
  const int b = blockIdx.y;
  const float* s = a.src[b];
  const long long len = a.len[b];
  float* d = dst + (long long)b * dst_stride;
  for (long long i = (long long)blockIdx.x * kPackThreads + threadIdx.x; i < dst_stride; i += (long long)gridDim.x * kPackThreads)
    d[i] = i < len ? __ldg(s + i) : 0.0f;
}

}  // namespace

extern "C" {

int sopro_ingest_trim(const float* const* rows, int32_t B, const int64_t* lens_host, const int32_t* rates_host, int64_t* ext,
                      void* stream) {
  if (!rows || !lens_host || !rates_host || !ext) return fail(SOPRO_ERR_INVALID, "null argument");
  if (B < 1) return fail(SOPRO_ERR_INVALID, "B = %d < 1", B);
  for (int b = 0; b < B; ++b) {
    if (lens_host[b] < 0 || lens_host[b] > kMaxLen) return fail(SOPRO_ERR_INVALID, "lens[%d] = %lld not in [0, 2^40]", b, (long long)lens_host[b]);
    if (rates_host[b] < kMinRate || rates_host[b] > kMaxRate)
      return fail(SOPRO_ERR_INVALID, "rate of row %d is %d Hz, not in [%d, %d]", b, rates_host[b], kMinRate, kMaxRate);
    if (lens_host[b] > 0 && !rows[b]) return fail(SOPRO_ERR_INVALID, "null row %d", b);
  }
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  for (int b0 = 0; b0 < B; b0 += kTrimRows) {
    const int n = std::min(kTrimRows, B - b0);
    TrimArgs a{};
    for (int i = 0; i < n; ++i) a.r[i] = trim_row(rows[b0 + i], lens_host[b0 + i], rates_host[b0 + i]);
    trim_kernel<<<n, kTrimThreads, 0, st>>>(a, reinterpret_cast<long long*>(ext) + 2LL * b0);
    CK(cudaGetLastError());
  }
  return SOPRO_OK;
}

int sopro_ingest_pack(const float* const* src, int32_t B, const int64_t* lens_host, float* dst, int64_t dst_stride, void* stream) {
  if (!src || !lens_host || !dst) return fail(SOPRO_ERR_INVALID, "null argument");
  if (B < 1 || dst_stride < 1 || dst_stride > kMaxLen) return fail(SOPRO_ERR_INVALID, "bad batch geometry (B=%d, dst_stride=%lld)", B, (long long)dst_stride);
  for (int b = 0; b < B; ++b) {
    if (lens_host[b] < 0 || lens_host[b] > dst_stride)
      return fail(SOPRO_ERR_INVALID, "lens[%d] = %lld not in [0, dst_stride = %lld]", b, (long long)lens_host[b], (long long)dst_stride);
    if (lens_host[b] > 0 && !src[b]) return fail(SOPRO_ERR_INVALID, "null row %d", b);
  }
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const unsigned pieces = (unsigned)std::min<long long>((dst_stride + kPackThreads - 1) / kPackThreads, 1024);
  for (int b0 = 0; b0 < B; b0 += kPackRows) {
    const int n = std::min(kPackRows, B - b0);
    PackArgs a{};
    for (int i = 0; i < n; ++i) {
      a.src[i] = src[b0 + i];
      a.len[i] = lens_host[b0 + i];
    }
    pack_kernel<<<dim3(pieces, n), kPackThreads, 0, st>>>(a, dst + (long long)b0 * dst_stride, dst_stride);
    CK(cudaGetLastError());
  }
  return SOPRO_OK;
}

}  // extern "C"
