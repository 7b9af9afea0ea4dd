// Band-limited resampling of output waveforms (24 kHz -> any supported rate), one-shot and streaming.
//
// The filter is torchaudio.functional.resample's default (sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99,
// rates reduced by their gcd): with o = sr_in / g, n = sr_out / g, base = 0.99 * min(o, n), width = ceil(6 o / base),
// output j = q n + p (phase p) is  sum_i k[p][i] * x[q o - width + i],  x = 0 outside [0, N), for ceil(n N / o) outputs.
// The taps are evaluated on the host in double and rounded to fp32 once; the taps outside the |t| < 6 window round to
// exactly zero, so each phase keeps only its nonzero span [first, first + span).
//
// resample_one() is the only place an output is summed: one fp32 FMA chain over its phase's span, in increasing input
// index.  The one-shot kernel and the stream kernel both call it on the same staged values, which is why a stream's
// outputs equal the one-shot result bit for bit under any chunk schedule.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <numeric>
#include <vector>

#include "../../include/sopro_b200.h"
#include "chunk_stream.cuh"

namespace {

using chunk::Src;
using chunk::src_at;

constexpr int kThreads = 256;
constexpr int kMaxPerThread = 8;         // outputs per thread: tiles of up to 2048 outputs per CTA
constexpr int kMinRate = 4000, kMaxRate = 192000, kMaxReduced = 4096;
constexpr int kTabSmemFloats = 12288;    // a phase table up to 48 KB is staged in shared memory, larger ones read from L2
constexpr int kInSmemFloats = 24576;     // staged input per CTA (96 KB) bounds the tile at extreme ratios
constexpr int kRowsPerLaunch = 256;      // rows of a ragged batch per launch (their lengths travel as a kernel parameter)
// the dynamic shared memory a launch may ask for, set once for both kernels: the attribute is per function, and every
// resampler of the process launches the same two
constexpr int kMaxSmemBytes = 4 * (kInSmemFloats + kTabSmemFloats + 2 + 2 * kMaxReduced);
constexpr double kPi = 3.141592653589793;

struct Geo {
  int o, n, width;  // reduced input / output rates, left context of a block's window
  int S;            // row stride of the tap table (the longest span)
  int tile;         // outputs per CTA
  int tab_smem;     // the tap table and the phase spans are staged in shared memory
};

// rates -> (o, n, width), or a message on refusal.  Pure host arithmetic.
bool reduce_rates(int32_t sr_in, int32_t sr_out, int* o, int* n, int* width, char* why, size_t why_len) {
  if (sr_in < kMinRate || sr_in > kMaxRate || sr_out < kMinRate || sr_out > kMaxRate) {
    snprintf(why, why_len, "sample rates must be integers in [%d, %d] (got %d -> %d)", kMinRate, kMaxRate, sr_in, sr_out);
    return false;
  }
  if (sr_in == sr_out) {
    snprintf(why, why_len, "input and output rates are both %d: nothing to resample", sr_in);
    return false;
  }
  const int g = std::gcd(sr_in, sr_out);
  *o = sr_in / g;
  *n = sr_out / g;
  if (*o > kMaxReduced || *n > kMaxReduced) {
    snprintf(why, why_len, "%d -> %d reduces to %d / %d; both must be <= %d", sr_in, sr_out, *o, *n, kMaxReduced);
    return false;
  }
  const double base = std::min(*o, *n) * 0.99;
  *width = (int)std::ceil(6.0 * *o / base);
  return true;
}

struct Filter {
  int o = 0, n = 0, width = 0, S = 0;
  std::vector<int> first, span;  // per phase
  std::vector<float> taps;       // [n][S], zero past each span
};

// torchaudio's _get_sinc_resample_kernel in double (same operation order), rounded to fp32, zeros trimmed per phase
int make_filter(int32_t sr_in, int32_t sr_out, Filter* f) {
  char why[256];
  if (!reduce_rates(sr_in, sr_out, &f->o, &f->n, &f->width, why, sizeof(why))) return fail(SOPRO_ERR_INVALID, "%s", why);
  const int o = f->o, n = f->n, width = f->width, full = 2 * width + o;
  const double base = std::min(o, n) * 0.99, scale = base / o;
  std::vector<std::vector<float>> rows(n);
  f->first.assign(n, 0);
  f->span.assign(n, 0);
  for (int p = 0; p < n; ++p) {
    // |t| < 6 <=> |(i - width) / o - p / n| < 6 / base: evaluate that range (with a margin), the rest is exactly zero
    const double c = width + (double)o * p / n, h = 6.0 * o / base;
    const int lo = std::max(0, (int)std::floor(c - h) - 2), hi = std::min(full, (int)std::ceil(c + h) + 3);
    std::vector<float> k(hi - lo);
    int a = -1, b = -1;
    for (int i = lo; i < hi; ++i) {
      double t = ((double)(-p) / n + (double)(i - width) / o) * base;
      t = std::min(6.0, std::max(-6.0, t));
      double w = std::cos(t * kPi / 6.0 / 2.0);
      w = w * w;
      t *= kPi;
      const double v = (t == 0.0 ? 1.0 : std::sin(t) / t) * (w * scale);
      k[i - lo] = (float)v;
      if (k[i - lo] != 0.0f) {
        if (a < 0) a = i;
        b = i;
      }
    }
    if (a < 0) return fail(SOPRO_ERR_INVALID, "phase %d of %d -> %d has no nonzero tap", p, sr_in, sr_out);
    f->first[p] = a;
    f->span[p] = b - a + 1;
    rows[p].assign(k.begin() + (a - lo), k.begin() + (b - lo + 1));
    f->S = std::max(f->S, f->span[p]);
  }
  f->taps.assign((size_t)n * f->S, 0.0f);
  for (int p = 0; p < n; ++p) std::copy(rows[p].begin(), rows[p].end(), f->taps.begin() + (size_t)p * f->S);
  return SOPRO_OK;
}

long long out_len(int o, int n, long long n_in) { return (n * n_in + o - 1) / o; }

// One output sample: its phase's nonzero taps against the staged input from the span's first sample on, one fp32 FMA
// chain in increasing input index.  Every output of either kernel is summed here.
__device__ __forceinline__ float resample_one(const float* __restrict__ tap, int span, const float* __restrict__ xs) {
  float acc = 0.0f;
#pragma unroll 4
  for (int s = 0; s < span; ++s) acc = fmaf(tap[s], xs[s], acc);
  return acc;
}

// Outputs [j0, j0 + tile) ∩ [.., j_end) of this CTA, j0 = j_begin + blockIdx.x * tile, written to y[j - j_begin].  The
// input window of those blocks (and, when it fits, the tap table) is staged in shared memory with coalesced loads.
__device__ __forceinline__ void resample_tile(const Geo& g, const float* __restrict__ tab_g, const int2* __restrict__ meta_g,
                                              const Src& src, long long j_begin, long long j_end, float* __restrict__ y) {
  extern __shared__ float4 smem4[];
  float* sm = reinterpret_cast<float*>(smem4);
  const long long j0 = j_begin + (long long)blockIdx.x * g.tile;
  if (j0 >= j_end) return;
  const long long j1 = min(j0 + (long long)g.tile, j_end);
  const long long q0 = j0 / g.n, q1 = (j1 - 1) / g.n;
  const long long in0 = q0 * g.o - g.width;
  const int in_len = (int)(q1 - q0) * g.o + 2 * g.width + g.o;
  const float* tab = tab_g;
  const int2* meta = meta_g;
  float* xs = sm;
  if (g.tab_smem) {
    const int tn = (g.n * g.S + 1) & ~1;  // keeps the int2 spans 8-byte aligned
    float* ts = sm;
    int2* ms = reinterpret_cast<int2*>(sm + tn);
    for (int i = threadIdx.x; i < g.n * g.S; i += kThreads) ts[i] = tab_g[i];
    for (int i = threadIdx.x; i < g.n; i += kThreads) ms[i] = meta_g[i];
    tab = ts;
    meta = ms;
    xs = reinterpret_cast<float*>(ms + g.n);
  }
  for (int i = threadIdx.x; i < in_len; i += kThreads) xs[i] = src_at(src, in0 + i);
  __syncthreads();
  const int count = (int)(j1 - j0), r0 = (int)(j0 - q0 * g.n);
  float* yt = y + (j0 - j_begin);
  for (int r = threadIdx.x; r < count; r += kThreads) {
    const int jl = r0 + r;  // output index from block q0's first output on
    const int ql = jl / g.n, p = jl - ql * g.n;
    const int2 m = meta[p];  // (first nonzero tap, span)
    yt[r] = resample_one(tab + (size_t)p * g.S, m.y, xs + ql * g.o + m.x);
  }
}

// one-shot, ragged batch: grid (tiles of the longest row, rows); row b reads x[b][0, lens[b]) only
__global__ void __launch_bounds__(kThreads) resample_batch_kernel(Geo g, const float* __restrict__ tab, const int2* __restrict__ meta,
                                                                  const float* __restrict__ x, long long x_stride, RowLens<kRowsPerLaunch> lens,
                                                                  float* __restrict__ y, long long y_stride) {
  const int b = blockIdx.y;
  const long long len = lens.v[b];
  const Src s{x + (long long)b * x_stride, nullptr, 0, len, len};
  resample_tile(g, tab, meta, s, 0, (g.n * len + g.o - 1) / g.o, y + (long long)b * y_stride);
}

// stream: outputs [j_begin, j_end) of one utterance from its carried tail and the new chunk
__global__ void __launch_bounds__(kThreads) resample_stream_kernel(Geo g, const float* __restrict__ tab, const int2* __restrict__ meta,
                                                                   Src s, long long j_begin, long long j_end, float* __restrict__ y) {
  resample_tile(g, tab, meta, s, j_begin, j_end, y);
}

size_t smem_bytes(const Geo& g) {
  const size_t in = (size_t)((g.tile - 1) / g.n + 1) * g.o + 2 * g.width + g.o;
  return 4 * (in + (g.tab_smem ? (size_t)((g.n * g.S + 1) & ~1) + 2 * (size_t)g.n : 0));
}

}  // namespace

struct sopro_resampler {
  int device = 0;
  Geo g{};
  float* tab = nullptr;  // [n][S]
  int2* meta = nullptr;  // [n] (first, span)
  size_t smem = 0;
};

// the tail holds the logical input [q_done * o - width, n_seen) of the utterance
struct sopro_resampler_stream : chunk::ChunkStream {
  sopro_resampler* r = nullptr;
  long long q_done = 0;  // blocks of n outputs emitted
};

namespace {
long long blocks_ready(const Geo& g, long long n_seen) { return std::max(0LL, (n_seen - g.width) / g.o); }

int launch_stream(sopro_resampler_stream_t* s, const Src& src, long long j_begin, long long j_end, float* y, cudaStream_t st) {
  const Geo& g = s->r->g;
  if (j_end <= j_begin) return SOPRO_OK;
  const unsigned tiles = (unsigned)((j_end - j_begin + g.tile - 1) / g.tile);
  resample_stream_kernel<<<tiles, kThreads, s->r->smem, st>>>(g, s->r->tab, s->r->meta, src, j_begin, j_end, y);
  CK(cudaGetLastError());
  return SOPRO_OK;
}
}  // namespace

extern "C" {

int sopro_resampler_filter(int32_t sr_in, int32_t sr_out, int32_t* geometry, int32_t* first, int32_t* span, float* taps) {
  if (!geometry) return fail(SOPRO_ERR_INVALID, "null argument");
  Filter f;
  const int rc = make_filter(sr_in, sr_out, &f);
  if (rc != SOPRO_OK) return rc;
  geometry[0] = f.o;
  geometry[1] = f.n;
  geometry[2] = f.width;
  geometry[3] = f.S;
  if (first) std::copy(f.first.begin(), f.first.end(), first);
  if (span) std::copy(f.span.begin(), f.span.end(), span);
  if (taps) std::copy(f.taps.begin(), f.taps.end(), taps);
  return SOPRO_OK;
}

int64_t sopro_resampled_length(int32_t sr_in, int32_t sr_out, int64_t n_in) {
  int o, n, w;
  char why[256];
  if (n_in < 0 || n_in > (1LL << 40) || !reduce_rates(sr_in, sr_out, &o, &n, &w, why, sizeof(why))) return -1;
  return out_len(o, n, n_in);
}

int sopro_resampler_create(int32_t sr_in, int32_t sr_out, int device, sopro_resampler_t** out) {
  if (!out) return fail(SOPRO_ERR_INVALID, "null argument");
  *out = nullptr;
  Filter f;
  int rc = make_filter(sr_in, sr_out, &f);  // refuses a rate before anything touches the device
  if (rc == SOPRO_OK) rc = open_device(device, "the resampler");
  if (rc != SOPRO_OK) return rc;
  Geo g{f.o, f.n, f.width, f.S, 0, f.n * f.S <= kTabSmemFloats ? 1 : 0};
  for (int per = kMaxPerThread; per >= 1; per /= 2) {  // the largest tile whose input window fits the staging budget
    g.tile = per * kThreads;
    if ((long long)((g.tile - 1) / g.n + 1) * g.o + 2 * g.width + g.o <= kInSmemFloats) break;
  }
  std::vector<int2> meta(f.n);
  for (int p = 0; p < f.n; ++p) meta[p] = make_int2(f.first[p], f.span[p]);
  sopro_resampler* r = new sopro_resampler();
  r->device = device;
  r->g = g;
  r->smem = smem_bytes(g);
  cudaError_t e = cudaMalloc(&r->tab, f.taps.size() * 4);
  if (e == cudaSuccess) e = cudaMalloc(&r->meta, meta.size() * sizeof(int2));
  if (e == cudaSuccess) e = cudaMemcpy(r->tab, f.taps.data(), f.taps.size() * 4, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(r->meta, meta.data(), meta.size() * sizeof(int2), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(resample_batch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmemBytes);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(resample_stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmemBytes);
  if (e != cudaSuccess) {
    cudaFree(r->tab);
    cudaFree(r->meta);
    delete r;
    return fail(SOPRO_ERR_CUDA, "resampler setup failed: %s", cudaGetErrorString(e));
  }
  *out = r;
  return SOPRO_OK;
}

int sopro_resampler_destroy(sopro_resampler_t* r) {
  if (!r) return SOPRO_OK;
  cudaSetDevice(r->device);
  cudaFree(r->tab);
  cudaFree(r->meta);
  delete r;
  return SOPRO_OK;
}

int sopro_resample(sopro_resampler_t* r, const float* x, int32_t B, int64_t x_stride, const int64_t* lens_host, float* y,
                   int64_t y_stride, void* stream) {
  if (!r || !x || !y) return fail(SOPRO_ERR_INVALID, "null argument");
  const Geo& g = r->g;
  long long most = 0;
  int rc = check_rows(x, B, x_stride, lens_host, 1LL << 40, &most);
  if (rc != SOPRO_OK) return rc;
  most = out_len(g.o, g.n, most);  // out_len is monotone in the row length
  if ((rc = check_out_rows(y, B, y_stride, most)) != SOPRO_OK) return rc;
  if (most == 0) return SOPRO_OK;
  CK(cudaSetDevice(r->device));
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const unsigned tiles = (unsigned)((most + g.tile - 1) / g.tile);
  for (int b0 = 0; b0 < B; b0 += kRowsPerLaunch) {
    const int rows = std::min(kRowsPerLaunch, B - b0);
    resample_batch_kernel<<<dim3(tiles, rows), kThreads, r->smem, st>>>(g, r->tab, r->meta, x + (long long)b0 * x_stride, x_stride,
                                                                        row_lens<kRowsPerLaunch>(lens_host, x_stride, b0, rows),
                                                                        y + (long long)b0 * y_stride, y_stride);
    CK(cudaGetLastError());
  }
  return SOPRO_OK;
}

int sopro_resampler_stream_create(sopro_resampler_t* r, int64_t max_chunk, sopro_resampler_stream_t** out) {
  if (!r) return fail(SOPRO_ERR_INVALID, "null argument");
  const int rc = chunk::check_create(max_chunk, out);
  if (rc != SOPRO_OK) return rc;
  CK(cudaSetDevice(r->device));
  sopro_resampler_stream* s = new sopro_resampler_stream();
  s->r = r;
  s->restart(-r->g.width);
  // the carried tail is always shorter than 2 width + o (header)
  return chunk::create(s, max_chunk, (size_t)(2 * r->g.width + r->g.o), "resampler", out);
}

int sopro_resampler_stream_destroy(sopro_resampler_stream_t* s) { return chunk::destroy(s); }

int sopro_resampler_stream_reset(sopro_resampler_stream_t* s) {
  if (!s) return fail(SOPRO_ERR_INVALID, "null argument");
  s->restart(-s->r->g.width);
  s->q_done = 0;
  return SOPRO_OK;
}

int64_t sopro_resampler_stream_ready(const sopro_resampler_stream_t* s, int64_t n_more, int final) {
  if (!chunk::can_run(s, n_more)) return -1;
  const Geo& g = s->r->g;
  const long long done = (long long)g.n * s->q_done;
  if (final) return out_len(g.o, g.n, s->tail.seen + n_more) - done;
  return (long long)g.n * blocks_ready(g, s->tail.seen + n_more) - done;
}

int sopro_resampler_push(sopro_resampler_stream_t* s, const float* x, int64_t n, float* y, void* stream) {
  int rc = chunk::check_push(s, n);
  if (rc != SOPRO_OK || n == 0) return rc;
  const Geo& g = s->r->g;
  const long long q_done = blocks_ready(g, s->tail.seen + n);
  if ((rc = chunk::check_io(x, n, y, q_done - s->q_done)) != SOPRO_OK) return rc;
  CK(cudaSetDevice(s->tail.device));
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  rc = launch_stream(s, s->tail.src(x, n), (long long)g.n * s->q_done, (long long)g.n * q_done, y, st);
  if (rc == SOPRO_OK) rc = s->tail.keep(q_done * g.o - g.width, x, n, st);
  if (rc != SOPRO_OK) return rc;
  s->q_done = q_done;
  return SOPRO_OK;
}

int sopro_resampler_finish(sopro_resampler_stream_t* s, float* y, void* stream) {
  int rc = chunk::check_finish(s);
  if (rc != SOPRO_OK) return rc;
  const Geo& g = s->r->g;
  const long long j_end = out_len(g.o, g.n, s->tail.seen), j_begin = (long long)g.n * s->q_done;
  if ((rc = chunk::check_io(nullptr, 0, y, j_end - j_begin)) != SOPRO_OK) return rc;
  CK(cudaSetDevice(s->tail.device));
  rc = launch_stream(s, s->tail.src(nullptr, 0), j_begin, j_end, y, reinterpret_cast<cudaStream_t>(stream));
  if (rc != SOPRO_OK) return rc;
  s->finished = true;
  return SOPRO_OK;
}

}  // extern "C"
