// Long-form synthesis: the speech extent of each segment's decoded row, and the join of those extents into one waveform.
// The definition (include/sopro_b200.h, oracle/longform_oracle.py in float64), at the codec's 24 kHz:
//   extents: the energy trim of sopro_b200.audio.trim_silence_energy.  Frames of 600 samples every 240,
//     K = floor((n - 600) / 240) + 1; e_k = sum x^2 / 600, dB_k = 10 log10(e_k + 1e-10) in fp64; thr = max(max dB - 40,
//     -40); frame k is voiced when dB_k > thr; start = max(0, first 240 - 720), end = min(n, last 240 + 600 + 720).
//     The row is left whole, (0, n), when n < 2400, nothing is voiced, or end - start < 12000.
//   join: for each non-empty extent in order, x[start, end) with a raised-cosine fade over its first and last
//     F = min(240, floor(span / 2)) samples, f[i] = 0.5 - 0.5 cos(pi (i + 0.5) / F) (double on the host, fp32 once; one
//     fp32 multiply per faded sample), and P zero samples between consecutive spans.  The general join takes a P per gap
//     and an optional gain per span, y = g * (f * x): the faded product rounded first, then one more fp32 multiply, as
//     the loudness stage scales an already-joined row.
//
// extents_kernel: one CTA per row.  A warp computes a frame: lane l sums x^2 over the frame's samples l, l + 32, ... in
// order (each product is exact in fp64), then a butterfly; every frame's dB therefore has one fixed value whatever the
// batch.  Pass 1 takes the maximum; pass 2 looks for the first voiced frame in rounds of one frame per warp from the
// start, and the last from the end, stopping at the first round that finds one.
// join_kernel: grid (pieces, segments); the segments of one launch share their F, and their fade table travels in the
// kernel parameters with the source pointers, so nothing is copied to the device first.
// The timeline mix (timed synthesis) is the last part of the file.
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
  int seg;           // the segment's index into the gains
};

struct JoinArgs {
  float f[kFadeMax];
  int F, nseg;
  JoinSeg s[kSegsPerLaunch];
};
static_assert(sizeof(JoinArgs) <= 4000, "the join's arguments fit the kernel parameter space");

__global__ void __launch_bounds__(kJoinThreads) join_kernel(const JoinArgs a, const float* __restrict__ gain, float* __restrict__ y) {
  const JoinSeg s = a.s[blockIdx.y];
  const long long total = s.span + s.pause;
  const float g = gain ? __ldg(gain + s.seg) : 1.0f;
  float* yo = y + s.off;
  for (long long j = (long long)blockIdx.x * kJoinThreads + threadIdx.x; j < total; j += (long long)gridDim.x * kJoinThreads) {
    float v = 0.0f;
    if (j < s.span) {
      v = __ldg(s.src + j);
      if (j < a.F)
        v = __fmul_rn(v, a.f[j]);
      else if (j >= s.span - a.F)
        v = __fmul_rn(v, a.f[s.span - 1 - j]);
      if (gain) v = __fmul_rn(g, v);
    }
    yo[j] = v;
  }
}

void fade(int F, float* f) {
  for (int i = 0; i < F; ++i) f[i] = (float)(0.5 - 0.5 * std::cos(kPi * (i + 0.5) / F));
}

int fade_len(long long span) { return (int)std::min<long long>(kFadeMax, span / 2); }

// ---- the streaming trim (include/sopro_b200.h): each row's samples as they are decoded, its frames classified once
// under the causal threshold, and the certain prefix of its extent published after every push.
// push_kernel: one CTA per row.  The CTA appends the row's new samples to its buffer, then, after a barrier, computes
// the newly complete frames in rounds of kPushRound, one warp per frame through frame_db (so every dB equals the
// one-shot kernel's), and one thread walks the round in frame order updating M, first and last.  Each frame reads only
// samples of its own row that are stored before the barrier by this CTA or by an earlier launch; no load of the row's
// buffer precedes the barrier, so the read-only path never holds a line older than the stores.
// emit_kernel: grid (pieces, items); a piece is a run of a span (faded as join_kernel fades it) or of pause zeros.
constexpr int kMaxStreamRows = 256;     // rows of one state (their counts travel as a kernel parameter)
constexpr int kPushRound = 256;         // frames per classification round
constexpr int kEmitPieces = 48;         // pieces of one emit launch
constexpr long long kMaxStreamLen = 1LL << 31;
constexpr long long kNoTail = 1LL << 62;

struct TrimRow {
  long long n;      // samples appended
  long long K;      // complete frames classified
  long long first, last;  // voiced frames (-1: none)
  double M;         // the largest dB among frames 0 .. K-1
  int final_;
};

// status row: n, decided, start, available bound, final (see the header)
constexpr int kStatus = 5;

struct PushArgs {
  long long count[kMaxStreamRows];
  unsigned char fin[kMaxStreamRows];
};
static_assert(sizeof(PushArgs) <= 4000, "the push's arguments fit the kernel parameter space");

__global__ void trim_reset_kernel(TrimRow* __restrict__ rows, long long* __restrict__ status, int n_rows) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n_rows) return;
  rows[b] = TrimRow{0, 0, -1, -1, -INFINITY, 0};
  for (int i = 0; i < kStatus; ++i) status[kStatus * b + i] = 0;
}

__global__ void __launch_bounds__(kExtThreads) push_kernel(const float* __restrict__ x, long long x_stride, const PushArgs a,
                                                           float* __restrict__ buf, long long cap, TrimRow* __restrict__ rows,
                                                           long long* __restrict__ status) {
  __shared__ double db[kPushRound];
  __shared__ TrimRow s;
  const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* xb = buf + (long long)b * cap;
  if (threadIdx.x == 0) s = rows[b];
  __syncthreads();
  const long long n0 = s.n, cnt = a.count[b], n = n0 + cnt;
  const float* src = x + (long long)b * x_stride;
  for (long long i = threadIdx.x; i < cnt; i += kExtThreads) xb[n0 + i] = src[i];
  __syncthreads();
  const long long K = n >= kFrame ? (n - kFrame) / kHop + 1 : 0;
  for (long long k0 = s.K; k0 < K; k0 += kPushRound) {
    const int m = (int)std::min<long long>(kPushRound, K - k0);
    for (int j = warp; j < m; j += kExtWarps) {
      const double v = frame_db(xb, k0 + j, lane);
      if (lane == 0) db[j] = v;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int j = 0; j < m; ++j) {  // frame k against thr_k = max(M_k - 40, -40), M_k over frames 0 .. k
        s.M = fmax(s.M, db[j]);
        if (db[j] > fmax(s.M - 40.0, -40.0)) {
          if (s.first < 0) s.first = k0 + j;
          s.last = k0 + j;
        }
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    s.n = n;
    s.K = K;
    s.final_ = s.final_ | a.fin[b];
    long long decided = 0, start = 0, avail = 0;
    const long long st = std::max(0LL, s.first * kHop - kPad);
    const long long end = s.last >= 0 ? std::min(n, s.last * kHop + kFrame + kPad) : 0;
    if (s.final_) {
      decided = 1;
      start = st;
      avail = end;
      if (n < kMinRow || s.last < 0 || end - st < kMinKeep) start = 0, avail = n;
    } else if (s.last >= 0 && end - st >= kMinKeep) {
      decided = 1;
      start = st;
      avail = end - kFadeMax;  // the fade-out may only touch the last 240 samples of the final extent
    }
    rows[b] = s;
    long long* o = status + kStatus * b;
    o[0] = n;
    o[1] = decided;
    o[2] = start;
    o[3] = avail;
    o[4] = s.final_;
  }
}

struct EmitPiece {
  const float* src;  // the row's buffer + the span's start; null for pause zeros
  long long j0, len, off;
  long long tail;    // span - F: the fade-out's first position (kNoTail while the span's end is unknown)
  int F;
};

struct EmitArgs {
  int n;
  EmitPiece p[kEmitPieces];
};
static_assert(sizeof(EmitArgs) <= 4000, "the emit's arguments fit the kernel parameter space");

__global__ void __launch_bounds__(kJoinThreads) emit_kernel(const EmitArgs a, const float* __restrict__ fades, float* __restrict__ y) {
  const EmitPiece p = a.p[blockIdx.y];
  const float* f = fades + (long long)p.F * (p.F - 1) / 2;  // the table of fade length F
  float* yo = y + p.off;
  for (long long i = (long long)blockIdx.x * kJoinThreads + threadIdx.x; i < p.len; i += (long long)gridDim.x * kJoinThreads) {
    float v = 0.0f;
    if (p.src) {
      const long long j = p.j0 + i;
      v = p.src[j];
      if (j < p.F)
        v = __fmul_rn(v, __ldg(f + j));
      else if (j >= p.tail)
        v = __fmul_rn(v, __ldg(f + (p.tail + p.F - 1 - j)));
    }
    yo[i] = v;
  }
}

// ---- the timeline mix (include/sopro_b200.h, sopro_timeline_mix): items placed at absolute offsets and summed where
// they overlap, y[t] = the first covering item's sample, then each later one added in item order.
// mix_kernel: one CTA per output tile of kMixTile samples, over a grid-stride range of tiles.  The host lists each
// tile's covering items in item order (a CSR); thread i owns samples i, i + 256, ... of the tile and keeps their sums in
// registers while it walks the list, so every sample's adds happen in item order whatever the tiling.
constexpr int kMixThreads = 256;
constexpr int kMixPer = 16;                         // samples per thread
constexpr int kMixTile = kMixThreads * kMixPer;     // 4096
constexpr int kMixMaxCtas = 4096;

struct MixItem {
  const float* src;
  long long off, len;
};

__global__ void __launch_bounds__(kMixThreads) mix_kernel(const MixItem* __restrict__ items, const long long* __restrict__ ptr,
                                                          const int* __restrict__ idx, long long n_tiles, float* __restrict__ y,
                                                          long long y_len) {
  for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const long long base = tile * kMixTile + threadIdx.x;
    float acc[kMixPer];
    unsigned have = 0;  // bit k: sample k has its first item
#pragma unroll
    for (int k = 0; k < kMixPer; ++k) acc[k] = 0.0f;
    const long long e = __ldg(ptr + tile + 1);
    for (long long j = __ldg(ptr + tile); j < e; ++j) {
      const MixItem it = items[__ldg(idx + j)];
      const long long lo = it.off, hi = it.off + it.len;
#pragma unroll
      for (int k = 0; k < kMixPer; ++k) {
        const long long t = base + (long long)k * kMixThreads;
        if (t >= lo && t < hi) {
          const float v = __ldg(it.src + (t - lo));
          acc[k] = (have >> k & 1u) ? __fadd_rn(acc[k], v) : v;
          have |= 1u << k;
        }
      }
    }
#pragma unroll
    for (int k = 0; k < kMixPer; ++k) {
      const long long t = base + (long long)k * kMixThreads;
      if (t < y_len) y[t] = acc[k];
    }
  }
}

}  // namespace

struct sopro_longform_stream {
  int rows = 0, device = 0;
  long long cap = 0;
  float* buf = nullptr;       // [rows][cap]
  float* fades = nullptr;     // the fade tables of F = 1 .. 240, back to back
  TrimRow* state = nullptr;   // [rows]
  long long* status = nullptr;  // [rows][5]
  std::vector<long long> n;   // host mirror of the samples pushed per row
  std::vector<char> fin;      // host mirror of the final flags
};

namespace {

int check_rows_range(const sopro_longform_stream* s, int row0, int n_rows) {
  if (!s) return fail(SOPRO_ERR_INVALID, "null argument");
  if (row0 < 0 || n_rows < 1 || row0 + n_rows > s->rows)
    return fail(SOPRO_ERR_INVALID, "rows [%d, %d) not inside the state's %d rows", row0, row0 + n_rows, s->rows);
  return SOPRO_OK;
}

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

int sopro_longform_join_gaps(const float* const* src, int32_t n_seg, const int64_t* lens_host, const int64_t* ext_host,
                             const int64_t* pauses_host, const float* gain, float* y, int64_t y_len, void* stream) {
  if (!src || !lens_host || !ext_host) return fail(SOPRO_ERR_INVALID, "null argument");
  if (n_seg < 1) return fail(SOPRO_ERR_INVALID, "n_seg = %d < 1", n_seg);
  long long total = 0, last = -1, spans = 0;
  for (int i = 0; i < n_seg; ++i) {
    const long long len = lens_host[i], s = ext_host[2 * i], e = ext_host[2 * i + 1];
    if (len < 0 || len > kMaxLen) return fail(SOPRO_ERR_INVALID, "lens[%d] = %lld not in [0, 2^40]", i, len);
    if (s < 0 || s > e || e > len)
      return fail(SOPRO_ERR_INVALID, "extent [%lld, %lld) of segment %d is not inside its %lld samples", s, e, i, len);
    if (e > s && !src[i]) return fail(SOPRO_ERR_INVALID, "null source for segment %d", i);
    if (e > s) {
      if (last >= 0) {
        if (!pauses_host) return fail(SOPRO_ERR_INVALID, "null argument");
        const long long p = pauses_host[spans - 1];
        if (p < 0 || p > kMaxPause)
          return fail(SOPRO_ERR_INVALID, "pause %lld of %lld samples not in [0, %lld]", spans - 1, p, kMaxPause);
        total += p;
      }
      total += e - s;
      last = i;
      ++spans;
    }
  }
  if (y_len != total) return fail(SOPRO_ERR_INVALID, "y_len = %lld, the joined length is %lld", (long long)y_len, total);
  if (total == 0) return SOPRO_OK;
  if (!y) return fail(SOPRO_ERR_INVALID, "null argument");
  // each span's place in y and the pause after it, then one launch per (fade length, run of at most kSegsPerLaunch
  // segments)
  std::vector<long long> off(n_seg, 0), after(n_seg, 0);
  std::vector<char> done(n_seg, 1);
  for (long long i = 0, o = 0, m = 0; i < n_seg; ++i) {
    const long long span = ext_host[2 * i + 1] - ext_host[2 * i];
    if (span == 0) continue;
    off[i] = o;
    after[i] = i == last ? 0 : pauses_host[m++];
    o += span + after[i];
    done[i] = 0;
  }
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  JoinArgs a{};
  long long most = 0;  // the longest span + pause of the pending launch
  auto launch = [&]() -> int {
    const unsigned gx = (unsigned)std::min<long long>((most + kJoinThreads - 1) / kJoinThreads, 1024);
    join_kernel<<<dim3(gx, a.nseg), kJoinThreads, 0, st>>>(a, gain, y);
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
      s.pause = after[j];
      s.seg = j;
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

int sopro_longform_join(const float* const* src, int32_t n_seg, const int64_t* lens_host, const int64_t* ext_host, int64_t pause,
                        float* y, int64_t y_len, void* stream) {
  if (pause < 0 || pause > kMaxPause) return fail(SOPRO_ERR_INVALID, "pause of %lld samples not in [0, %lld]", (long long)pause, kMaxPause);
  const std::vector<int64_t> pauses(std::max(n_seg, 1), pause);
  return sopro_longform_join_gaps(src, n_seg, lens_host, ext_host, pauses.data(), nullptr, y, y_len, stream);
}

int sopro_longform_stream_destroy(sopro_longform_stream_t* s) {
  if (!s) return SOPRO_OK;
  cudaFree(s->buf);
  cudaFree(s->fades);
  cudaFree(s->state);
  cudaFree(s->status);
  delete s;
  return SOPRO_OK;
}

int sopro_longform_stream_create(int32_t rows, int64_t max_len, int device, sopro_longform_stream_t** out) {
  if (!out) return fail(SOPRO_ERR_INVALID, "null argument");
  *out = nullptr;
  if (rows < 1 || rows > kMaxStreamRows) return fail(SOPRO_ERR_INVALID, "rows = %d not in [1, %d]", rows, kMaxStreamRows);
  if (max_len < 1 || max_len > kMaxStreamLen)
    return fail(SOPRO_ERR_INVALID, "max_len = %lld not in [1, 2^31]", (long long)max_len);
  const int rc = open_device(device, "the streaming trim");
  if (rc != SOPRO_OK) return rc;
  auto* s = new sopro_longform_stream;
  s->rows = rows;
  s->device = device;
  s->cap = (max_len + 31) / 32 * 32;  // every row starts on a 128-byte line
  s->n.assign(rows, 0);
  s->fin.assign(rows, 0);
  std::vector<float> fades((size_t)kFadeMax * (kFadeMax + 1) / 2);
  for (int F = 1; F <= kFadeMax; ++F) fade(F, fades.data() + (size_t)F * (F - 1) / 2);
  const cudaError_t e[] = {cudaMalloc(&s->buf, sizeof(float) * (size_t)rows * s->cap),
                           cudaMalloc(&s->fades, sizeof(float) * fades.size()),
                           cudaMalloc(&s->state, sizeof(TrimRow) * rows),
                           cudaMalloc(&s->status, sizeof(long long) * kStatus * rows)};
  for (cudaError_t ei : e)
    if (ei != cudaSuccess) {
      sopro_longform_stream_destroy(s);
      return fail(SOPRO_ERR_CUDA, "cudaMalloc failed: %s (streaming trim of %d rows x %lld samples)", cudaGetErrorString(ei),
                  rows, (long long)max_len);
    }
  cudaError_t ec = cudaMemcpy(s->fades, fades.data(), sizeof(float) * fades.size(), cudaMemcpyHostToDevice);
  if (ec == cudaSuccess) {
    trim_reset_kernel<<<(rows + 127) / 128, 128>>>(s->state, s->status, rows);
    ec = cudaGetLastError();
  }
  if (ec == cudaSuccess) ec = cudaDeviceSynchronize();
  if (ec != cudaSuccess) {
    sopro_longform_stream_destroy(s);
    return fail(SOPRO_ERR_CUDA, "streaming trim set-up failed: %s", cudaGetErrorString(ec));
  }
  *out = s;
  return SOPRO_OK;
}

int sopro_longform_stream_reset(sopro_longform_stream_t* s, int32_t row0, int32_t n_rows, void* stream) {
  const int rc = check_rows_range(s, row0, n_rows);
  if (rc != SOPRO_OK) return rc;
  trim_reset_kernel<<<(n_rows + 127) / 128, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(s->state + row0,
                                                                                            s->status + kStatus * row0, n_rows);
  CK(cudaGetLastError());
  for (int b = row0; b < row0 + n_rows; ++b) s->n[b] = 0, s->fin[b] = 0;
  return SOPRO_OK;
}

int sopro_longform_stream_push(sopro_longform_stream_t* s, const float* x, int64_t x_stride, int32_t row0, int32_t n_rows,
                               const int64_t* counts_host, const int32_t* final_host, void* stream) {
  int rc = check_rows_range(s, row0, n_rows);
  if (rc != SOPRO_OK) return rc;
  if (!counts_host || !final_host) return fail(SOPRO_ERR_INVALID, "null argument");
  PushArgs a{};
  long long most = 0;
  for (int i = 0; i < n_rows; ++i) {
    const int b = row0 + i;
    const long long c = counts_host[i];
    if (c < 0 || c > s->cap - s->n[b])
      return fail(SOPRO_ERR_INVALID, "row %d: %lld samples after %lld exceed the capacity %lld", b, c, s->n[b], s->cap);
    if (s->fin[b] && (c > 0 || final_host[i]))
      return fail(SOPRO_ERR_INVALID, "row %d is final: it takes no more samples until a reset", b);
    a.count[i] = c;
    a.fin[i] = final_host[i] ? 1 : 0;
    most = std::max(most, c);
  }
  if (most > 0 && !x) return fail(SOPRO_ERR_INVALID, "null argument");
  if (n_rows > 1 && x_stride < most)
    return fail(SOPRO_ERR_INVALID, "x_stride %lld < the largest count %lld", (long long)x_stride, most);
  push_kernel<<<n_rows, kExtThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, x_stride, a, s->buf + (long long)row0 * s->cap, s->cap, s->state + row0, s->status + kStatus * row0);
  CK(cudaGetLastError());
  for (int i = 0; i < n_rows; ++i) {
    s->n[row0 + i] += a.count[i];
    s->fin[row0 + i] |= (char)a.fin[i];
  }
  return SOPRO_OK;
}

int sopro_longform_stream_status(const sopro_longform_stream_t* s, int32_t row0, int32_t n_rows, int64_t* status_host,
                                 void* stream) {
  const int rc = check_rows_range(s, row0, n_rows);
  if (rc != SOPRO_OK) return rc;
  if (!status_host) return fail(SOPRO_ERR_INVALID, "null argument");
  CK(cudaMemcpyAsync(status_host, s->status + kStatus * row0, sizeof(long long) * kStatus * n_rows, cudaMemcpyDeviceToHost,
                     reinterpret_cast<cudaStream_t>(stream)));
  return SOPRO_OK;
}

int sopro_longform_stream_emit(const sopro_longform_stream_t* s, const int64_t* pieces_host, int32_t n_pieces, float* y,
                               int64_t y_len, void* stream) {
  if (!s || !pieces_host) return fail(SOPRO_ERR_INVALID, "null argument");
  if (n_pieces < 0) return fail(SOPRO_ERR_INVALID, "n_pieces = %d < 0", n_pieces);
  long long total = 0;
  for (int i = 0; i < n_pieces; ++i) {
    const int64_t* q = pieces_host + 5 * i;
    const long long row = q[0], a = q[1], b = q[2], st = q[3], e = q[4];
    if (row < -1 || row >= s->rows) return fail(SOPRO_ERR_INVALID, "piece %d: row %lld not in [-1, %d)", i, row, s->rows);
    if (row == -1) {
      if (a != 0 || b < 0 || b > kMaxPause) return fail(SOPRO_ERR_INVALID, "piece %d: a pause of [%lld, %lld)", i, a, b);
    } else {
      const long long n = s->n[row];
      if (st < 0 || st > a || a > b || b > n || (e >= 0 && (e < b || e > n)) || e < -1)
        return fail(SOPRO_ERR_INVALID, "piece %d: samples [%lld, %lld) of the span [%lld, %lld) of row %lld (%lld pushed)", i, a,
                    b, st, e, row, n);
    }
    total += b - a;
  }
  if (y_len != total) return fail(SOPRO_ERR_INVALID, "y_len = %lld, the pieces hold %lld", (long long)y_len, total);
  if (total == 0) return SOPRO_OK;
  if (!y) return fail(SOPRO_ERR_INVALID, "null argument");
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  EmitArgs args{};
  long long most = 0, off = 0;
  for (int i = 0; i < n_pieces; ++i) {
    const int64_t* q = pieces_host + 5 * i;
    const long long row = q[0], len = q[2] - q[1];
    if (len == 0) continue;
    EmitPiece& p = args.p[args.n++];
    p.len = len;
    p.off = off;
    off += len;
    if (row < 0) {
      p.src = nullptr;
      p.j0 = 0;
      p.tail = kNoTail;
      p.F = 0;
    } else {
      const long long start = q[3], end = q[4];
      p.src = s->buf + row * s->cap + start;
      p.j0 = q[1] - start;
      p.F = end < 0 ? kFadeMax : fade_len(end - start);  // an undecided end belongs to a span of >= 12000 samples
      p.tail = end < 0 ? kNoTail : end - start - p.F;
    }
    most = std::max(most, len);
    if (args.n == kEmitPieces) {
      const unsigned gx = (unsigned)std::min<long long>((most + kJoinThreads - 1) / kJoinThreads, 1024);
      emit_kernel<<<dim3(gx, args.n), kJoinThreads, 0, st>>>(args, s->fades, y);
      CK(cudaGetLastError());
      args.n = 0;
      most = 0;
    }
  }
  if (args.n > 0) {
    const unsigned gx = (unsigned)std::min<long long>((most + kJoinThreads - 1) / kJoinThreads, 1024);
    emit_kernel<<<dim3(gx, args.n), kJoinThreads, 0, st>>>(args, s->fades, y);
    CK(cudaGetLastError());
  }
  return SOPRO_OK;
}

int sopro_timeline_mix(const float* const* src, int32_t n_items, const int64_t* lens_host, const int64_t* offs_host, float* y,
                       int64_t y_len, void* stream) {
  if (n_items < 0) return fail(SOPRO_ERR_INVALID, "n_items = %d < 0", n_items);
  if (y_len < 0 || y_len > kMaxLen) return fail(SOPRO_ERR_INVALID, "y_len = %lld not in [0, 2^40]", (long long)y_len);
  if (n_items > 0 && (!src || !lens_host || !offs_host)) return fail(SOPRO_ERR_INVALID, "null argument");
  const long long n_tiles = (y_len + kMixTile - 1) / kMixTile;
  std::vector<long long> ptr(n_tiles + 1, 0);
  for (int i = 0; i < n_items; ++i) {
    const long long len = lens_host[i], off = offs_host[i];
    if (len < 0 || off < 0) return fail(SOPRO_ERR_INVALID, "item %d: length %lld, offset %lld (both must be >= 0)", i, len, off);
    if (off > y_len - len)
      return fail(SOPRO_ERR_INVALID, "item %d: [%lld, %lld + %lld) is not inside y_len = %lld", i, off, off, len, (long long)y_len);
    if (len == 0) continue;
    if (!src[i]) return fail(SOPRO_ERR_INVALID, "null source for item %d", i);
    for (long long t = off / kMixTile; t <= (off + len - 1) / kMixTile; ++t) ++ptr[t + 1];
  }
  if (y_len == 0) return SOPRO_OK;
  if (!y) return fail(SOPRO_ERR_INVALID, "null argument");
  for (long long t = 0; t < n_tiles; ++t) ptr[t + 1] += ptr[t];
  // each tile's items in item order, then one stream-ordered upload of the items, the CSR and its lists
  std::vector<int> idx(ptr[n_tiles]);
  std::vector<long long> fill(ptr.begin(), ptr.end() - 1);
  std::vector<MixItem> items(n_items);
  for (int i = 0; i < n_items; ++i) {
    const long long len = lens_host[i], off = offs_host[i];
    items[i] = MixItem{src[i], off, len};
    if (len == 0) continue;
    for (long long t = off / kMixTile; t <= (off + len - 1) / kMixTile; ++t) idx[fill[t]++] = i;
  }
  const size_t b_items = sizeof(MixItem) * items.size(), b_ptr = sizeof(long long) * ptr.size();
  const size_t b_idx = sizeof(int) * idx.size(), total = b_items + b_ptr + b_idx;
  std::vector<unsigned char> blob(total);
  std::memcpy(blob.data(), items.data(), b_items);
  std::memcpy(blob.data() + b_items, ptr.data(), b_ptr);
  std::memcpy(blob.data() + b_items + b_ptr, idx.data(), b_idx);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  unsigned char* d = nullptr;
  CK(cudaMallocAsync(reinterpret_cast<void**>(&d), total, st));
  cudaError_t e = cudaMemcpyAsync(d, blob.data(), total, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) {
    const unsigned grid = (unsigned)std::min<long long>(n_tiles, kMixMaxCtas);
    mix_kernel<<<grid, kMixThreads, 0, st>>>(reinterpret_cast<const MixItem*>(d), reinterpret_cast<const long long*>(d + b_items),
                                             reinterpret_cast<const int*>(d + b_items + b_ptr), n_tiles, y, y_len);
    e = cudaGetLastError();
  }
  const cudaError_t f = cudaFreeAsync(d, st);
  CK(e);
  CK(f);
  return SOPRO_OK;
}

}  // extern "C"
