// Speaking-rate control: pitch-preserving time-scale modification of output waveforms (WSOLA, Verhelst & Roelands
// 1993) at the codec's 24 kHz, one-shot and streaming.
//
// Fixed geometry: frame N = 480, synthesis hop Hs = N / 2 = 240, search tolerance D = 160 (321 candidates), periodic
// Hann window w[n] = sin^2(pi n / N) (evaluated on the host in double, rounded to fp32 once).  The speed is quantised to
// S = round(speed * 65536) in [16384, 262144].  For L input samples (x = 0 outside [0, L)):
//   M = ceil(L * 65536 / S) outputs, K = ceil(M / Hs) + 1 frames (0 when M = 0),
//   a_k = floor((k Hs S + 32768) / 65536)                                   (nominal analysis position, int64)
//   d_0 = 0;  k >= 1: p_{k-1} = a_{k-1} + d_{k-1}, t_k[n] = x[p_{k-1} + n]   (the natural continuation of frame k-1)
//         c_k(d) = sum_n t_k[n] x[a_k + d - N/2 + n],  d_k = argmax over [-D, D]; ties -> smallest |d|, then the negative
//   y[m] = sum_k w[m - k Hs + N/2] x[p_k + m - k Hs]  (the two frames covering m, in increasing k), cut to [0, M).
//
// stretch_frame() is the only place a frame is computed: the search, then the overlap-add of its samples.  The one-shot
// kernel and the stream kernel both call it on the same staged values, so a stream's outputs equal the one-shot result
// bit for bit under any chunk schedule.  The chain of frames is serial per utterance; one CTA runs it, and stages the
// next frame's window (a_{k+1} does not depend on d_k) while the current frame searches.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../include/sopro_b200.h"
#include "chunk_stream.cuh"

namespace {

using chunk::Src;
using chunk::src_at;

constexpr int kN = 480, kHs = 240, kHalf = kN / 2, kDelta = 160, kCand = 2 * kDelta + 1;
constexpr int kMinS = 16384, kMaxS = 262144, kOne = 65536;  // speed 0.25 .. 4.0 in 1/65536 steps
// frame k's staged window: x[a_k - D - N/2, a_k + D + Hs + N/2) -- the candidates [a_k - 400, a_k + 400) and every
// possible next template x[p_k, p_k + N), p_k <= a_k + D
constexpr int kLead = kDelta + kHalf, kWin = kLead + kDelta + kHs + kHalf;
// search layout: lane l scores candidates [l R, l R + R) (register-blocked sliding dot product), warp w the n-slice
// [w G, w G + G); the per-warp partial sums are then added in increasing w
constexpr int kWarps = 16, kThreads = 32 * kWarps, kR = 11, kG = kN / kWarps, kCandPad = 32 * kR;
constexpr int kRowsPerLaunch = 128;  // rows of a ragged batch per launch (their lengths travel as a kernel parameter)
constexpr long long kMaxLen = 1LL << 40;
static_assert(kN % kWarps == 0 && kCandPad >= kCand && kHs == kHalf, "geometry");
static_assert(kCandPad - 1 + kN - 1 + 1 <= kWin, "the search's last register load stays in the window");
constexpr double kPi = 3.141592653589793;

struct Window {
  float w[kN];
};

// the stream's device-resident state between launches
struct Carry {
  long long p;          // p_{k_done - 1}
  float pending[kHs];   // frame k_done - 1's second half, w[Hs + n] * x[p + n]: outputs [(k_done - 1) Hs, k_done Hs)
};

__host__ __device__ __forceinline__ long long pos_a(long long k, int S) { return (k * kHs * (long long)S + 32768) >> 16; }
__host__ __device__ __forceinline__ long long out_len(int S, long long L) { return (L * kOne + S - 1) / S; }
__host__ __device__ __forceinline__ long long n_frames(long long M) { return M == 0 ? 0 : (M + kHs - 1) / kHs + 1; }

Window make_window() {
  Window w;
  for (int n = 0; n < kN; ++n) {
    const double s = std::sin(kPi * n / kN);
    w.w[n] = (float)(s * s);
  }
  return w;
}

// (score, d) beats (s2, d2): the larger score; on a tie the smaller |d|, then the negative d
__device__ __forceinline__ bool beats(float s1, int d1, float s2, int d2) {
  if (s1 > s2) return true;
  if (s2 > s1) return false;
  const int a1 = d1 < 0 ? -d1 : d1, a2 = d2 < 0 ? -d2 : d2;
  return a1 != a2 ? a1 < a2 : d1 < d2;
}

struct Smem {
  float buf[3][kWin];              // window k in buf[k % 3]; template of k inside buf[(k - 1) % 3]; k + 1 prefetched
  float part[kWarps][kCandPad];    // per-warp partial scores
  float best_s[kCandPad / 32];
  int best_d[kCandPad / 32];
};

// One frame: d_k (search of the window `win` = x[a_k - 400, a_k + 640) against the template `tmpl` = t_k, skipped for
// frame 0), then its overlap-add: thread n < Hs finishes output (k - 1) Hs + n = pending + w[n] x[p_k - Hs + n] (one
// fma, the earlier frame's product first) and keeps w[Hs + n] x[p_k + n] as the next pending sample.  Returns d_k.
// Entered and left with every thread synchronised; the search's scratch is sm.part / sm.best_*.
__device__ __forceinline__ int stretch_frame(Smem& sm, const float* __restrict__ win, const float* __restrict__ tmpl, bool search,
                                             float w_lo, float w_hi, float& pending, float& out) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  int d = 0;
  if (search) {
    const int c0 = lane * kR, n0 = wid * kG;
    float acc[kR], xr[kR];
#pragma unroll
    for (int j = 0; j < kR; ++j) {
      acc[j] = 0.0f;
      xr[j] = win[c0 + n0 + j];  // candidate c0 + j at n = n0
    }
#pragma unroll
    for (int i = 0; i < kG; ++i) {
      const float t = tmpl[n0 + i];  // a broadcast: every lane of the warp reads the same n
#pragma unroll
      for (int j = 0; j < kR; ++j) acc[j] = __fmaf_rn(t, xr[j], acc[j]);
#pragma unroll
      for (int j = 0; j + 1 < kR; ++j) xr[j] = xr[j + 1];
      xr[kR - 1] = win[c0 + n0 + i + kR];
    }
#pragma unroll
    for (int j = 0; j < kR; ++j) sm.part[wid][c0 + j] = acc[j];
    __syncthreads();
    if (tid < kCandPad) {
      float s = sm.part[0][tid];
#pragma unroll
      for (int w = 1; w < kWarps; ++w) s = __fadd_rn(s, sm.part[w][tid]);
      int dd = tid - kDelta;
      if (tid >= kCand) {  // the padding candidates never win
        s = -INFINITY;
        dd = 1 << 20;
      }
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {  // a fixed tree: lane 0 ends with the warp's best
        const float s2 = __shfl_down_sync(0xffffffffu, s, off);
        const int d2 = __shfl_down_sync(0xffffffffu, dd, off);
        if (beats(s2, d2, s, dd)) {
          s = s2;
          dd = d2;
        }
      }
      if (lane == 0) {
        sm.best_s[wid] = s;
        sm.best_d[wid] = dd;
      }
    }
    __syncthreads();
    float s = sm.best_s[0];
    d = sm.best_d[0];
#pragma unroll
    for (int w = 1; w < kCandPad / 32; ++w)
      if (beats(sm.best_s[w], sm.best_d[w], s, d)) {
        s = sm.best_s[w];
        d = sm.best_d[w];
      }
  }
  if (tid < kHs) {
    const float* seg = win + (d + kDelta);  // x[p_k - Hs + n] = win[d + 160 + n]
    out = __fmaf_rn(w_lo, seg[tid], pending);
    pending = __fmul_rn(w_hi, seg[kHs + tid]);
  }
  return d;
}

// Frames [k_begin, k_end) of one utterance, in order.  Frame k >= 1 finishes output block k - 1, written to
// y[(k - 1) Hs + n - y_origin] where below m_end.  With k_begin >= 1, p_prev and pending are frame k_begin - 1's.
__device__ void stretch_frames(const Src& src, int S, long long k_begin, long long k_end, long long p_prev, float pending,
                               const Window& wp, float* __restrict__ y, long long y_origin, long long m_end,
                               int* __restrict__ offsets, Carry* __restrict__ carry_out) {
  __shared__ Smem sm;
  const int tid = threadIdx.x;
  const float w_lo = tid < kHs ? wp.w[tid] : 0.0f, w_hi = tid < kHs ? wp.w[kHs + tid] : 0.0f;
  // stage window k_begin and, for a frame that searches, its template t = x[p_prev, p_prev + N)
  {
    const long long base = pos_a(k_begin, S) - kLead;
    float* wb = sm.buf[k_begin % 3];
    for (int i = tid; i < kWin; i += kThreads) wb[i] = src_at(src, base + i);
    if (k_begin >= 1) {
      float* tb = sm.buf[(k_begin + 2) % 3];
      for (int i = tid; i < kN; i += kThreads) tb[i] = src_at(src, p_prev + i);
    }
  }
  __syncthreads();
  const float* tmpl = sm.buf[(k_begin + 2) % 3];
  long long p = p_prev;
  for (long long k = k_begin; k < k_end; ++k) {
    const long long a = pos_a(k, S);
    // the next frame's window does not depend on this frame's search: its loads are in flight while the search runs
    constexpr int kPer = (kWin + kThreads - 1) / kThreads;
    float nx[kPer];
    const bool more = k + 1 < k_end;
    const long long nbase = pos_a(k + 1, S) - kLead;
#pragma unroll
    for (int r = 0; r < kPer; ++r) {
      const int i = tid + r * kThreads;
      nx[r] = (more && i < kWin) ? src_at(src, nbase + i) : 0.0f;
    }
    const float* win = sm.buf[k % 3];
    float out = 0.0f;
    const int d = stretch_frame(sm, win, tmpl, k >= 1, w_lo, w_hi, pending, out);
    p = a + d;
    if (k >= 1 && tid < kHs) {
      const long long m = (k - 1) * kHs + tid;
      if (m < m_end) y[m - y_origin] = out;
    }
    if (offsets && tid == 0) offsets[k] = d;
    tmpl = win + (d + kLead);  // t_{k+1}[n] = x[p_k + n]
    if (more) {
      float* nb = sm.buf[(k + 1) % 3];
#pragma unroll
      for (int r = 0; r < kPer; ++r) {
        const int i = tid + r * kThreads;
        if (i < kWin) nb[i] = nx[r];
      }
    }
    __syncthreads();
  }
  if (carry_out) {
    if (tid < kHs) carry_out->pending[tid] = pending;
    if (tid == 0) carry_out->p = p;
  }
}

// one-shot, ragged batch: one CTA per row; row b reads x[b][0, lens[b]) only
__global__ void __launch_bounds__(kThreads, 1) stretch_batch_kernel(Window wp, const float* __restrict__ x, long long x_stride, RowLens<kRowsPerLaunch> lens,
                                                                    int S, float* __restrict__ y, long long y_stride,
                                                                    int* __restrict__ offsets, long long k_stride) {
  const int b = blockIdx.x;
  const long long L = lens.v[b];
  const Src s{x + (long long)b * x_stride, nullptr, 0, L, L};
  const long long M = out_len(S, L);
  stretch_frames(s, S, 0, n_frames(M), 0, 0.0f, wp, y + (long long)b * y_stride, 0, M,
                 offsets ? offsets + (long long)b * k_stride : nullptr, nullptr);
}

// one row of a batch with a speed per row: its valid samples and its S
struct RowSpeed {
  long long len;
  int S;
};

// one-shot, ragged batch, a speed per row: one CTA per row.  A row at S = 65536 is copied through; any other row runs
// the frames stretch_batch_kernel runs for it at its own S, so its outputs equal that kernel's bit for bit.  A separate
// kernel, so the one-speed kernel keeps S as a parameter and its code is unchanged.
__global__ void __launch_bounds__(kThreads, 1) stretch_rows_kernel(Window wp, const float* __restrict__ x, long long x_stride,
                                                                   const RowSpeed* __restrict__ rows, float* __restrict__ y,
                                                                   long long y_stride, int* __restrict__ offsets, long long k_stride) {
  const int b = blockIdx.x;
  const long long L = rows[b].len;
  const int S = rows[b].S;
  const float* xb = x + (long long)b * x_stride;
  float* yb = y + (long long)b * y_stride;
  if (S == kOne) {  // uniform per CTA: the whole block returns before stretch_frames' barriers
    for (long long m = threadIdx.x; m < L; m += kThreads) yb[m] = xb[m];
    return;
  }
  const Src s{xb, nullptr, 0, L, L};
  const long long M = out_len(S, L);
  stretch_frames(s, S, 0, n_frames(M), 0, 0.0f, wp, yb, 0, M, offsets ? offsets + (long long)b * k_stride : nullptr, nullptr);
}

// stream: frames [k_begin, k_end) of one utterance from its carried tail and the new chunk; the carried p / pending
// are read at the start (k_begin >= 1) and the new ones written back at the end
__global__ void __launch_bounds__(kThreads, 1) stretch_stream_kernel(Window wp, Src s, int S, long long k_begin, long long k_end,
                                                                     Carry* carry, float* __restrict__ y, long long y_origin,
                                                                     long long m_end) {
  long long p_prev = 0;
  float pending = 0.0f;
  if (k_begin >= 1) {
    p_prev = carry->p;
    if (threadIdx.x < kHs) pending = carry->pending[threadIdx.x];
  }
  __syncthreads();  // every thread has read the carry before any writes it back
  stretch_frames(s, S, k_begin, k_end, p_prev, pending, wp, y, y_origin, m_end, nullptr, carry);
}

// host arithmetic of the stream rule
long long frame_need(long long k, int S) {  // input samples frame k's search and overlap-add read
  const long long own = pos_a(k, S) + kDelta + kHalf;
  return k == 0 ? own : std::max(own, pos_a(k - 1, S) + kDelta + kHs + kHalf);
}
long long frames_ready(int S, long long k_done, long long n_seen) {
  long long k = k_done;
  while (frame_need(k, S) <= n_seen) ++k;
  return k;
}
long long tail_base(long long k_done, int S) {  // the first sample frame k_done may read (its candidates or template)
  if (k_done == 0) return pos_a(0, S) - kLead;
  return std::min(pos_a(k_done, S) - kLead, pos_a(k_done - 1, S) - kDelta);
}
// the carried tail is shorter than max(D + N/2 + Ha + D + N/2, 2 (D + N/2) + Hs) + 1 samples (Ha <= 4 Hs + 1)
constexpr long long kCarryCap = 2048;
static_assert(kCarryCap >= 2 * kLead + 4 * kHs + 2 && kCarryCap >= 2 * kLead + kHs + 1, "carry capacity");

}  // namespace

// the tail holds the logical input [tail_base(k_done), n_seen) of the utterance
struct sopro_stretch_stream : chunk::ChunkStream {
  int S = 0;
  Carry* state = nullptr;
  long long k_done = 0;  // frames computed

  cudaError_t alloc_own() { return cudaMalloc(&state, sizeof(Carry)); }
  void free_own() { cudaFree(state); }
};

namespace {
long long emitted(const sopro_stretch_stream* s) { return std::max(0LL, s->k_done - 1) * kHs; }

int launch_stream(sopro_stretch_stream* s, const Src& src, long long k_begin, long long k_end, float* y, long long m_end,
                  cudaStream_t st) {
  if (k_end <= k_begin) return SOPRO_OK;
  static const Window wp = make_window();
  stretch_stream_kernel<<<1, kThreads, 0, st>>>(wp, src, s->S, k_begin, k_end, s->state, y, emitted(s), m_end);
  CK(cudaGetLastError());
  return SOPRO_OK;
}

bool valid_S(int32_t S) { return S >= kMinS && S <= kMaxS; }
}  // namespace

extern "C" {

int sopro_stretch_speed(double speed, int32_t* S) {
  if (!S) return fail(SOPRO_ERR_INVALID, "null argument");
  if (!(speed >= 0.25 && speed <= 4.0))  // also refuses NaN
    return fail(SOPRO_ERR_INVALID, "speed must be a real number in [0.25, 4.0] (got %g)", speed);
  *S = (int32_t)std::nearbyint(speed * kOne);  // exact product (a power of two), rounded half to even
  return SOPRO_OK;
}

int64_t sopro_stretched_length(int32_t S, int64_t n_in) {
  if (!valid_S(S) || n_in < 0 || n_in > kMaxLen) return -1;
  return out_len(S, n_in);
}

int64_t sopro_stretch_positions(int32_t S, int64_t n_in, int64_t* a) {
  if (!valid_S(S) || n_in < 0 || n_in > kMaxLen) return -1;
  const long long K = n_frames(out_len(S, n_in));
  if (a)
    for (long long k = 0; k < K; ++k) a[k] = pos_a(k, S);
  return K;
}

int sopro_stretch_window(float* w) {
  if (!w) return fail(SOPRO_ERR_INVALID, "null argument");
  const Window wp = make_window();
  std::memcpy(w, wp.w, sizeof(wp.w));
  return SOPRO_OK;
}

int sopro_stretch(const float* x, int32_t B, int64_t x_stride, const int64_t* lens_host, int32_t S, float* y, int64_t y_stride,
                  int32_t* offsets, void* stream) {
  if (!x || !y) return fail(SOPRO_ERR_INVALID, "null argument");
  if (!valid_S(S)) return fail(SOPRO_ERR_INVALID, "S = %d not in [%d, %d] (speed 0.25 .. 4 in 1/65536 steps)", S, kMinS, kMaxS);
  long long most = 0;
  int rc = check_rows(x, B, x_stride, lens_host, kMaxLen, &most);
  if (rc != SOPRO_OK) return rc;
  most = out_len(S, most);  // out_len is monotone in the row length
  if ((rc = check_out_rows(y, B, y_stride, most)) != SOPRO_OK) return rc;
  if (most == 0) return SOPRO_OK;
  const long long k_max = n_frames(most);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  static const Window wp = make_window();
  for (int b0 = 0; b0 < B; b0 += kRowsPerLaunch) {
    const int rows = std::min(kRowsPerLaunch, B - b0);
    stretch_batch_kernel<<<rows, kThreads, 0, st>>>(wp, x + (long long)b0 * x_stride, x_stride,
                                                    row_lens<kRowsPerLaunch>(lens_host, x_stride, b0, rows), S,
                                                    y + (long long)b0 * y_stride, y_stride,
                                                    offsets ? offsets + (long long)b0 * k_max : nullptr, k_max);
    CK(cudaGetLastError());
  }
  return SOPRO_OK;
}

int sopro_stretch_rows(const float* x, int32_t B, int64_t x_stride, const int64_t* lens_host, const int32_t* S_host, float* y,
                       int64_t y_stride, int32_t* offsets, void* stream) {
  if (!x || !y || !S_host) return fail(SOPRO_ERR_INVALID, "null argument");
  long long most = 0;
  int rc = check_rows(x, B, x_stride, lens_host, kMaxLen, &most);
  if (rc != SOPRO_OK) return rc;
  std::vector<RowSpeed> rows(B);
  long long m_max = 0;
  for (int b = 0; b < B; ++b) {
    const int S = S_host[b];
    if (!valid_S(S))
      return fail(SOPRO_ERR_INVALID, "S_host[%d] = %d not in [%d, %d] (speed 0.25 .. 4 in 1/65536 steps)", b, S, kMinS, kMaxS);
    rows[b] = RowSpeed{lens_host ? lens_host[b] : x_stride, S};
    m_max = std::max(m_max, out_len(S, rows[b].len));
  }
  if ((rc = check_out_rows(y, B, y_stride, m_max)) != SOPRO_OK) return rc;
  if (m_max == 0) return SOPRO_OK;
  // the rows' lengths and speeds go to the device in one stream-ordered copy, so one launch takes any batch size
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  static const Window wp = make_window();
  RowSpeed* d_rows = nullptr;
  CK(cudaMallocAsync(&d_rows, sizeof(RowSpeed) * B, st));
  cudaError_t e = cudaMemcpyAsync(d_rows, rows.data(), sizeof(RowSpeed) * B, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) {
    stretch_rows_kernel<<<B, kThreads, 0, st>>>(wp, x, x_stride, d_rows, y, y_stride, offsets, n_frames(m_max));
    e = cudaGetLastError();
  }
  const cudaError_t f = cudaFreeAsync(d_rows, st);
  CK(e);
  CK(f);
  return SOPRO_OK;
}

int sopro_stretch_stream_create(int64_t max_chunk, int device, sopro_stretch_stream_t** out) {
  int rc = chunk::check_create(max_chunk, out);
  if (rc == SOPRO_OK) rc = open_device(device, "the time-stretch");
  if (rc != SOPRO_OK) return rc;
  sopro_stretch_stream* s = new sopro_stretch_stream();
  s->unset = "speed";
  return chunk::create(s, max_chunk, kCarryCap, "stretch", out);
}

int sopro_stretch_stream_destroy(sopro_stretch_stream_t* s) { return chunk::destroy(s); }

int sopro_stretch_stream_reset(sopro_stretch_stream_t* s, int32_t S) {
  if (!s) return fail(SOPRO_ERR_INVALID, "null argument");
  if (!valid_S(S)) return fail(SOPRO_ERR_INVALID, "S = %d not in [%d, %d]", S, kMinS, kMaxS);
  s->S = S;
  s->restart(tail_base(0, S));
  s->k_done = 0;
  return SOPRO_OK;
}

int64_t sopro_stretch_stream_ready(const sopro_stretch_stream_t* s, int64_t n_more, int final) {
  if (!chunk::can_run(s, n_more)) return -1;
  const long long n = s->tail.seen + n_more;
  if (final) return out_len(s->S, n) - emitted(s);
  return std::max(0LL, frames_ready(s->S, s->k_done, n) - 1) * kHs - emitted(s);
}

int sopro_stretch_push(sopro_stretch_stream_t* s, const float* x, int64_t n, float* y, void* stream) {
  int rc = chunk::check_push(s, n);
  if (rc != SOPRO_OK || n == 0) return rc;
  const long long k_done = frames_ready(s->S, s->k_done, s->tail.seen + n);
  if ((rc = chunk::check_io(x, n, y, std::max(0LL, k_done - 1) * kHs - emitted(s))) != SOPRO_OK) return rc;
  CK(cudaSetDevice(s->tail.device));
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  rc = launch_stream(s, s->tail.src(x, n), s->k_done, k_done, y, 1LL << 62, st);
  if (rc == SOPRO_OK) rc = s->tail.keep(tail_base(k_done, s->S), x, n, st);
  if (rc != SOPRO_OK) return rc;
  s->k_done = k_done;
  return SOPRO_OK;
}

int sopro_stretch_finish(sopro_stretch_stream_t* s, float* y, void* stream) {
  int rc = chunk::check_finish(s);
  if (rc != SOPRO_OK) return rc;
  const long long M = out_len(s->S, s->tail.seen), K = n_frames(M);
  if ((rc = chunk::check_io(nullptr, 0, y, M - emitted(s))) != SOPRO_OK) return rc;
  CK(cudaSetDevice(s->tail.device));
  rc = launch_stream(s, s->tail.src(nullptr, 0), s->k_done, K, y, M, reinterpret_cast<cudaStream_t>(stream));
  if (rc != SOPRO_OK) return rc;
  s->finished = true;
  return SOPRO_OK;
}

}  // extern "C"
