// Reference-voice denoising: a stationary-noise Wiener suppressor with the decision-directed a priori SNR estimate
// (Ephraim-Malah) over a ragged batch of 24 kHz rows.  The definition is in include/sopro_b200.h; oracle/denoise_oracle.py
// restates it in float64.
//
// Five launches per 128 rows, every one a function of the row's own samples in an order fixed by positions:
//   dn_analyze_kernel  grid (frame tiles, rows): each CTA transforms kFramesPerCta frames with a shared-memory radix-2
//                      FFT (512-point complex, fp32; twiddles and window computed in double, rounded once) -> P [m][k]
//                      f32 and E[m] (one thread sums P in double, k ascending);
//   dn_select_kernel   one CTA per row: the K quietest candidate frames by a radix select on the bits of E (non-negative
//                      doubles order as their bits), ties to the lower m by a block scan -> sel[] ascending; a row with
//                      n < N or a non-finite E is flagged to pass through;
//   dn_gain_kernel     one thread per (row, bin): lambda = the mean of P over sel (m ascending), then the xi / G
//                      recursion over the frames in double, G overwriting P;
//   dn_synth_kernel    as analyze (bit-identical X), times G, inverse FFT, times the window -> the frame's 512 outputs;
//   dn_overlap_kernel  y[i] = frame q's second half + frame q + 1's first half (q = i / R), zeros past the row.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdint>

#include "../../include/sopro_b200.h"
#include "common.cuh"

namespace {

constexpr int kN = SOPRO_DENOISE_FRAME, kR = SOPRO_DENOISE_HOP, kBins = kN / 2 + 1, kLogN = 9;
static_assert((1 << kLogN) == kN && kR * 2 == kN, "geometry");
constexpr int kT = 256;                // FFT CTAs: one butterfly per thread per stage
constexpr int kFramesPerCta = 8;       // frames per FFT CTA (the twiddle and window tables are built once per CTA)
constexpr int kSelT = 1024;            // select: one CTA per row
constexpr int kGainT = 288;            // gain: 257 bins, rounded up to whole warps
constexpr int kOaT = 256;
constexpr int kRowsPerLaunch = 128;    // rows per launch (their lengths travel as a kernel parameter)
constexpr long long kMaxLen = 1LL << 36;
constexpr double kAlpha = 0.98, kGMin = 0.1;

__host__ __device__ inline long long frames_of(long long n) { return (n + kR - 1) / kR + 1; }
__host__ __device__ inline long long candidates_of(long long n) { return n / kR - 1; }
__host__ __device__ inline long long noise_count(long long n) { return std::max(1LL, candidates_of(n) / 10); }

// the workspace: sel [B][kmax] i32, flag [B] i32, E [B][M] f64, P / G [B][M][kBins] f32, frames [B][M][kN] f32
struct Layout {
  long long M = 0, kmax = 0;
  size_t sel = 0, flag = 0, E = 0, P = 0, F = 0, total = 0;
};

Layout layout(int B, long long max_len) {
  auto up = [](size_t v) { return (v + 255) & ~(size_t)255; };
  Layout l;
  l.M = frames_of(max_len);
  l.kmax = max_len >= kN ? noise_count(max_len) : 1;
  l.sel = 0;
  l.flag = up((size_t)B * l.kmax * sizeof(int));
  l.E = l.flag + up((size_t)B * sizeof(int));
  l.P = l.E + up((size_t)B * l.M * sizeof(double));
  l.F = l.P + up((size_t)B * l.M * kBins * sizeof(float));
  l.total = l.F + up((size_t)B * l.M * kN * sizeof(float));
  return l;
}

// W[k] = exp(-2 pi i k / N) for k < N / 2 and w[j] = sqrt(0.5 - 0.5 cos(2 pi j / N)), each in double, rounded once
struct Tables {
  float2 W[kN / 2];
  float win[kN];
};

__device__ void build_tables(Tables& t) {
  for (int k = threadIdx.x; k < kN / 2; k += blockDim.x) {
    double s, c;
    sincospi(2.0 * k / kN, &s, &c);
    t.W[k] = make_float2(__double2float_rn(c), __double2float_rn(-s));
  }
  for (int j = threadIdx.x; j < kN; j += blockDim.x) t.win[j] = __double2float_rn(sqrt(0.5 - 0.5 * cospi(2.0 * j / kN)));
}

__device__ __forceinline__ int bitrev(int j) { return (int)(__brev((unsigned)j) >> (32 - kLogN)); }

// in-place radix-2 decimation-in-time over s (bit-reversed input, natural output); `inv` conjugates the twiddles
__device__ __forceinline__ void fft(float2* s, const Tables& t, bool inv) {
  const int tid = threadIdx.x;
#pragma unroll
  for (int lg = 0; lg < kLogN; ++lg) {
    const int half = 1 << lg;
    const int pos = tid & (half - 1);
    const int i0 = ((tid >> lg) << (lg + 1)) + pos, i1 = i0 + half;
    float2 w = t.W[pos << (kLogN - 1 - lg)];
    if (inv) w.y = -w.y;
    const float2 a = s[i0], b = s[i1];
    const float2 bw = make_float2(__fsub_rn(__fmul_rn(b.x, w.x), __fmul_rn(b.y, w.y)), __fadd_rn(__fmul_rn(b.x, w.y), __fmul_rn(b.y, w.x)));
    s[i0] = make_float2(__fadd_rn(a.x, bw.x), __fadd_rn(a.y, bw.y));
    s[i1] = make_float2(__fsub_rn(a.x, bw.x), __fsub_rn(a.y, bw.y));
    __syncthreads();
  }
}

// X of frame m of the row x[0, n): s[k] for k in [0, N) (bins 0 .. N/2 are the real FFT's).  Ends synchronised.
__device__ __forceinline__ void analyze_frame(const float* __restrict__ x, long long n, long long m, float2* s, const Tables& t) {
  const long long start = (m - 1) * kR;
  for (int j = threadIdx.x; j < kN; j += kT) {
    const long long i = start + j;
    const float v = (i >= 0 && i < n) ? __fmul_rn(__ldg(x + i), t.win[j]) : 0.0f;
    s[bitrev(j)] = make_float2(v, 0.0f);
  }
  __syncthreads();
  fft(s, t, false);
}

__device__ __forceinline__ float power(float2 v) { return __fmaf_rn(v.x, v.x, __fmul_rn(v.y, v.y)); }

__global__ void __launch_bounds__(kT) dn_analyze_kernel(const float* __restrict__ x, long long x_stride, RowLens<kRowsPerLaunch> lens,
                                                        long long M_stride, double* __restrict__ E, float* __restrict__ P) {
  __shared__ Tables t;
  __shared__ float2 s[kN];
  __shared__ float p[kBins];
  const int b = blockIdx.y;
  const long long n = lens.v[b];
  if (n < kN) return;
  const long long M = frames_of(n), m0 = (long long)blockIdx.x * kFramesPerCta;
  if (m0 >= M) return;
  build_tables(t);
  const float* xb = x + (long long)b * x_stride;
  for (long long m = m0; m < std::min(M, m0 + kFramesPerCta); ++m) {
    __syncthreads();  // t is built; the previous frame's s and p are consumed
    analyze_frame(xb, n, m, s, t);
    float* Pm = P + ((long long)b * M_stride + m) * kBins;
    for (int k = threadIdx.x; k < kBins; k += kT) {
      const float v = power(s[k]);
      p[k] = v;
      Pm[k] = v;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      double e = 0.0;
      for (int k = 0; k < kBins; ++k) e += (double)p[k];
      E[(long long)b * M_stride + m] = e;
    }
  }
}

// exclusive prefix count of `f` over the CTA in thread order -> the thread's rank; the CTA's count -> *total.  Ends
// synchronised; `scratch` holds kSelT / 32 + 1 ints.
__device__ __forceinline__ int block_rank(bool f, int* scratch, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned ball = __ballot_sync(0xffffffffu, f);
  if (lane == 0) scratch[warp] = __popc(ball);
  __syncthreads();
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int w = 0; w < kSelT / 32; ++w) {
      const int c = scratch[w];
      scratch[w] = acc;
      acc += c;
    }
    scratch[kSelT / 32] = acc;
  }
  __syncthreads();
  const int r = scratch[warp] + __popc(ball & ((1u << lane) - 1u));
  *total = scratch[kSelT / 32];
  __syncthreads();
  return r;
}

__global__ void __launch_bounds__(kSelT) dn_select_kernel(RowLens<kRowsPerLaunch> lens, long long M_stride, const double* __restrict__ E,
                                                          long long kmax, int* __restrict__ sel, int* __restrict__ flag) {
  __shared__ unsigned hist[256];
  __shared__ int scratch[kSelT / 32 + 1];
  __shared__ unsigned long long s_prefix;
  __shared__ long long s_rank;
  const int b = blockIdx.x, tid = threadIdx.x;
  const long long n = lens.v[b];
  int* sb = sel + (long long)b * kmax;
  const double* Eb = E + (long long)b * M_stride;
  for (long long i = tid; i < kmax; i += kSelT) sb[i] = -1;
  bool pass = n < kN;
  if (!pass) {
    bool bad = false;
    for (long long m = tid; m < frames_of(n); m += kSelT) bad |= !isfinite(Eb[m]);
    pass = __syncthreads_or(bad) != 0;
  }
  if (tid == 0) flag[b] = pass ? 1 : 0;
  if (pass) return;
  const long long C = candidates_of(n), K = noise_count(n);
  // radix select of the K-th smallest key over m = 1 .. C, 8 bits at a time from the top
  if (tid == 0) {
    s_prefix = 0ull;
    s_rank = K;  // 1-based rank within the keys that match the prefix so far
  }
  for (int shift = 56; shift >= 0; shift -= 8) {
    for (int i = tid; i < 256; i += kSelT) hist[i] = 0u;
    __syncthreads();
    const unsigned long long prefix = s_prefix;
    const unsigned long long hi_mask = shift == 56 ? 0ull : ~0ull << (shift + 8);
    for (long long m = 1 + tid; m <= C; m += kSelT) {
      const unsigned long long key = (unsigned long long)__double_as_longlong(Eb[m]);
      if ((key & hi_mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (tid == 0) {
      long long r = s_rank;
      int d = 0;
      for (; d < 255 && r > (long long)hist[d]; ++d) r -= hist[d];
      s_prefix = prefix | ((unsigned long long)d << shift);
      s_rank = r;
    }
    __syncthreads();
  }
  const unsigned long long T = s_prefix;
  const long long take_eq = s_rank;  // keys equal to T to take, lowest m first
  long long eq_base = 0, out_base = 0;
  for (long long m0 = 1; m0 <= C; m0 += kSelT) {
    const long long m = m0 + tid;
    const unsigned long long key = m <= C ? (unsigned long long)__double_as_longlong(Eb[m]) : ~0ull;
    const bool eq = m <= C && key == T;
    int n_eq, n_sel;
    const int eq_rank = block_rank(eq, scratch, &n_eq);
    const bool take = m <= C && (key < T || (eq && eq_base + eq_rank < take_eq));
    const int pos = block_rank(take, scratch, &n_sel);
    if (take) sb[out_base + pos] = (int)m;
    eq_base += n_eq;
    out_base += n_sel;
  }
}

__global__ void __launch_bounds__(kGainT) dn_gain_kernel(RowLens<kRowsPerLaunch> lens, long long M_stride, const int* __restrict__ sel,
                                                         long long kmax, const int* __restrict__ flag, float* __restrict__ P) {
  const int b = blockIdx.x, k = threadIdx.x;
  const long long n = lens.v[b];
  if (k >= kBins || flag[b]) return;
  const long long M = frames_of(n), K = noise_count(n);
  float* Pb = P + (long long)b * M_stride * kBins + k;
  const int* sb = sel + (long long)b * kmax;
  double lam = 0.0;
  for (long long i = 0; i < K; ++i) lam += (double)Pb[(long long)sb[i] * kBins];
  lam /= (double)K;
  if (lam == 0.0) {
    for (long long m = 0; m < M; ++m) Pb[m * kBins] = 1.0f;
    return;
  }
  double g_prev = 0.0, gam_prev = 0.0;
  for (long long m = 0; m < M; ++m) {
    const double gam = (double)Pb[m * kBins] / lam;
    const double post = fmax(gam - 1.0, 0.0);
    const double xi = m == 0 ? post : kAlpha * g_prev * g_prev * gam_prev + (1.0 - kAlpha) * post;
    const double g = fmax(xi / (1.0 + xi), kGMin);
    Pb[m * kBins] = (float)g;
    g_prev = g;
    gam_prev = gam;
  }
}

__global__ void __launch_bounds__(kT) dn_synth_kernel(const float* __restrict__ x, long long x_stride, RowLens<kRowsPerLaunch> lens,
                                                      long long M_stride, const int* __restrict__ flag, const float* __restrict__ G,
                                                      float* __restrict__ F) {
  __shared__ Tables t;
  __shared__ float2 s[kN];
  __shared__ float2 u[kN];
  const int b = blockIdx.y;
  const long long n = lens.v[b];
  if (n < kN || flag[b]) return;
  const long long M = frames_of(n), m0 = (long long)blockIdx.x * kFramesPerCta;
  if (m0 >= M) return;
  build_tables(t);
  const float* xb = x + (long long)b * x_stride;
  for (long long m = m0; m < std::min(M, m0 + kFramesPerCta); ++m) {
    __syncthreads();
    analyze_frame(xb, n, m, s, t);
    const float* Gm = G + ((long long)b * M_stride + m) * kBins;
    // Y = G X on bins 0 .. N/2 (DC and Nyquist real), Y[N - k] = conj(Y[k]); placed bit-reversed for the inverse
    for (int k = threadIdx.x; k < kBins; k += kT) {
      const float g = Gm[k];
      float2 y = make_float2(__fmul_rn(g, s[k].x), __fmul_rn(g, s[k].y));
      if (k == 0 || k == kN / 2) y.y = 0.0f;
      u[bitrev(k)] = y;
      if (k > 0 && k < kN / 2) u[bitrev(kN - k)] = make_float2(y.x, -y.y);
    }
    __syncthreads();
    fft(u, t, true);
    float* Fm = F + ((long long)b * M_stride + m) * kN;
    for (int j = threadIdx.x; j < kN; j += kT) Fm[j] = __fmul_rn(__fmul_rn(u[j].x, 1.0f / kN), t.win[j]);
  }
}

__global__ void __launch_bounds__(kOaT) dn_overlap_kernel(const float* __restrict__ x, long long x_stride, RowLens<kRowsPerLaunch> lens,
                                                          long long M_stride, const int* __restrict__ flag, const float* __restrict__ F,
                                                          float* __restrict__ y, long long y_stride) {
  const int b = blockIdx.y;
  const long long n = lens.v[b];
  const bool pass = flag[b] != 0;
  const float* xb = x + (long long)b * x_stride;
  const float* Fb = F + (long long)b * M_stride * kN;
  float* yb = y + (long long)b * y_stride;
  for (long long i = (long long)blockIdx.x * kOaT + threadIdx.x; i < x_stride; i += (long long)gridDim.x * kOaT) {
    float v = 0.0f;
    if (i < n) {
      if (pass) {
        v = xb[i];
      } else {
        const long long q = i / kR, r = i - q * kR;
        v = __fadd_rn(Fb[q * kN + kR + r], Fb[(q + 1) * kN + r]);
      }
    }
    yb[i] = v;
  }
}

}  // namespace

extern "C" {

int sopro_denoise_sizes(int32_t B, int64_t max_len, int64_t* ws_bytes) {
  if (!ws_bytes) return fail(SOPRO_ERR_INVALID, "null argument");
  if (B < 1 || max_len < 0 || max_len > kMaxLen) return fail(SOPRO_ERR_INVALID, "bad geometry (B=%d, max_len=%lld)", B, (long long)max_len);
  *ws_bytes = (int64_t)layout(B, max_len).total;
  return SOPRO_OK;
}

int sopro_denoise(const float* x, int32_t B, int64_t x_stride, const int64_t* lens_host, void* ws, float* y, int64_t y_stride,
                  void* stream) {
  long long most = 0;
  int rc = check_rows(x, B, x_stride, lens_host, kMaxLen, &most);
  if (rc != SOPRO_OK) return rc;
  if (!ws || (!y && x_stride > 0)) return fail(SOPRO_ERR_INVALID, "null argument");
  if (B > 1 && y_stride < x_stride) return fail(SOPRO_ERR_INVALID, "y_stride %lld < x_stride %lld", (long long)y_stride, (long long)x_stride);
  if (x_stride == 0) return SOPRO_OK;
  const Layout l = layout(B, most);
  char* w = static_cast<char*>(ws);
  int* sel = reinterpret_cast<int*>(w + l.sel);
  int* flag = reinterpret_cast<int*>(w + l.flag);
  double* E = reinterpret_cast<double*>(w + l.E);
  float* P = reinterpret_cast<float*>(w + l.P);
  float* F = reinterpret_cast<float*>(w + l.F);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const unsigned tiles = (unsigned)((l.M + kFramesPerCta - 1) / kFramesPerCta);
  const unsigned oa = (unsigned)std::min<long long>((x_stride + kOaT - 1) / kOaT, 2048);
  for (int b0 = 0; b0 < B; b0 += kRowsPerLaunch) {
    const int rows = std::min(kRowsPerLaunch, B - b0);
    const RowLens<kRowsPerLaunch> L = row_lens<kRowsPerLaunch>(lens_host, x_stride, b0, rows);
    const float* xb = x + (long long)b0 * x_stride;
    double* Eb = E + (long long)b0 * l.M;
    float* Pb = P + (long long)b0 * l.M * kBins;
    float* Fb = F + (long long)b0 * l.M * kN;
    int* sb = sel + (long long)b0 * l.kmax;
    int* fb = flag + b0;
    if (most >= kN) {
      dn_analyze_kernel<<<dim3(tiles, rows), kT, 0, st>>>(xb, x_stride, L, l.M, Eb, Pb);
      CK(cudaGetLastError());
    }
    dn_select_kernel<<<rows, kSelT, 0, st>>>(L, l.M, Eb, l.kmax, sb, fb);
    CK(cudaGetLastError());
    if (most >= kN) {
      dn_gain_kernel<<<rows, kGainT, 0, st>>>(L, l.M, sb, l.kmax, fb, Pb);
      CK(cudaGetLastError());
      dn_synth_kernel<<<dim3(tiles, rows), kT, 0, st>>>(xb, x_stride, L, l.M, fb, Pb, Fb);
      CK(cudaGetLastError());
    }
    dn_overlap_kernel<<<dim3(oa, rows), kOaT, 0, st>>>(xb, x_stride, L, l.M, fb, Fb, y + (long long)b0 * y_stride, y_stride);
    CK(cudaGetLastError());
  }
  return SOPRO_OK;
}

}  // extern "C"
