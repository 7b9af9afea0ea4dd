// Loudness normalisation: the ITU-R BS.1770-4 integrated loudness of each output row, and a gain to a target, on the
// device.  The definition (include/sopro_b200.h, oracle/loudness_oracle.py in float64):
//   K-weighting: two biquads in cascade from zero state (libebur128's coefficients, evaluated on the host in double);
//   sub-block s = floor((sr + 5) / 10) samples; block j = sub-blocks j .. j + 3, J = max(0, floor(n / s) - 3);
//   z_j = sum y^2 over the block / (4 s); absolute gate z_j > 10^((-70 + 0.691) / 10); relative gate z_j > 0.1 * the mean
//   z over the blocks past the absolute gate; L = -0.691 + 10 log10(mean z over the blocks past both), -inf when none;
//   g = fp32(min(10^((T - L) / 20), 10^(-1/20) / max|x|)), rounded once toward zero (1 when L = -inf); y = g * x, one
//   fp32 multiply.
//
// The filter, the y^2 sums and the gating run in fp64.  The cascade in direct form I is a linear recurrence on the
// state (u[n-1], u[n-2], y[n-1], y[n-2]) (u: the shelf's output), driven by x; the input history is read from x itself.
// So it runs as a chunked scan over pieces of P = 32 samples at fixed absolute positions:
//   scan kernel:   each thread filters its piece from zero state (v_i, kept in the workspace); a Kogge-Stone scan with
//                  the powers A^(P 2^k) gives the CTA's aggregate;
//   carry kernel:  per row, the CTAs' start states in increasing order (s_c = A^(P T) s_{c-1} + agg_{c-1});
//   energy kernel: the scan again with the CTA's start state, then each piece re-filtered from its true start state,
//                  y^2 summed per piece into the (at most two) sub-blocks it touches, and max|x| per CTA;
//   sub-block kernel: a warp per sub-block sums its pieces' y^2 in a fixed order;
//   gate kernel:   one CTA per row: blocks, both gates, L and g;
//   apply kernel:  y = g * x over [0, lens[b]).
// Every sum has a fixed order and every piece a fixed position, so a row's result depends only on its own samples.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>

#include "../../include/sopro_b200.h"
#include "common.cuh"

namespace {

constexpr int kP = 32;                  // samples per piece (one thread)
constexpr int kLogT = 8, kT = 1 << kLogT;  // threads per CTA
constexpr long long kSpan = (long long)kP * kT;  // samples per CTA
constexpr int kStage = kP * kT + 2;     // a CTA's samples and the two before them
constexpr int kRowsPerLaunch = 128;     // rows of a ragged batch per launch (their lengths travel as a kernel parameter)
constexpr long long kMaxLen = 1LL << 40;
constexpr int kMinRate = 4000, kMaxRate = 192000;
constexpr double kPi = 3.141592653589793;

struct Mat {
  double m[4][4];
};

// the filter as the kernels use it: the shelf's numerator, both negated denominators, and A^(P 2^k) for k = 0 .. log2 T
struct Filt {
  double b0, b1, b2, na11, na12, na21, na22;
  Mat pw[kLogT + 1];
};

struct Gate {
  int s;            // sub-block samples
  double abs_e;     // 10^((-70 + 0.691) / 10): the absolute gate as an energy
  double rel;       // 10^(-10 / 10): the relative gate's factor on the mean energy
  double ceil_amp;  // 10^(-1 / 20): the sample-peak ceiling
};

struct St {
  double v[4];
};

bool valid_rate(int sr) { return sr >= kMinRate && sr <= kMaxRate; }
int sub_block(int sr) { return (sr + 5) / 10; }

// libebur128's derivation from the analog prototype, in double; c = stage 1 (b0, b1, b2, a1, a2), stage 2 (same)
void coeffs(int sr, double c[10]) {
  double f0 = 1681.974450955533, G = 3.999843853973347, Q = 0.7071752369554196;
  double K = std::tan(kPi * f0 / sr);
  const double Vh = std::pow(10.0, G / 20.0), Vb = std::pow(Vh, 0.4996667741545416);
  double a0 = 1.0 + K / Q + K * K;
  c[0] = (Vh + Vb * K / Q + K * K) / a0;
  c[1] = 2.0 * (K * K - Vh) / a0;
  c[2] = (Vh - Vb * K / Q + K * K) / a0;
  c[3] = 2.0 * (K * K - 1.0) / a0;
  c[4] = (1.0 - K / Q + K * K) / a0;
  f0 = 38.13547087602444;
  Q = 0.5003270373238773;
  K = std::tan(kPi * f0 / sr);
  a0 = 1.0 + K / Q + K * K;
  c[5] = 1.0;
  c[6] = -2.0;
  c[7] = 1.0;
  c[8] = 2.0 * (K * K - 1.0) / a0;
  c[9] = (1.0 - K / Q + K * K) / a0;
}

Mat matmul(const Mat& a, const Mat& b) {
  Mat r{};
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      double acc = 0.0;
      for (int k = 0; k < 4; ++k) acc += a.m[i][k] * b.m[k][j];
      r.m[i][j] = acc;
    }
  return r;
}

Filt make_filt(int sr) {
  double c[10];
  coeffs(sr, c);
  Filt f{};
  f.b0 = c[0];
  f.b1 = c[1];
  f.b2 = c[2];
  f.na11 = -c[3];
  f.na12 = -c[4];
  f.na21 = -c[8];
  f.na22 = -c[9];
  // one sample: (u1, u2, y1, y2) -> (u, u1, y, y1), u = f - a11 u1 - a12 u2, y = u - 2 u1 + u2 - a21 y1 - a22 y2
  Mat A{};
  A.m[0][0] = -c[3];
  A.m[0][1] = -c[4];
  A.m[1][0] = 1.0;
  A.m[2][0] = -c[3] - 2.0;
  A.m[2][1] = 1.0 - c[4];
  A.m[2][2] = -c[8];
  A.m[2][3] = -c[9];
  A.m[3][2] = 1.0;
  Mat p = A;
  for (int i = 1; i < kP; ++i) p = matmul(p, A);  // A^P
  f.pw[0] = p;
  for (int k = 1; k <= kLogT; ++k) f.pw[k] = matmul(f.pw[k - 1], f.pw[k - 1]);
  return f;
}

Gate make_gate(int sr) {
  return Gate{sub_block(sr), std::pow(10.0, (-70.0 + 0.691) / 10.0), std::pow(10.0, -10.0 / 10.0), std::pow(10.0, -1.0 / 20.0)};
}

// the workspace: per row, R = ceil(max_len / (P T)) CTAs and floor(max_len / s) sub-blocks
struct Layout {
  long long R = 0, nsb = 0;
  size_t v = 0, e = 0, agg = 0, carry = 0, cmax = 0, E = 0, L = 0, g = 0, total = 0;
};

Layout layout(int B, long long max_len, int sr) {
  Layout l;
  l.R = (max_len + kSpan - 1) / kSpan;
  l.nsb = max_len / sub_block(sr);
  size_t off = 0;
  auto take = [&](size_t bytes) {
    const size_t o = off;
    off += (bytes + 255) & ~(size_t)255;
    return o;
  };
  const size_t rows = (size_t)B;
  l.v = take(rows * l.R * kT * sizeof(St));
  l.e = take(rows * l.R * kT * 2 * sizeof(double));
  l.agg = take(rows * l.R * sizeof(St));
  l.carry = take(rows * l.R * sizeof(St));
  l.cmax = take(rows * l.R * sizeof(float));
  l.E = take(rows * l.nsb * sizeof(double));
  l.L = take(rows * sizeof(double));
  l.g = take(rows * sizeof(float));
  l.total = off;
  return l;
}

// s = M p + s, each row one fma chain in increasing column
__device__ __forceinline__ void mat_acc(const Mat& M, const double p[4], double s[4]) {
  double r[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    double acc = s[i];
#pragma unroll
    for (int j = 0; j < 4; ++j) acc = fma(M.m[i][j], p[j], acc);
    r[i] = acc;
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) s[i] = r[i];
}

__device__ __forceinline__ int sidx(int i) { return i + (i >> 5); }  // one pad word per 32: a piece per bank

// x[base - 2, base + P T) of a row with n samples into shared memory (zeros outside [0, n); nothing past n is read)
__device__ __forceinline__ void stage(float* xs, const float* __restrict__ x, long long base, long long n) {
  for (int i = threadIdx.x; i < kStage; i += kT) {
    const long long g = base - 2 + i;
    xs[sidx(i)] = (g >= 0 && g < n) ? x[g] : 0.0f;
  }
}

// the thread's piece from state st (u1, u2, y1, y2); with kEnergy, y^2 of the samples below `end` goes to e_lo before
// `split` and to e_hi from it, in sample order
template <bool kEnergy>
__device__ __forceinline__ void filter_piece(const Filt& f, const float* xs, double st[4], long long g0, long long split,
                                             long long end, double& e_lo, double& e_hi) {
  const int i0 = threadIdx.x * kP;  // the piece's first sample is staged at i0 + 2
  double x2 = xs[sidx(i0)], x1 = xs[sidx(i0 + 1)];
  double u1 = st[0], u2 = st[1], y1 = st[2], y2 = st[3];
#pragma unroll 8
  for (int k = 0; k < kP; ++k) {
    const double x0 = xs[sidx(i0 + 2 + k)];
    const double u = fma(f.na11, u1, fma(f.na12, u2, fma(f.b0, x0, fma(f.b1, x1, f.b2 * x2))));
    const double y = fma(f.na21, y1, fma(f.na22, y2, fma(-2.0, u1, u) + u2));
    if (kEnergy) {
      const long long g = g0 + k;
      if (g < end) {
        if (g < split) e_lo = fma(y, y, e_lo);
        else e_hi = fma(y, y, e_hi);
      }
    }
    x2 = x1;
    x1 = x0;
    u2 = u1;
    u1 = u;
    y2 = y1;
    y1 = y;
  }
  st[0] = u1;
  st[1] = u2;
  st[2] = y1;
  st[3] = y2;
}

// inclusive Kogge-Stone scan of the threads' states: s_i <- s_i + A^(P 2^k) s_{i - 2^k}, k = 0 .. log2 T - 1
__device__ __forceinline__ void cta_scan(const Filt& f, double s[4], double (*sc)[kT]) {
  const int tid = threadIdx.x;
#pragma unroll
  for (int k = 0; k < kLogT; ++k) {
#pragma unroll
    for (int r = 0; r < 4; ++r) sc[r][tid] = s[r];
    __syncthreads();
    if (tid >= (1 << k)) {
      double p[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) p[r] = sc[r][tid - (1 << k)];
      mat_acc(f.pw[k], p, s);
    }
    __syncthreads();
  }
}

struct Smem {
  float xs[kStage + kStage / 32 + 1];
  double sc[4][kT];
};

// pass 1: grid (R, rows); piece end states from zero state, and the CTA's aggregate
__global__ void __launch_bounds__(kT) loud_scan_kernel(Filt f, const float* __restrict__ x, long long x_stride, RowLens<kRowsPerLaunch> lens,
                                                       St* __restrict__ v, St* __restrict__ agg, long long R) {
  __shared__ Smem sm;
  const int b = blockIdx.y, tid = threadIdx.x;
  const long long c = blockIdx.x, n = lens.v[b], base = c * kSpan;
  if (base >= n) return;
  stage(sm.xs, x + (long long)b * x_stride, base, n);
  __syncthreads();
  double s[4] = {0.0, 0.0, 0.0, 0.0}, e0 = 0.0, e1 = 0.0;
  filter_piece<false>(f, sm.xs, s, 0, 0, 0, e0, e1);
  St& out = v[((long long)b * R + c) * kT + tid];
#pragma unroll
  for (int r = 0; r < 4; ++r) out.v[r] = s[r];
  cta_scan(f, s, sm.sc);
  if (tid == kT - 1) {
#pragma unroll
    for (int r = 0; r < 4; ++r) agg[(long long)b * R + c].v[r] = s[r];
  }
}

// per row, in increasing CTA order: carry_c = A^(P T) carry_{c-1} + agg_{c-1}, carry_0 = 0; the aggregates are staged
// through shared memory kT at a time, so the serial chain waits on no global load
__global__ void __launch_bounds__(kT) loud_carry_kernel(Filt f, RowLens<kRowsPerLaunch> lens, const St* __restrict__ agg, St* __restrict__ carry,
                                                        long long R) {
  __shared__ St buf[kT];
  const int b = blockIdx.x, tid = threadIdx.x;
  const long long Rb = (lens.v[b] + kSpan - 1) / kSpan;
  const St* ab = agg + (long long)b * R;
  double s[4] = {0.0, 0.0, 0.0, 0.0};
  for (long long c0 = 0; c0 < Rb; c0 += kT) {
    const long long c = c0 + tid;
    if (c >= 1 && c < Rb) buf[tid] = ab[c - 1];
    __syncthreads();
    if (tid == 0) {
      const int m = (int)std::min<long long>(kT, Rb - c0);
      for (int i = 0; i < m; ++i) {
        if (c0 + i > 0) {
          double a[4];
#pragma unroll
          for (int r = 0; r < 4; ++r) a[r] = buf[i].v[r];
          mat_acc(f.pw[kLogT], s, a);
#pragma unroll
          for (int r = 0; r < 4; ++r) s[r] = a[r];
        }
#pragma unroll
        for (int r = 0; r < 4; ++r) buf[i].v[r] = s[r];
      }
    }
    __syncthreads();
    if (c < Rb) carry[(long long)b * R + c] = buf[tid];
    __syncthreads();
  }
}

// pass 2: grid (R, rows); each piece re-filtered from its true start state; y^2 per piece and sub-block; max|x| per CTA
__global__ void __launch_bounds__(kT) loud_energy_kernel(Filt f, int sbs, const float* __restrict__ x, long long x_stride,
                                                         RowLens<kRowsPerLaunch> lens, const St* __restrict__ v, const St* __restrict__ carry,
                                                         double* __restrict__ e, float* __restrict__ cmax, long long R) {
  __shared__ Smem sm;
  __shared__ float wmax[kT / 32];
  const int b = blockIdx.y, tid = threadIdx.x;
  const long long c = blockIdx.x, n = lens.v[b], base = c * kSpan;
  if (base >= n) return;
  stage(sm.xs, x + (long long)b * x_stride, base, n);
  const long long piece = ((long long)b * R + c) * kT + tid;
  double s[4], c0[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    s[r] = v[piece].v[r];
    c0[r] = carry[(long long)b * R + c].v[r];
  }
  if (tid == 0) mat_acc(f.pw[0], c0, s);  // piece 0 ends at A^P carry + v_0; the scan carries it to every piece
  cta_scan(f, s, sm.sc);                  // (its barriers also cover the staging)
#pragma unroll
  for (int r = 0; r < 4; ++r) sm.sc[r][tid] = s[r];
  __syncthreads();
  double st[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) st[r] = tid ? sm.sc[r][tid - 1] : c0[r];
  const long long g0 = base + (long long)tid * kP, end = (n / sbs) * sbs, split = (g0 / sbs + 1) * sbs;
  double e_lo = 0.0, e_hi = 0.0;
  filter_piece<true>(f, sm.xs, st, g0, split, end, e_lo, e_hi);
  e[2 * piece] = e_lo;
  e[2 * piece + 1] = e_hi;
  float m = 0.0f;
  for (int k = 0; k < kP; ++k)
    if (g0 + k < n) m = fmaxf(m, fabsf(sm.xs[sidx(tid * kP + 2 + k)]));
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
  if ((tid & 31) == 0) wmax[tid >> 5] = m;
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < kT / 32; ++w) m = fmaxf(m, wmax[w]);
    cmax[(long long)b * R + c] = m;
  }
}

// grid (ceil(nsb / 8), rows): warp w sums sub-block q = 8 blockIdx.x + w over the pieces it touches -- lane l the
// pieces i0 + l, i0 + l + 32, ... in order, then a butterfly over the lanes (a fixed order that depends on q and s alone)
__global__ void __launch_bounds__(kT) loud_subblock_kernel(int sbs, RowLens<kRowsPerLaunch> lens, const double* __restrict__ e, double* __restrict__ E,
                                                           long long R, long long nsb_stride) {
  const int b = blockIdx.y, lane = threadIdx.x & 31;
  const long long s = sbs, q = (long long)blockIdx.x * (kT / 32) + (threadIdx.x >> 5);
  if (q >= lens.v[b] / s) return;  // whole warps leave together
  const double* eb = e + 2 * (long long)b * R * kT;
  const long long i0 = q * s / kP, i1 = ((q + 1) * s - 1) / kP;
  double acc = 0.0;
  for (long long i = i0 + lane; i <= i1; i += 32) acc += eb[2 * i + ((i * kP) / s == q ? 0 : 1)];
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  if (lane == 0) E[(long long)b * nsb_stride + q] = acc;
}

// a fixed tree over the CTA's threads
__device__ __forceinline__ void block_sum(double& v, long long& cnt, double* red, long long* redc) {
  const int tid = threadIdx.x;
  red[tid] = v;
  redc[tid] = cnt;
  __syncthreads();
  for (int h = kT / 2; h > 0; h >>= 1) {
    if (tid < h) {
      red[tid] += red[tid + h];
      redc[tid] += redc[tid + h];
    }
    __syncthreads();
  }
  v = red[0];
  cnt = redc[0];
  __syncthreads();
}

__device__ __forceinline__ double block_z(const double* E, long long j, double inv4s) {
  return (((E[j] + E[j + 1]) + E[j + 2]) + E[j + 3]) * inv4s;
}

// one CTA per row: blocks, both gates, L, max|x| and (normalize) the gain
__global__ void __launch_bounds__(kT) loud_gate_kernel(Gate gt, RowLens<kRowsPerLaunch> lens, const float* __restrict__ cmax,
                                                       const double* __restrict__ E, long long R, long long nsb_stride,
                                                       double* __restrict__ lufs, int normalize, double target,
                                                       float* __restrict__ gain) {
  __shared__ double red[kT];
  __shared__ long long redc[kT];
  __shared__ float wmax[kT / 32];
  const int b = blockIdx.x, tid = threadIdx.x;
  const long long n = lens.v[b], s = gt.s, nsb = n / s, J = nsb >= 3 ? nsb - 3 : 0, Rb = (n + kSpan - 1) / kSpan;
  const double* Eb = E + (long long)b * nsb_stride;
  float m = 0.0f;
  for (long long c = tid; c < Rb; c += kT) m = fmaxf(m, cmax[(long long)b * R + c]);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
  if ((tid & 31) == 0) wmax[tid >> 5] = m;
  __syncthreads();
  for (int w = 0; w < kT / 32; ++w) m = fmaxf(m, wmax[w]);
  const double inv4s = 1.0 / (4.0 * (double)s);
  double sum = 0.0;
  long long cnt = 0;
  for (long long j = tid; j < J; j += kT) {
    const double z = block_z(Eb, j, inv4s);
    if (z > gt.abs_e) {
      sum += z;
      ++cnt;
    }
  }
  block_sum(sum, cnt, red, redc);
  double L = -INFINITY;
  if (cnt > 0) {
    const double rel_e = sum / (double)cnt * gt.rel;
    sum = 0.0;
    cnt = 0;
    for (long long j = tid; j < J; j += kT) {
      const double z = block_z(Eb, j, inv4s);
      if (z > gt.abs_e && z > rel_e) {
        sum += z;
        ++cnt;
      }
    }
    block_sum(sum, cnt, red, redc);
    if (cnt > 0) L = -0.691 + 10.0 * log10(sum / (double)cnt);
  }
  if (tid == 0) {
    lufs[b] = L;
    if (normalize) {
      double g64 = 1.0;
      if (isfinite(L)) g64 = fmin(pow(10.0, (target - L) / 20.0), gt.ceil_amp / (double)m);
      // toward zero: 10^(-1/20) lies just below the midpoint above its fp32 value, so a gain rounded up by half an ulp
      // would put the peak sample one ulp over fp32(10^(-1/20))
      gain[b] = __double2float_rz(g64);
    }
  }
}

// y = g * x over [0, lens[b]); y may alias x
__global__ void __launch_bounds__(kT) loud_apply_kernel(const float* x, long long x_stride, RowLens<kRowsPerLaunch> lens, const float* __restrict__ gain,
                                                        float* y, long long y_stride) {
  const int b = blockIdx.y;
  const long long n = lens.v[b];
  const float g = gain[b];
  const float* xb = x + (long long)b * x_stride;
  float* yb = y + (long long)b * y_stride;
  for (long long j = (long long)blockIdx.x * kT + threadIdx.x; j < n; j += (long long)gridDim.x * kT) yb[j] = __fmul_rn(g, xb[j]);
}

int check_batch(const float* x, int B, long long x_stride, const int64_t* lens_host, int sr, void* ws, long long* most) {
  if (!ws) return fail(SOPRO_ERR_INVALID, "null argument");
  if (!valid_rate(sr)) return fail(SOPRO_ERR_INVALID, "sample rate %d not in [%d, %d]", sr, kMinRate, kMaxRate);
  return check_rows(x, B, x_stride, lens_host, kMaxLen, most);
}

// the meter over rows [b0, b0 + rows): L -> lufs[b0 ..], and with `normalize` g -> gain[b0 ..]
int run_meter(const Filt& f, const Gate& gt, const Layout& l, const float* x, long long x_stride, const RowLens<kRowsPerLaunch>& L, int b0,
              int rows, char* ws, double* lufs, int normalize, double target, float* gain, cudaStream_t st) {
  St* v = reinterpret_cast<St*>(ws + l.v) + (long long)b0 * l.R * kT;
  double* e = reinterpret_cast<double*>(ws + l.e) + 2LL * b0 * l.R * kT;
  St* agg = reinterpret_cast<St*>(ws + l.agg) + (long long)b0 * l.R;
  St* carry = reinterpret_cast<St*>(ws + l.carry) + (long long)b0 * l.R;
  float* cmax = reinterpret_cast<float*>(ws + l.cmax) + (long long)b0 * l.R;
  double* E = reinterpret_cast<double*>(ws + l.E) + (long long)b0 * l.nsb;
  const float* xb = x + (long long)b0 * x_stride;
  if (l.R > 0) {
    const dim3 grid((unsigned)l.R, rows);
    loud_scan_kernel<<<grid, kT, 0, st>>>(f, xb, x_stride, L, v, agg, l.R);
    CK(cudaGetLastError());
    loud_carry_kernel<<<rows, kT, 0, st>>>(f, L, agg, carry, l.R);
    CK(cudaGetLastError());
    loud_energy_kernel<<<grid, kT, 0, st>>>(f, gt.s, xb, x_stride, L, v, carry, e, cmax, l.R);
    CK(cudaGetLastError());
  }
  if (l.nsb > 0) {
    loud_subblock_kernel<<<dim3((unsigned)((l.nsb + kT / 32 - 1) / (kT / 32)), rows), kT, 0, st>>>(gt.s, L, e, E, l.R, l.nsb);
    CK(cudaGetLastError());
  }
  loud_gate_kernel<<<rows, kT, 0, st>>>(gt, L, cmax, E, l.R, l.nsb, lufs + b0, normalize, target, gain ? gain + b0 : nullptr);
  CK(cudaGetLastError());
  return SOPRO_OK;
}

bool valid_target(double T) { return T >= -60.0 && T <= 0.0; }  // also refuses NaN

}  // namespace

extern "C" {

int sopro_loudness_filter(int32_t sr, double* c) {
  if (!c) return fail(SOPRO_ERR_INVALID, "null argument");
  if (!valid_rate(sr)) return fail(SOPRO_ERR_INVALID, "sample rate %d not in [%d, %d]", sr, kMinRate, kMaxRate);
  coeffs(sr, c);
  return SOPRO_OK;
}

int sopro_loudness_target(double T) {
  if (!valid_target(T)) return fail(SOPRO_ERR_INVALID, "loudness target must be a real number in [-60, 0] LUFS (got %g)", T);
  return SOPRO_OK;
}

int64_t sopro_loudness_workspace(int32_t B, int64_t max_len, int32_t sr) {
  if (B < 1 || max_len < 0 || max_len > kMaxLen || !valid_rate(sr)) return -1;
  return (int64_t)layout(B, max_len, sr).total;
}

int sopro_loudness_measure(const float* x, int32_t B, int64_t x_stride, const int64_t* lens_host, int32_t sr, void* ws,
                           double* lufs_dev, void* stream) {
  long long most = 0;
  const int rc = check_batch(x, B, x_stride, lens_host, sr, ws, &most);
  if (rc != SOPRO_OK) return rc;
  if (!lufs_dev) return fail(SOPRO_ERR_INVALID, "null argument");
  const Filt f = make_filt(sr);
  const Gate gt = make_gate(sr);
  const Layout l = layout(B, most, sr);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  for (int b0 = 0; b0 < B; b0 += kRowsPerLaunch) {
    const int rows = std::min(kRowsPerLaunch, B - b0);
    const RowLens<kRowsPerLaunch> L = row_lens<kRowsPerLaunch>(lens_host, x_stride, b0, rows);
    const int r = run_meter(f, gt, l, x, x_stride, L, b0, rows, static_cast<char*>(ws), lufs_dev, 0, 0.0, nullptr, st);
    if (r != SOPRO_OK) return r;
  }
  return SOPRO_OK;
}

int sopro_loudness_normalize(const float* x, int32_t B, int64_t x_stride, const int64_t* lens_host, int32_t sr, double T,
                             float* y, int64_t y_stride, void* ws, double* lufs_dev, float* gain_dev, void* stream) {
  if (!valid_target(T)) return fail(SOPRO_ERR_INVALID, "loudness target must be a real number in [-60, 0] LUFS (got %g)", T);
  long long most = 0;
  int rc = check_batch(x, B, x_stride, lens_host, sr, ws, &most);
  if (rc == SOPRO_OK) rc = check_out_rows(y, B, y_stride, most);
  if (rc != SOPRO_OK) return rc;
  const Filt f = make_filt(sr);
  const Gate gt = make_gate(sr);
  const Layout l = layout(B, most, sr);
  char* w = static_cast<char*>(ws);
  double* lufs = lufs_dev ? lufs_dev : reinterpret_cast<double*>(w + l.L);
  float* gain = gain_dev ? gain_dev : reinterpret_cast<float*>(w + l.g);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  for (int b0 = 0; b0 < B; b0 += kRowsPerLaunch) {
    const int rows = std::min(kRowsPerLaunch, B - b0);
    const RowLens<kRowsPerLaunch> L = row_lens<kRowsPerLaunch>(lens_host, x_stride, b0, rows);
    const int r = run_meter(f, gt, l, x, x_stride, L, b0, rows, w, lufs, 1, T, gain, st);
    if (r != SOPRO_OK) return r;
    if (most > 0) {
      const long long gx = std::min<long long>((most + kT - 1) / kT, 4096);
      loud_apply_kernel<<<dim3((unsigned)gx, rows), kT, 0, st>>>(x + (long long)b0 * x_stride, x_stride, L, gain + b0,
                                                                  y + (long long)b0 * y_stride, y_stride);
      CK(cudaGetLastError());
    }
  }
  return SOPRO_OK;
}

}  // extern "C"
