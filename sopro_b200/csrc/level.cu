// Live loudness: a causal BS.1770 leveller whose gain follows the integrated loudness of the audio so far, one-shot
// over a ragged batch or streamed chunk by chunk.  The definition is in include/sopro_b200.h (oracle/loudness_live_oracle.py
// in float64); it reuses the one-shot meter's K-weighting, sub-blocks, blocks and gates (loudness.cu), and releases
// audio in whole sub-blocks so that each one's peak is known before it goes out.
//
// Everything below is a function of sub-block k and the row's samples, never of how the row was pushed:
//   agg_k:  the filter's state at the end of sub-block k from zero state at its start (one CTA: a piece of P samples per
//           thread from its start, a Kogge-Stone scan with the powers A^(P 2^i), then the short last piece filtered);
//   s_k:    the state at the end of sub-block k, s_k = A^s s_{k-1} + agg_k, s_{-1} = 0 (one 4x4 fma chain);
//   E_k:    y^2 over sub-block k from the start state s_{k-1} (the scan again, each piece re-filtered, a fixed tree);
//   gates:  z_j = (((E_j + E_{j+1}) + E_{j+2}) + E_{j+3}) / (4 s); the absolute-gated sum and count run in increasing j;
//           M_k's relative-gated sum over j in [0, k - 2) is one CTA's strided sum and fixed tree, an order set by k alone;
//   gains:  a_k = min(10^((T - M_k) / 20), 10^(B / 20)), 1 when M_k = -inf;
//   output: per released range, g = fp32_rz(min(r, c)) with r the ramp in double and c = 10^(-1/20) / max|x| over the
//           range; y = g * x, one fp32 multiply.
// The one-shot (sopro_level) runs each step for every sub-block in parallel (the two serial chains, s_k and the absolute
// sums, one thread per row); the stream runs them in sub-block order in one CTA per push.  Both call the same device
// functions, so a stream's output equals the one-shot's bit for bit under any push schedule.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>

#include "../../include/sopro_b200.h"
#include "chunk_stream.cuh"
#include "common.cuh"

namespace {

using chunk::Src;
using chunk::src_at;

constexpr int kLogT = 8, kT = 1 << kLogT;  // threads per CTA (and pieces per sub-block at most)
constexpr int kRowsPerLaunch = 128;
constexpr long long kMaxLen = 1LL << 40;
constexpr int kMinRate = 4000, kMaxRate = 192000;
// the largest gain a_k may take: a first block that barely passes the -70 LUFS absolute gate (a breath, room tone)
// would otherwise be raised by 50 dB or more before any speech has been metered
constexpr double kMaxBoostDb = 30.0;
// the block-energy store a new stream starts with: ten minutes at 10 sub-blocks a second (48 KB); it doubles as needed
constexpr long long kStoreStart = 6000;

struct Mat {
  double m[4][4];
};

// the filter: the shelf's numerator, both negated denominators, P, A^(P 2^i) for i = 0 .. log2 T - 1, and A^s
struct LFilt {
  double b0, b1, b2, na11, na12, na21, na22;
  int s, P;
  Mat pw[kLogT];
  Mat As;
};

struct LGate {
  int s;
  double abs_e;     // 10^((-70 + 0.691) / 10)
  double rel;       // 10^(-10 / 10)
  double ceil_amp;  // 10^(-1 / 20)
  double boost;     // 10^(kMaxBoostDb / 20)
  double T;         // the target, LUFS
};

struct St {
  double v[4];
};

// what a stream carries on the device from one push to the next
struct LvDev {
  double st[4];  // s_{k-1}
  double sabs;   // the absolutely gated sum and count so far
  long long cabs;
  double a_prev;  // a_{k-1}
};

bool valid_rate(int sr) { return sr >= kMinRate && sr <= kMaxRate; }
bool valid_target(double T) { return T >= -60.0 && T <= 0.0; }
int sub_block(int sr) { return (sr + 5) / 10; }

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

// A^e by squaring, e >= 1
Mat matpow(const Mat& A, long long e) {
  Mat r = A, b = A;
  --e;
  while (e > 0) {
    if (e & 1) r = matmul(r, b);
    b = matmul(b, b);
    e >>= 1;
  }
  return r;
}

LFilt make_filt(int sr) {
  double c[10];
  sopro_loudness_filter(sr, c);  // the one-shot meter's coefficients
  LFilt f{};
  f.b0 = c[0];
  f.b1 = c[1];
  f.b2 = c[2];
  f.na11 = -c[3];
  f.na12 = -c[4];
  f.na21 = -c[8];
  f.na22 = -c[9];
  f.s = sub_block(sr);
  f.P = (f.s + kT - 1) / kT;
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
  f.pw[0] = matpow(A, f.P);
  for (int k = 1; k < kLogT; ++k) f.pw[k] = matmul(f.pw[k - 1], f.pw[k - 1]);
  f.As = matpow(A, f.s);
  return f;
}

LGate make_gate(int sr, double T) {
  return LGate{sub_block(sr), std::pow(10.0, (-70.0 + 0.691) / 10.0), std::pow(10.0, -10.0 / 10.0), std::pow(10.0, -1.0 / 20.0),
               std::pow(10.0, kMaxBoostDb / 20.0), T};
}

// the one-shot workspace: per row and sub-block agg, s, E, the absolute sums and counts, a and M
struct Layout {
  long long nsb = 0;
  size_t agg = 0, S = 0, E = 0, sabs = 0, cabs = 0, a = 0, M = 0, total = 0;
};

Layout layout(int B, long long max_len, int sr) {
  Layout l;
  l.nsb = max_len / sub_block(sr);
  size_t off = 0;
  auto take = [&](size_t bytes) {
    const size_t o = off;
    off += (bytes + 255) & ~(size_t)255;
    return o;
  };
  const size_t n = (size_t)B * (size_t)l.nsb;
  l.agg = take(n * sizeof(St));
  l.S = take(n * sizeof(St));
  l.E = take(n * sizeof(double));
  l.sabs = take(n * sizeof(double));
  l.cabs = take(n * sizeof(long long));
  l.a = take(n * sizeof(double));
  l.M = take(n * sizeof(double));
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

// samples [g0, g1) from state st (u1, u2, y1, y2), the input history read through the source; with kEnergy, y^2 is
// summed into e in sample order
template <bool kEnergy>
__device__ __forceinline__ void lv_piece(const LFilt& f, const Src& src, long long g0, long long g1, double st[4], double& e) {
  double x2 = src_at(src, g0 - 2), x1 = src_at(src, g0 - 1);
  double u1 = st[0], u2 = st[1], y1 = st[2], y2 = st[3];
  for (long long g = g0; g < g1; ++g) {
    const double x0 = src_at(src, g);
    const double u = fma(f.na11, u1, fma(f.na12, u2, fma(f.b0, x0, fma(f.b1, x1, __dmul_rn(f.b2, x2)))));
    const double y = fma(f.na21, y1, fma(f.na22, y2, __dadd_rn(fma(-2.0, u1, u), u2)));
    if (kEnergy) e = fma(y, y, e);
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

struct Shm {
  double sc[4][kT];
  double red[kT];
  long long redc[kT];
  float wmax[kT / 32];
};

// inclusive Kogge-Stone scan of the threads' piece states: s_i <- s_i + A^(P 2^k) s_{i - 2^k}
__device__ __forceinline__ void lv_scan(const LFilt& f, double s[4], Shm& sm) {
  const int tid = threadIdx.x;
#pragma unroll
  for (int k = 0; k < kLogT; ++k) {
#pragma unroll
    for (int r = 0; r < 4; ++r) sm.sc[r][tid] = s[r];
    __syncthreads();
    if (tid >= (1 << k)) {
      double p[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) p[r] = sm.sc[r][tid - (1 << k)];
      mat_acc(f.pw[k], p, s);
    }
    __syncthreads();
  }
}

// the start states of sub-block k's pieces, given the state c at its start (zero for agg): every piece but the last is
// filtered from zero, c enters through piece 0, the scan carries it; thread i's start state -> st
__device__ __forceinline__ void lv_starts(const LFilt& f, const Src& src, long long k, const double c[4], double st[4], Shm& sm) {
  const int tid = threadIdx.x, np = (f.s + f.P - 1) / f.P;
  const long long g0 = k * f.s + (long long)tid * f.P;
  double v[4] = {0.0, 0.0, 0.0, 0.0}, e = 0.0;
  if (tid < np - 1) lv_piece<false>(f, src, g0, g0 + f.P, v, e);
  if (tid == 0) mat_acc(f.pw[0], c, v);
  lv_scan(f, v, sm);
#pragma unroll
  for (int r = 0; r < 4; ++r) sm.sc[r][tid] = v[r];
  __syncthreads();
#pragma unroll
  for (int r = 0; r < 4; ++r) st[r] = tid ? sm.sc[r][tid - 1] : c[r];
  __syncthreads();
}

// thread i's piece of sub-block k: [g0, g1), empty past the last
__device__ __forceinline__ void lv_piece_range(const LFilt& f, long long k, long long& g0, long long& g1) {
  const long long e = (k + 1) * f.s;
  g0 = std::min(k * f.s + (long long)threadIdx.x * f.P, e);
  g1 = std::min(g0 + f.P, e);
}

// agg_k -> out (every thread)
__device__ __forceinline__ void lv_agg(const LFilt& f, const Src& src, long long k, double out[4], Shm& sm) {
  const int tid = threadIdx.x, np = (f.s + f.P - 1) / f.P;
  const double zero[4] = {0.0, 0.0, 0.0, 0.0};
  double st[4], e = 0.0;
  lv_starts(f, src, k, zero, st, sm);
  if (tid == np - 1) {
    long long g0, g1;
    lv_piece_range(f, k, g0, g1);
    lv_piece<false>(f, src, g0, g1, st, e);
#pragma unroll
    for (int r = 0; r < 4; ++r) sm.sc[r][0] = st[r];
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < 4; ++r) out[r] = sm.sc[r][0];
  __syncthreads();
}

// a fixed tree over the CTA's threads (every thread gets the sums)
__device__ __forceinline__ void lv_tree(double& v, long long& cnt, Shm& sm) {
  const int tid = threadIdx.x;
  sm.red[tid] = v;
  sm.redc[tid] = cnt;
  __syncthreads();
  for (int h = kT / 2; h > 0; h >>= 1) {
    if (tid < h) {
      sm.red[tid] = __dadd_rn(sm.red[tid], sm.red[tid + h]);
      sm.redc[tid] += sm.redc[tid + h];
    }
    __syncthreads();
  }
  v = sm.red[0];
  cnt = sm.redc[0];
  __syncthreads();
}

// E_k from the start state c (every thread)
__device__ __forceinline__ double lv_energy(const LFilt& f, const Src& src, long long k, const double c[4], Shm& sm) {
  double st[4], e = 0.0;
  lv_starts(f, src, k, c, st, sm);
  long long g0, g1;
  lv_piece_range(f, k, g0, g1);
  lv_piece<true>(f, src, g0, g1, st, e);
  long long n = 0;
  lv_tree(e, n, sm);
  return e;
}

__device__ __forceinline__ double lv_z(const double* E, long long j, double inv4s) {
  return __dmul_rn(__dadd_rn(__dadd_rn(__dadd_rn(E[j], E[j + 1]), E[j + 2]), E[j + 3]), inv4s);
}

// the absolute gate's running sum and count after block j (one thread)
__device__ __forceinline__ void lv_abs_step(const LGate& gt, const double* E, long long j, double& sabs, long long& cabs) {
  const double z = lv_z(E, j, 1.0 / (4.0 * (double)gt.s));
  if (z > gt.abs_e) {
    sabs = __dadd_rn(sabs, z);
    ++cabs;
  }
}

// M over blocks [0, J), given the absolute gate's sum and count over them (every thread)
__device__ __forceinline__ double lv_meter(const LGate& gt, const double* E, long long J, double sabs, long long cabs, Shm& sm) {
  if (cabs == 0) return -INFINITY;
  const double inv4s = 1.0 / (4.0 * (double)gt.s);
  const double rel_e = __dmul_rn(__ddiv_rn(sabs, (double)cabs), gt.rel);
  double sum = 0.0;
  long long cnt = 0;
  for (long long j = threadIdx.x; j < J; j += kT) {
    const double z = lv_z(E, j, inv4s);
    if (z > gt.abs_e && z > rel_e) {
      sum = __dadd_rn(sum, z);
      ++cnt;
    }
  }
  lv_tree(sum, cnt, sm);
  return cnt > 0 ? __dadd_rn(-0.691, __dmul_rn(10.0, log10(__ddiv_rn(sum, (double)cnt)))) : -INFINITY;
}

__device__ __forceinline__ double lv_gain(const LGate& gt, double M) {
  return isfinite(M) ? fmin(pow(10.0, __ddiv_rn(__dsub_rn(gt.T, M), 20.0)), gt.boost) : 1.0;
}

// y[t - t0] for t in [t0, t1): g = fp32_rz(min(a0 + (a1 - a0) (i + 1) / s, c)), i = t - t0, c = 10^(-1/20) / max|x| over
// [t0, t1) (every thread)
__device__ __forceinline__ void lv_release(const LGate& gt, const Src& src, long long t0, long long t1, double a0, double a1,
                                           float* __restrict__ y, Shm& sm) {
  const int tid = threadIdx.x;
  float m = 0.0f;
  for (long long t = t0 + tid; t < t1; t += kT) m = fmaxf(m, fabsf(src_at(src, t)));
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
  if ((tid & 31) == 0) sm.wmax[tid >> 5] = m;
  __syncthreads();
  for (int w = 0; w < kT / 32; ++w) m = fmaxf(m, sm.wmax[w]);
  __syncthreads();
  const double c = m > 0.0f ? gt.ceil_amp / (double)m : INFINITY, d = __dsub_rn(a1, a0), s = (double)gt.s;
  for (long long t = t0 + tid; t < t1; t += kT) {
    const double r = __dadd_rn(a0, __dmul_rn(d, __ddiv_rn((double)(t - t0 + 1), s)));
    y[t - t0] = __fmul_rn(__double2float_rz(fmin(r, c)), src_at(src, t));
  }
}

__device__ __forceinline__ Src row_src(const float* x, long long n) { return Src{x, nullptr, 0, n, n}; }

// one-shot, grid (sub-blocks, rows): agg_k
__global__ void __launch_bounds__(kT) lv_agg_kernel(LFilt f, const float* __restrict__ x, long long x_stride, RowLens<kRowsPerLaunch> lens,
                                                    St* __restrict__ agg, long long nsb) {
  __shared__ Shm sm;
  const int b = blockIdx.y;
  const long long k = blockIdx.x, n = lens.v[b];
  if (k >= n / f.s) return;
  double a[4];
  lv_agg(f, row_src(x + (long long)b * x_stride, n), k, a, sm);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int r = 0; r < 4; ++r) agg[(long long)b * nsb + k].v[r] = a[r];
  }
}

// one-shot, one thread per row: s_k = A^s s_{k-1} + agg_k in increasing k
__global__ void lv_chain_kernel(LFilt f, RowLens<kRowsPerLaunch> lens, const St* __restrict__ agg, St* __restrict__ S, long long nsb, int rows) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= rows) return;
  const long long m = lens.v[b] / f.s;
  double s[4] = {0.0, 0.0, 0.0, 0.0};
  for (long long k = 0; k < m; ++k) {
    double a[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) a[r] = agg[(long long)b * nsb + k].v[r];
    mat_acc(f.As, s, a);
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      s[r] = a[r];
      S[(long long)b * nsb + k].v[r] = a[r];
    }
  }
}

// one-shot, grid (sub-blocks, rows): E_k from s_{k-1}
__global__ void __launch_bounds__(kT) lv_energy_kernel(LFilt f, const float* __restrict__ x, long long x_stride, RowLens<kRowsPerLaunch> lens,
                                                       const St* __restrict__ S, double* __restrict__ E, long long nsb) {
  __shared__ Shm sm;
  const int b = blockIdx.y;
  const long long k = blockIdx.x, n = lens.v[b];
  if (k >= n / f.s) return;
  double c[4] = {0.0, 0.0, 0.0, 0.0};
  if (k > 0) {
#pragma unroll
    for (int r = 0; r < 4; ++r) c[r] = S[(long long)b * nsb + k - 1].v[r];
  }
  const double e = lv_energy(f, row_src(x + (long long)b * x_stride, n), k, c, sm);
  if (threadIdx.x == 0) E[(long long)b * nsb + k] = e;
}

// one-shot, one thread per row: the absolute gate's sum and count over blocks [0, k - 2) for every k >= 3
__global__ void lv_abs_kernel(LGate gt, RowLens<kRowsPerLaunch> lens, const double* __restrict__ E, double* __restrict__ sabs,
                              long long* __restrict__ cabs, long long nsb, int rows) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= rows) return;
  const long long m = lens.v[b] / gt.s;
  const double* Eb = E + (long long)b * nsb;
  double sa = 0.0;
  long long ca = 0;
  for (long long k = 3; k < m; ++k) {
    lv_abs_step(gt, Eb, k - 3, sa, ca);
    sabs[(long long)b * nsb + k] = sa;
    cabs[(long long)b * nsb + k] = ca;
  }
}

// one-shot, grid (sub-blocks, rows): M_k and a_k for k >= 3 (NaN below)
__global__ void __launch_bounds__(kT) lv_meter_kernel(LGate gt, RowLens<kRowsPerLaunch> lens, const double* __restrict__ E,
                                                      const double* __restrict__ sabs, const long long* __restrict__ cabs,
                                                      double* __restrict__ A, double* __restrict__ Mo, long long nsb) {
  __shared__ Shm sm;
  const int b = blockIdx.y;
  const long long k = blockIdx.x, o = (long long)b * nsb + k;
  if (k >= lens.v[b] / gt.s) return;
  if (k < 3) {
    if (threadIdx.x == 0) A[o] = Mo[o] = NAN;
    return;
  }
  const double M = lv_meter(gt, E + (long long)b * nsb, k - 2, sabs[o], cabs[o], sm);
  if (threadIdx.x == 0) {
    Mo[o] = M;
    A[o] = lv_gain(gt, M);
  }
}

// one-shot, grid (sub-blocks + 1, rows): CTA q releases sub-block q (the tail for q = floor(n / s)) by rules 3-5
__global__ void __launch_bounds__(kT) lv_apply_kernel(LGate gt, const float* __restrict__ x, long long x_stride, RowLens<kRowsPerLaunch> lens,
                                                      const double* __restrict__ A, long long nsb, float* __restrict__ y, long long y_stride) {
  __shared__ Shm sm;
  const int b = blockIdx.y;
  const long long q = blockIdx.x, n = lens.v[b], s = gt.s, m = n / s;
  if (q > m) return;
  const double* Ab = A + (long long)b * nsb;
  const long long t0 = q * s, t1 = q < m ? t0 + s : n;
  if (t1 <= t0) return;
  double a0 = 1.0, a1 = 1.0;
  if (m >= 4) {
    if (q == m) a0 = a1 = Ab[m - 1];
    else if (q <= 3) a0 = a1 = Ab[3];
    else {
      a0 = Ab[q - 1];
      a1 = Ab[q];
    }
  }
  lv_release(gt, row_src(x + (long long)b * x_stride, n), t0, t1, a0, a1, y + (long long)b * y_stride + t0, sm);
}

// a stream's push: sub-blocks [k0, k1) complete, each metered and released in order; with `final`, the rest of the row's
// n samples after them.  y receives the released samples from sample `out0` on.
__global__ void __launch_bounds__(kT) lv_stream_kernel(LFilt f, LGate gt, Src src, long long k0, long long k1, int final, long long n,
                                                       double* __restrict__ E, LvDev* __restrict__ dev, float* __restrict__ y, long long out0) {
  __shared__ Shm sm;
  __shared__ LvDev d;
  const long long s = f.s;
  if (threadIdx.x == 0) {
    if (k0 > 0) d = *dev;
    else d = LvDev{{0.0, 0.0, 0.0, 0.0}, 0.0, 0, 1.0};
  }
  __syncthreads();
  for (long long k = k0; k < k1; ++k) {
    double agg[4], c[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) c[r] = d.st[r];
    lv_agg(f, src, k, agg, sm);
    const double e = lv_energy(f, src, k, c, sm);
    if (threadIdx.x == 0) {
      mat_acc(f.As, c, agg);
#pragma unroll
      for (int r = 0; r < 4; ++r) d.st[r] = agg[r];
      E[k] = e;
      if (k >= 3) lv_abs_step(gt, E, k - 3, d.sabs, d.cabs);
    }
    __syncthreads();
    if (k < 3) continue;
    const double a = lv_gain(gt, lv_meter(gt, E, k - 2, d.sabs, d.cabs, sm));
    if (k == 3) {
      for (long long q = 0; q < 4; ++q) lv_release(gt, src, q * s, (q + 1) * s, a, a, y + (q * s - out0), sm);
    } else {
      lv_release(gt, src, k * s, (k + 1) * s, d.a_prev, a, y + (k * s - out0), sm);
    }
    __syncthreads();
    if (threadIdx.x == 0) d.a_prev = a;
    __syncthreads();
  }
  if (final) {
    const long long m = n / s;
    if (m < 4)
      for (long long q = 0; q < m; ++q) lv_release(gt, src, q * s, (q + 1) * s, 1.0, 1.0, y + (q * s - out0), sm);
    if (n > m * s) {
      const double a = m >= 4 ? d.a_prev : 1.0;
      lv_release(gt, src, m * s, n, a, a, y + (m * s - out0), sm);
    }
  }
  if (threadIdx.x == 0) *dev = d;
}

// samples released once n have arrived: every complete sub-block once four are, none before
long long released(long long n, long long s) {
  const long long m = n / s;
  return m >= 4 ? m * s : 0;
}

}  // namespace

// the tail holds [released - 2, seen): the unreleased samples and the two before them (the filter's input history)
struct sopro_level_stream : chunk::ChunkStream {
  int sr = 0;
  LFilt f{};
  LGate gt{};
  LvDev* dev = nullptr;
  double* E = nullptr;         // the block-energy store, stream-ordered
  long long cap = 0;           // its capacity in sub-blocks
  cudaStream_t last = nullptr;  // the stream of the last launch, where the store is freed

  cudaError_t alloc_own() {
    cudaError_t e = cudaMalloc(&dev, sizeof(LvDev));
    if (e == cudaSuccess) e = cudaMallocAsync(&E, (size_t)kStoreStart * sizeof(double), 0);
    if (e == cudaSuccess) e = cudaStreamSynchronize(0);
    if (e == cudaSuccess) cap = kStoreStart;
    return e;
  }
  void free_own() {
    cudaFree(dev);
    cudaFreeAsync(E, last);
  }
};

namespace {

// room in the store for sub-blocks [0, m): doubled, copied and freed in stream order, so no call waits on the device
int grow(sopro_level_stream* s, long long m, cudaStream_t st) {
  if (m <= s->cap) return SOPRO_OK;
  long long cap = s->cap;
  while (cap < m) cap *= 2;
  double* p = nullptr;
  CK(cudaMallocAsync(&p, (size_t)cap * sizeof(double), st));
  const long long have = s->tail.seen / s->f.s;
  if (have > 0) CK(cudaMemcpyAsync(p, s->E, (size_t)have * sizeof(double), cudaMemcpyDeviceToDevice, st));
  CK(cudaFreeAsync(s->E, st));
  s->E = p;
  s->cap = cap;
  return SOPRO_OK;
}

int launch(sopro_level_stream* s, const float* x, long long n, int final, float* y, cudaStream_t st) {
  const long long sb = s->f.s, seen = s->tail.seen, k0 = seen / sb, k1 = (seen + n) / sb;
  if (k1 == k0 && !final) return SOPRO_OK;
  int rc = grow(s, k1, st);
  if (rc != SOPRO_OK) return rc;
  s->last = st;
  lv_stream_kernel<<<1, kT, 0, st>>>(s->f, s->gt, s->tail.src(x, n), k0, k1, final, seen + n, s->E, s->dev, y, released(seen, sb));
  CK(cudaGetLastError());
  return SOPRO_OK;
}

}  // namespace

extern "C" {

int64_t sopro_level_workspace(int32_t B, int64_t max_len, int32_t sr) {
  if (B < 1 || max_len < 0 || max_len > kMaxLen || !valid_rate(sr)) return -1;
  return (int64_t)layout(B, max_len, sr).total;
}

int sopro_level(const float* x, int32_t B, int64_t x_stride, const int64_t* lens_host, int32_t sr, double T, float* y,
                int64_t y_stride, void* ws, double* meter_dev, double* gain_dev, void* stream) {
  if (!valid_target(T)) return fail(SOPRO_ERR_INVALID, "loudness target must be a real number in [-60, 0] LUFS (got %g)", T);
  if (!ws) return fail(SOPRO_ERR_INVALID, "null argument");
  if (!valid_rate(sr)) return fail(SOPRO_ERR_INVALID, "sample rate %d not in [%d, %d]", sr, kMinRate, kMaxRate);
  long long most = 0;
  int rc = check_rows(x, B, x_stride, lens_host, kMaxLen, &most);
  if (rc == SOPRO_OK) rc = check_out_rows(y, B, y_stride, most);
  if (rc != SOPRO_OK) return rc;
  const LFilt f = make_filt(sr);
  const LGate gt = make_gate(sr, T);
  const Layout l = layout(B, most, sr);
  char* w = static_cast<char*>(ws);
  St* agg = reinterpret_cast<St*>(w + l.agg);
  St* S = reinterpret_cast<St*>(w + l.S);
  double* E = reinterpret_cast<double*>(w + l.E);
  double* sabs = reinterpret_cast<double*>(w + l.sabs);
  long long* cabs = reinterpret_cast<long long*>(w + l.cabs);
  double* A = gain_dev ? gain_dev : reinterpret_cast<double*>(w + l.a);
  double* M = meter_dev ? meter_dev : reinterpret_cast<double*>(w + l.M);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  for (int b0 = 0; b0 < B; b0 += kRowsPerLaunch) {
    const int rows = std::min(kRowsPerLaunch, B - b0);
    const RowLens<kRowsPerLaunch> L = row_lens<kRowsPerLaunch>(lens_host, x_stride, b0, rows);
    const float* xb = x + (long long)b0 * x_stride;
    const long long o = (long long)b0 * l.nsb;
    if (l.nsb > 0) {
      const dim3 grid((unsigned)l.nsb, rows);
      lv_agg_kernel<<<grid, kT, 0, st>>>(f, xb, x_stride, L, agg + o, l.nsb);
      CK(cudaGetLastError());
      lv_chain_kernel<<<(rows + 31) / 32, 32, 0, st>>>(f, L, agg + o, S + o, l.nsb, rows);
      CK(cudaGetLastError());
      lv_energy_kernel<<<grid, kT, 0, st>>>(f, xb, x_stride, L, S + o, E + o, l.nsb);
      CK(cudaGetLastError());
      lv_abs_kernel<<<(rows + 31) / 32, 32, 0, st>>>(gt, L, E + o, sabs + o, cabs + o, l.nsb, rows);
      CK(cudaGetLastError());
      lv_meter_kernel<<<grid, kT, 0, st>>>(gt, L, E + o, sabs + o, cabs + o, A + o, M + o, l.nsb);
      CK(cudaGetLastError());
    }
    if (most > 0) {
      lv_apply_kernel<<<dim3((unsigned)(l.nsb + 1), rows), kT, 0, st>>>(gt, xb, x_stride, L, A + o, l.nsb,
                                                                         y + (long long)b0 * y_stride, y_stride);
      CK(cudaGetLastError());
    }
  }
  return SOPRO_OK;
}

int sopro_level_stream_create(int64_t max_chunk, int32_t sr, int device, sopro_level_stream_t** out) {
  int rc = chunk::check_create(max_chunk, out);
  if (rc == SOPRO_OK && !valid_rate(sr)) rc = fail(SOPRO_ERR_INVALID, "sample rate %d not in [%d, %d]", sr, kMinRate, kMaxRate);
  if (rc == SOPRO_OK) rc = open_device(device, "the live leveller");
  if (rc != SOPRO_OK) return rc;
  sopro_level_stream* s = new sopro_level_stream();
  s->sr = sr;
  s->f = make_filt(sr);
  s->unset = "target";
  return chunk::create(s, max_chunk, (size_t)(4 * s->f.s + 2), "live leveller", out);
}

int sopro_level_stream_destroy(sopro_level_stream_t* s) { return chunk::destroy(s); }

int sopro_level_stream_reset(sopro_level_stream_t* s, double T) {
  if (!s) return fail(SOPRO_ERR_INVALID, "null argument");
  if (!valid_target(T)) return fail(SOPRO_ERR_INVALID, "loudness target must be a real number in [-60, 0] LUFS (got %g)", T);
  s->gt = make_gate(s->sr, T);
  s->restart(-2);
  return SOPRO_OK;
}

int64_t sopro_level_stream_ready(const sopro_level_stream_t* s, int64_t n_more, int final) {
  if (!chunk::can_run(s, n_more)) return -1;
  const long long seen = s->tail.seen, sb = s->f.s;
  return (final ? seen + n_more : released(seen + n_more, sb)) - released(seen, sb);
}

int sopro_level_push(sopro_level_stream_t* s, const float* x, int64_t n, float* y, void* stream) {
  int rc = chunk::check_push(s, n);
  if (rc != SOPRO_OK || n == 0) return rc;
  const long long sb = s->f.s, seen = s->tail.seen;
  if ((rc = chunk::check_io(x, n, y, released(seen + n, sb) - released(seen, sb))) != SOPRO_OK) return rc;
  CK(cudaSetDevice(s->tail.device));
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  rc = launch(s, x, n, 0, y, st);
  if (rc == SOPRO_OK) rc = s->tail.keep(released(seen + n, sb) - 2, x, n, st);
  return rc;
}

int sopro_level_finish(sopro_level_stream_t* s, float* y, void* stream) {
  int rc = chunk::check_finish(s);
  if (rc != SOPRO_OK) return rc;
  const long long seen = s->tail.seen, left = seen - released(seen, s->f.s);
  if ((rc = chunk::check_io(nullptr, 0, y, left)) != SOPRO_OK) return rc;
  if (left > 0) {
    CK(cudaSetDevice(s->tail.device));
    rc = launch(s, nullptr, 0, 1, y, reinterpret_cast<cudaStream_t>(stream));
    if (rc != SOPRO_OK) return rc;
  }
  s->finished = true;
  return SOPRO_OK;
}

}  // extern "C"
