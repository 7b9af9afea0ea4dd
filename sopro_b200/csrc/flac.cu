// Lossless FLAC (RFC 9639) encoding of mono rows as 16-bit PCM, on the device.  The contract (include/sopro_b200.h,
// oracle/flac_oracle.py): x -> trunc(clamp(x, -1, 1) * 32767.0f), NaN -> 0; blocks of 4096 samples (the last of a row
// shorter); per block the smallest of CONSTANT, FIXED 0-4, LPC 1-12 (Levinson-Durbin in double with one rounding per
// operation, precision 12) and VERBATIM, each sized exactly, ties to the earlier; partitioned Rice with the exact
// cheapest parameter per partition, method and partition order.
//
// A block is (row, first sample, length, frame or sample number); the one-shot batch and the stream share the kernels:
//   analysis kernel: one CTA per block.  Samples to shared memory, the int64 autocorrelation, Levinson and the
//                    quantisation on one thread, then for every candidate the residuals and their exact Rice cost: each
//                    thread sums u >> k (k = 0 .. 30) over its 1/256 of the block, and a butterfly over the threads
//                    merges those sums partition order by partition order (8 .. 0), each group's leader adding its
//                    cheapest parameter's cost.  The decision and the frame's byte size go to a descriptor.
//   layout kernel:   one CTA per launch: a scan of the frame sizes (with each row's 42-byte STREAMINFO ahead of its
//                    frames) gives every frame's byte offset, each row's offset and size, and the min/max frame sizes;
//                    it writes the STREAMINFO blocks.
//   pack kernel:     one CTA per frame.  The winner's residuals again, its parameters from the same butterfly, per-thread
//                    code lengths and a scan for bit offsets; codes are OR-ed into the frame's 32-bit words in shared
//                    memory, the CRC-16 is per-thread table CRCs combined by multiplication by x^(8 len) mod the
//                    polynomial, and the frame's bytes go out with one writer per byte.
// Integer sums are order-free and the double arithmetic runs on one thread in a fixed order, so a row's bytes depend only
// on its own samples.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>

#include "../../include/sopro_b200.h"
#include "chunk_stream.cuh"

namespace {

constexpr int kBlock = 4096;            // samples per frame
constexpr int kT = 256;                 // threads per CTA; thread t owns samples [t n / 256, (t + 1) n / 256)
constexpr int kLogT = 8;
constexpr int kMaxLpc = 12, kMaxFixed = 4, kPrec = 12, kNK = 31;
constexpr int kRowsPerLaunch = 128;
constexpr int kInfoBytes = 42;          // fLaC + metadata header + STREAMINFO
constexpr int kMaxHdr = 16;             // frame header bound: 4 + 7 (UTF-8) + 2 (block size) + 1 (CRC-8), rounded up
constexpr int kMaxFrame = kMaxHdr + 1 + 2 * kBlock + 2;  // VERBATIM plus headers: the largest frame
constexpr int kWords = (kMaxFrame + 3) / 4 + 1;
constexpr long long kMaxLen = (1LL << 36) - 1;  // STREAMINFO's 36-bit total
constexpr int kMinRate = 4000, kMaxRate = 192000;
constexpr int kStreamMin = 16;          // frames shorter than this may only end a stream

enum Kind { kConst = 0, kVerbatim = 1, kFixed = 2, kLpc = 3 };

bool valid_rate(int sr) { return sr >= kMinRate && sr <= kMaxRate; }

int rate_code(int sr) {
  switch (sr) {
    case 8000: return 0x4;
    case 16000: return 0x5;
    case 22050: return 0x6;
    case 24000: return 0x7;
    case 32000: return 0x8;
    case 44100: return 0x9;
    case 48000: return 0xA;
    case 96000: return 0xB;
    case 88200: return 0x1;
    case 176400: return 0x2;
    case 192000: return 0x3;
    default: return 0x0;  // from STREAMINFO
  }
}

long long blocks_of(long long n) { return (n + kBlock - 1) / kBlock; }

// the rows of one launch: samples in this call and the prefix of their block counts
struct Rows {
  long long len[kRowsPerLaunch];
  long long blk0[kRowsPerLaunch + 1];
};

// where the samples of row r come from: a carried prefix (the stream's, at most 15 samples), then x + r * x_stride
struct Src {
  const float* x;
  long long x_stride;
  const float* carry;
  int carry_n;
};

struct Job {
  Src src;
  int rows;
  int variable;      // 0: fixed blocking, numbered by frame; 1: variable, numbered by first sample
  long long num0;    // the first sample's number (variable blocking)
  int sr, sr_code;
  int header;        // write each row's STREAMINFO ahead of its frames
};

struct Desc {
  int kind, order, shift, porder, method, hdr, bytes;
  short q[kMaxLpc];
};

__device__ __forceinline__ int q16(float v) {
  if (v != v) v = 0.0f;
  v = fminf(fmaxf(v, -1.0f), 1.0f);
  return (int)truncf(__fmul_rn(v, 32767.0f));
}

__device__ __forceinline__ int row_of(const Rows& R, int rows, long long blk) {
  int lo = 0, hi = rows - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (R.blk0[mid] <= blk) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// block -> (row, first sample, length, number)
__device__ __forceinline__ void block_geo(const Job& J, const Rows& R, long long blk, int& row, long long& first, int& n,
                                          long long& number) {
  row = row_of(R, J.rows, blk);
  const long long j = blk - R.blk0[row];
  first = j * kBlock;
  n = (int)min((long long)kBlock, R.len[row] - first);
  number = J.variable ? J.num0 + first : j;
}

__device__ __forceinline__ void load_block(const Src& S, int row, long long first, int n, int* s) {
  const float* xr = S.x + (long long)row * S.x_stride;
  for (int i = threadIdx.x; i < n; i += kT) {
    const long long g = first + i;
    s[i] = q16(g < S.carry_n ? S.carry[g] : xr[g - S.carry_n]);
  }
}

__host__ __device__ __forceinline__ int utf8_len(long long v) {
  if (v < 0x80) return 1;
  int nb = 2;
  while (nb < 7 && v >= (1LL << (5 * nb + 1))) ++nb;
  return nb;
}

__device__ __forceinline__ int header_bytes(int n, long long number) {
  return 4 + utf8_len(number) + (n == kBlock ? 0 : n <= 256 ? 1 : 2) + 1;
}

__device__ __forceinline__ int residual(const int* s, int i, int kind, int p, const short* q, int shift) {
  if (kind == kFixed) {
    switch (p) {
      case 0: return s[i];
      case 1: return s[i] - s[i - 1];
      case 2: return s[i] - 2 * s[i - 1] + s[i - 2];
      case 3: return s[i] - 3 * s[i - 1] + 3 * s[i - 2] - s[i - 3];
      default: return s[i] - 4 * s[i - 1] + 6 * s[i - 2] - 4 * s[i - 3] + s[i - 4];
    }
  }
  long long acc = 0;
  for (int j = 0; j < p; ++j) acc += (long long)q[j] * s[i - 1 - j];
  return s[i] - (int)(acc >> shift);
}

__device__ __forceinline__ unsigned zig(int r) { return r >= 0 ? 2u * (unsigned)r : 2u * (unsigned)(-(r + 1)) + 1u; }

// the largest partition order the block admits at predictor order p
__device__ __forceinline__ int max_porder(int n, int p) {
  int o = 0;
  while (o < 8 && n % (1 << (o + 1)) == 0 && (n >> (o + 1)) >= p) ++o;
  return o;
}

struct RiceSmem {
  unsigned long long wsum[kT / 32][kNK + 1];  // per warp: sum of u >> k, then the residual count
  unsigned long long cost[9][2];              // per partition order: sum of the partitions' cheapest cost, per method
  unsigned char kp[256];                      // plan mode: the parameter of each partition
};

// a partition's cheapest cost under method 0 (k <= 14) and 1 (k <= 30), ties to the smaller k
__device__ __forceinline__ void part_cost(const unsigned long long (&S)[kNK + 1], unsigned long long& c0, int& k0,
                                          unsigned long long& c1, int& k1) {
  const unsigned long long m = S[kNK];
  c0 = ~0ull;
  c1 = ~0ull;
  k0 = k1 = 0;
#pragma unroll
  for (int k = 0; k < kNK; ++k) {
    const unsigned long long c = m * (unsigned long long)(k + 1) + S[k];
    if (k <= 14 && c < c0) {
      c0 = c;
      k0 = k;
    }
    if (c < c1) {
      c1 = c;
      k1 = k;
    }
  }
}

// at group level l (groups of 2^l threads = partitions of order 8 - l), with the group's sums in S; every lane of the
// warp calls it (o <= omax is uniform), and the leaders' costs are summed over the warp before one atomic per warp
template <bool kPlan>
__device__ __forceinline__ void level(const unsigned long long (&S)[kNK + 1], int l, int part, bool leader, int omax,
                                      int plan_o, int plan_m, RiceSmem& R) {
  const int o = kLogT - l;
  if (o > omax) return;
  unsigned long long c0 = 0, c1 = 0;
  int k0 = 0, k1 = 0;
  if (leader) part_cost(S, c0, k0, c1, k1);
  if (kPlan) {
    if (leader && o == plan_o) R.kp[part] = (unsigned char)(plan_m ? k1 : k0);
    return;
  }
  if (!leader) c0 = c1 = 0;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    c0 += __shfl_xor_sync(0xffffffffu, c0, d);
    c1 += __shfl_xor_sync(0xffffffffu, c1, d);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(&R.cost[o][0], c0);
    atomicAdd(&R.cost[o][1], c1);
  }
}

// The exact partitioned-Rice cost of the residuals of one candidate.  Every thread calls it.  Without kPlan thread 0
// returns the residual section's bits (method, order and parameters included) and sets (porder, method); with kPlan the
// parameters of (plan_o, plan_m) land in R.kp.  u(i) gives the folded residual of sample i >= p.
template <bool kPlan, class U>
__device__ long long rice(int n, int p, U u, RiceSmem& R, int plan_o, int plan_m, int* porder, int* method) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int omax = max_porder(n, p);
  if (!kPlan) {
    if (tid < 18) R.cost[tid >> 1][tid & 1] = 0;
    __syncthreads();
  }
  // a thread owns at most 16 samples and u < 2^32, so the sums of u >> k for k >= 4 fit in 32 bits
  constexpr int kWide = 4;
  unsigned long long S[kNK + 1];
  unsigned S32[kNK];
#pragma unroll
  for (int k = 0; k <= kNK; ++k) S[k] = 0;
#pragma unroll
  for (int k = kWide; k < kNK; ++k) S32[k] = 0;
  const int lo = (tid * n) >> kLogT, hi = ((tid + 1) * n) >> kLogT;
  for (int i = max(lo, p); i < hi; ++i) {
    const unsigned v = u(i);
#pragma unroll
    for (int k = 0; k < kWide; ++k) S[k] += v >> k;
#pragma unroll
    for (int k = kWide; k < kNK; ++k) S32[k] += v >> k;
    S[kNK] += 1;
  }
#pragma unroll
  for (int k = kWide; k < kNK; ++k) S[k] = S32[k];
  level<kPlan>(S, 0, tid, true, omax, plan_o, plan_m, R);
#pragma unroll
  for (int l = 1; l <= 5; ++l) {
#pragma unroll
    for (int k = 0; k <= kNK; ++k) S[k] += __shfl_xor_sync(0xffffffffu, S[k], 1 << (l - 1));
    level<kPlan>(S, l, tid >> l, (tid & ((1 << l) - 1)) == 0, omax, plan_o, plan_m, R);
  }
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k <= kNK; ++k) R.wsum[warp][k] = S[k];
  }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int k = 0; k <= kNK; ++k) S[k] = lane < kT / 32 ? R.wsum[lane][k] : 0ull;
#pragma unroll
    for (int l = 6; l <= kLogT; ++l) {
#pragma unroll
      for (int k = 0; k <= kNK; ++k) S[k] += __shfl_xor_sync(0xffffffffu, S[k], 1 << (l - 6));
      level<kPlan>(S, l, lane >> (l - 5), lane < kT / 32 && (lane & ((1 << (l - 5)) - 1)) == 0, omax, plan_o, plan_m, R);
    }
  }
  __syncthreads();
  long long best = -1;
  if (!kPlan && tid == 0) {
    for (int o = 0; o <= omax; ++o) {
      const unsigned long long t0 = R.cost[o][0] + (4ull << o), t1 = R.cost[o][1] + (5ull << o);
      const long long t = (long long)(t0 <= t1 ? t0 : t1);
      if (best < 0 || t < best) {
        best = t;
        *porder = o;
        *method = t0 <= t1 ? 0 : 1;
      }
    }
    best += 6;
  }
  __syncthreads();  // R is reused by the next candidate
  return best;
}

struct AnaSmem {
  int s[kBlock];
  unsigned long long R[kMaxLpc + 1];
  short q[kMaxLpc][kMaxLpc];
  int shift[kMaxLpc];
  int nlpc;  // orders 1 .. nlpc came out of the recursion; shift[p - 1] < 0 marks a skipped order
  RiceSmem rice;
};

// Levinson-Durbin and the quantisation at precision 12, one IEEE rounding per operation (no FMA contraction)
__device__ void lpc_orders(AnaSmem& sm) {
  double R[kMaxLpc + 1], a[kMaxLpc], na[kMaxLpc];
  for (int l = 0; l <= kMaxLpc; ++l) R[l] = (double)(long long)sm.R[l];
  double err = R[0];
  int np = 0;
  for (int p = 1; p <= kMaxLpc; ++p) {
    if (!(err > 0.0 && isfinite(err))) break;
    double acc = R[p];
    for (int j = 0; j < p - 1; ++j) acc = __dsub_rn(acc, __dmul_rn(a[j], R[p - 1 - j]));
    const double k = __ddiv_rn(acc, err);
    bool fin = isfinite(k);
    for (int j = 0; j < p - 1; ++j) {
      na[j] = __dsub_rn(a[j], __dmul_rn(k, a[p - 2 - j]));
      fin = fin && isfinite(na[j]);
    }
    na[p - 1] = k;
    if (!fin) break;
    for (int j = 0; j < p; ++j) a[j] = na[j];
    np = p;
    // quantise this order
    double cmax = 0.0;
    for (int j = 0; j < p; ++j) cmax = fmax(cmax, fabs(a[j]));
    int e = 0;
    frexp(cmax, &e);
    const int shift = min(kPrec - 1 - e, 15);
    if (cmax == 0.0 || shift < 0) {
      sm.shift[p - 1] = -1;
    } else {
      sm.shift[p - 1] = shift;
      const double scale = ldexp(1.0, shift);
      double qe = 0.0;
      for (int j = 0; j < p; ++j) {
        qe = __dadd_rn(qe, __dmul_rn(a[j], scale));
        const int qi = (int)fmin(fmax(round(qe), -2048.0), 2047.0);
        sm.q[p - 1][j] = (short)qi;
        qe = __dsub_rn(qe, (double)qi);
      }
    }
    const double t = __dsub_rn(1.0, __dmul_rn(k, k));
    err = __dmul_rn(err, t);
  }
  sm.nlpc = np;
}

__global__ void __launch_bounds__(kT) flac_analysis_kernel(Job J, Rows Rw, Desc* __restrict__ desc) {
  __shared__ AnaSmem sm;
  const int tid = threadIdx.x;
  int row, n;
  long long first, number;
  block_geo(J, Rw, blockIdx.x, row, first, n, number);
  load_block(J.src, row, first, n, sm.s);
  if (tid <= kMaxLpc) sm.R[tid] = 0;
  __syncthreads();
  const int lo = (tid * n) >> kLogT, hi = ((tid + 1) * n) >> kLogT;
  bool eq = true;
  for (int i = lo; i < hi; ++i) eq = eq && sm.s[i] == sm.s[0];
  const bool constant = __syncthreads_and(eq);
  for (int l = 0; l <= kMaxLpc; ++l) {
    long long acc = 0;
    for (int i = max(lo, l); i < hi; ++i) acc += (long long)sm.s[i] * sm.s[i - l];
    if (acc) atomicAdd(&sm.R[l], (unsigned long long)acc);
  }
  __syncthreads();
  if (tid == 0) {
    sm.nlpc = 0;
    if (sm.R[0] != 0) lpc_orders(sm);
  }
  __syncthreads();
  long long best = constant ? 8 + 16 : -1;
  int bkind = kConst, border = 0, bporder = 0, bmethod = 0, bshift = 0;
  int porder = 0, method = 0;
  for (int p = 0; p <= kMaxFixed && p <= n; ++p) {
    const int* s = sm.s;
    const long long r = rice<false>(n, p, [&](int i) { return zig(residual(s, i, kFixed, p, nullptr, 0)); }, sm.rice, 0, 0,
                                    &porder, &method);
    if (tid == 0) {
      const long long bits = 8 + 16LL * p + r;
      if (best < 0 || bits < best) {
        best = bits;
        bkind = kFixed;
        border = p;
        bporder = porder;
        bmethod = method;
      }
    }
  }
  const int nlpc = sm.nlpc;
  for (int p = 1; p <= nlpc && p <= n; ++p) {
    const int shift = sm.shift[p - 1];
    if (shift < 0) continue;
    const int* s = sm.s;
    const short* q = sm.q[p - 1];
    const long long r = rice<false>(n, p, [&](int i) { return zig(residual(s, i, kLpc, p, q, shift)); }, sm.rice, 0, 0,
                                    &porder, &method);
    if (tid == 0) {
      const long long bits = 8 + 16LL * p + 4 + 5 + (long long)kPrec * p + r;
      if (bits < best) {
        best = bits;
        bkind = kLpc;
        border = p;
        bporder = porder;
        bmethod = method;
        bshift = shift;
      }
    }
  }
  if (tid == 0) {
    if (8 + 16LL * n < best) {
      best = 8 + 16LL * n;
      bkind = kVerbatim;
    }
    Desc d{};
    d.kind = bkind;
    d.order = border;
    d.shift = bshift;
    d.porder = bporder;
    d.method = bmethod;
    d.hdr = header_bytes(n, number);
    d.bytes = d.hdr + (int)((best + 7) / 8) + 2;
    if (bkind == kLpc)
      for (int j = 0; j < border; ++j) d.q[j] = sm.q[border - 1][j];
    desc[blockIdx.x] = d;
  }
}

// inclusive scan of v over the CTA (blockDim.x a multiple of 32, at most 1024); returns the CTA total
__device__ __forceinline__ long long cta_scan(long long& v, long long* wtot) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const long long o = __shfl_up_sync(0xffffffffu, v, d);
    if (lane >= d) v += o;
  }
  if (lane == 31) wtot[warp] = v;
  __syncthreads();
  if (warp == 0) {
    long long w = lane < nw ? wtot[lane] : 0;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const long long o = __shfl_up_sync(0xffffffffu, w, d);
      if (lane >= d) w += o;
    }
    if (lane < nw) wtot[lane] = w;
  }
  __syncthreads();
  if (warp > 0) v += wtot[warp - 1];
  const long long total = wtot[nw - 1];
  __syncthreads();
  return total;
}

__device__ __forceinline__ void put_be(unsigned char* p, unsigned long long v, int nbytes) {
  for (int i = 0; i < nbytes; ++i) p[i] = (unsigned char)(v >> (8 * (nbytes - 1 - i)));
}

constexpr int kLayT = 1024;

// One CTA: items are, per row, its STREAMINFO (42 bytes when J.header, else 0) then its frames.  An exclusive scan of the
// item sizes from *cursor gives every frame's offset and every row's offset and size; the row's min / max frame sizes
// and its STREAMINFO follow.  *cursor advances past this launch's rows.
__global__ void __launch_bounds__(kLayT) flac_layout_kernel(Job J, Rows Rw, const Desc* __restrict__ desc, long long* __restrict__ foff,
                                                            long long* __restrict__ cursor, unsigned char* __restrict__ out,
                                                            long long* __restrict__ row_off, long long* __restrict__ row_bytes) {
  __shared__ long long wtot[32];
  __shared__ long long rstart[kRowsPerLaunch + 1];
  __shared__ unsigned fmin_[kRowsPerLaunch], fmax_[kRowsPerLaunch];
  const int tid = threadIdx.x, rows = J.rows;
  const long long nblk = Rw.blk0[rows], nitems = nblk + rows, base = *cursor;
  for (int r = tid; r < rows; r += kLayT) {
    fmin_[r] = 0xffffffffu;
    fmax_[r] = 0;
  }
  __syncthreads();
  long long run = base;
  for (long long c0 = 0; c0 < nitems; c0 += kLayT) {
    const long long it = c0 + tid;
    long long v = 0, b = -1;
    int r = -1;
    if (it < nitems) {
      // row r holds items [blk0[r] + r, blk0[r + 1] + r + 1)
      int lo = 0, hi = rows - 1;
      while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (Rw.blk0[mid] + mid <= it) lo = mid;
        else hi = mid - 1;
      }
      r = lo;
      if (it == Rw.blk0[r] + r) {
        v = J.header ? kInfoBytes : 0;
      } else {
        b = it - r - 1;
        v = desc[b].bytes;
        atomicMin(&fmin_[r], (unsigned)v);
        atomicMax(&fmax_[r], (unsigned)v);
      }
    }
    const long long mine = v;
    const long long total = cta_scan(v, wtot);
    const long long off = run + v - mine;  // exclusive
    if (b >= 0) foff[b] = off;
    else if (r >= 0) rstart[r] = off;
    run += total;
    __syncthreads();
  }
  if (tid == 0) rstart[rows] = run;
  __syncthreads();
  for (int r = tid; r < rows; r += kLayT) {
    const long long o = rstart[r], sz = rstart[r + 1] - o;
    row_off[r] = o;
    row_bytes[r] = sz;
    if (J.header) {
      unsigned char* h = out + o;
      const bool any = Rw.len[r] > 0;
      h[0] = 'f';
      h[1] = 'L';
      h[2] = 'a';
      h[3] = 'C';
      h[4] = 0x80;
      put_be(h + 5, 34, 3);
      put_be(h + 8, kBlock, 2);
      put_be(h + 10, kBlock, 2);
      put_be(h + 12, any ? fmin_[r] : 0, 3);
      put_be(h + 15, any ? fmax_[r] : 0, 3);
      const unsigned long long v = ((unsigned long long)J.sr << 44) | (15ull << 36) | (unsigned long long)Rw.len[r];
      put_be(h + 18, v, 8);
      for (int i = 26; i < kInfoBytes; ++i) h[i] = 0;
    }
  }
  if (tid == 0) *cursor = run;
}

struct PackSmem {
  int s[kBlock];
  unsigned u[kBlock];
  unsigned w[kWords];
  unsigned short tab[256];
  unsigned crc[kT];
  long long wtot[32];
  unsigned char hdr[kMaxHdr];
  RiceSmem rice;
};

// OR the low `width` (<= 32) bits of v into the big-endian bit stream at bit position pos
__device__ __forceinline__ void put_bits(unsigned* w, long long pos, unsigned v, int width) {
  if (width == 0) return;
  if (width < 32) v &= (1u << width) - 1u;
  const int wi = (int)(pos >> 5), off = (int)(pos & 31);
  if (off + width <= 32) {
    atomicOr(&w[wi], v << (32 - off - width));
  } else {
    const int hi_bits = 32 - off, lo_bits = width - hi_bits;
    atomicOr(&w[wi], v >> lo_bits);
    atomicOr(&w[wi + 1], v << (32 - lo_bits));
  }
}

__device__ __forceinline__ unsigned get_byte(const unsigned* w, int j) { return (w[j >> 2] >> (24 - 8 * (j & 3))) & 0xFFu; }

__device__ unsigned crc8_bytes(const unsigned char* p, int n) {
  unsigned c = 0;
  for (int i = 0; i < n; ++i) {
    c ^= p[i];
    for (int b = 0; b < 8; ++b) c = (c & 0x80) ? ((c << 1) ^ 0x07) & 0xFF : (c << 1) & 0xFF;
  }
  return c;
}

// a * b mod x^16 + x^15 + x^2 + 1 over GF(2)
__device__ __forceinline__ unsigned gf16_mul(unsigned a, unsigned b) {
  unsigned r = 0;
  for (int i = 15; i >= 0; --i)
    if (b >> i & 1) r ^= a << i;
  for (int i = 30; i >= 16; --i)
    if (r >> i & 1) r ^= 0x18005u << (i - 16);
  return r;
}

// x^(8 nbytes) mod the CRC-16 polynomial: multiplying a CRC by it appends nbytes zero bytes
__device__ unsigned gf16_xpow_bytes(long long nbytes) {
  unsigned r = 1, b = 1u << 8;  // x^8
  while (nbytes) {
    if (nbytes & 1) r = gf16_mul(r, b);
    b = gf16_mul(b, b);
    nbytes >>= 1;
  }
  return r;
}

__global__ void __launch_bounds__(kT) flac_pack_kernel(Job J, Rows Rw, const Desc* __restrict__ desc, const long long* __restrict__ foff,
                                                       unsigned char* __restrict__ out) {
  __shared__ PackSmem sm;
  const int tid = threadIdx.x;
  int row, n;
  long long first, number;
  block_geo(J, Rw, blockIdx.x, row, first, n, number);
  const Desc d = desc[blockIdx.x];
  load_block(J.src, row, first, n, sm.s);
  for (int i = tid; i < kWords; i += kT) sm.w[i] = 0;
  {
    unsigned c = (unsigned)tid << 8;
    for (int b = 0; b < 8; ++b) c = (c & 0x8000) ? ((c << 1) ^ 0x8005) & 0xFFFF : (c << 1) & 0xFFFF;
    sm.tab[tid] = (unsigned short)c;
  }
  if (tid == 0) {
    unsigned char* h = sm.hdr;
    int k = 0;
    h[k++] = 0xFF;
    h[k++] = J.variable ? 0xF9 : 0xF8;
    const int bcode = n == kBlock ? 0xC : n <= 256 ? 0x6 : 0x7;
    h[k++] = (unsigned char)(bcode << 4 | J.sr_code);
    h[k++] = 0x08;
    const int nb = utf8_len(number);
    if (nb == 1) {
      h[k++] = (unsigned char)number;
    } else {
      h[k++] = (unsigned char)(((0xFF00 >> nb) & 0xFF) | (number >> (6 * (nb - 1))));
      for (int i = nb - 2; i >= 0; --i) h[k++] = (unsigned char)(0x80 | ((number >> (6 * i)) & 0x3F));
    }
    if (bcode == 0x6) h[k++] = (unsigned char)(n - 1);
    if (bcode == 0x7) {
      h[k++] = (unsigned char)((n - 1) >> 8);
      h[k++] = (unsigned char)(n - 1);
    }
    h[k] = (unsigned char)crc8_bytes(h, k);
  }
  __syncthreads();
  if (tid < d.hdr) put_bits(sm.w, 8LL * tid, sm.hdr[tid], 8);
  const long long sub = 8LL * d.hdr;  // the subframe's first bit
  const int p = d.order;
  if (tid == 0) {
    const int type = d.kind == kConst ? 0 : d.kind == kVerbatim ? 1 : d.kind == kFixed ? 8 + p : 32 + p - 1;
    put_bits(sm.w, sub, (unsigned)type << 1, 8);
    if (d.kind == kConst) put_bits(sm.w, sub + 8, (unsigned)sm.s[0], 16);
  }
  if (d.kind == kVerbatim) {
    for (int i = tid; i < n; i += kT) put_bits(sm.w, sub + 8 + 16LL * i, (unsigned)sm.s[i], 16);
  } else if (d.kind != kConst) {
    if (tid < p) put_bits(sm.w, sub + 8 + 16LL * tid, (unsigned)sm.s[tid], 16);
    long long res = sub + 8 + 16LL * p;
    if (d.kind == kLpc) {
      if (tid == 0) {
        put_bits(sm.w, res, kPrec - 1, 4);
        put_bits(sm.w, res + 4, (unsigned)d.shift, 5);
      }
      if (tid < p) put_bits(sm.w, res + 9 + (long long)kPrec * tid, (unsigned)d.q[tid], kPrec);
      res += 9 + (long long)kPrec * p;
    }
    if (tid == 0) {
      put_bits(sm.w, res, (unsigned)d.method, 2);
      put_bits(sm.w, res + 2, (unsigned)d.porder, 4);
    }
    res += 6;
    for (int i = p + tid; i < n; i += kT) sm.u[i] = zig(residual(sm.s, i, d.kind, p, d.q, d.shift));
    __syncthreads();
    const unsigned* u = sm.u;
    rice<true>(n, p, [&](int i) { return u[i]; }, sm.rice, d.porder, d.method, nullptr, nullptr);
    // thread t's samples lie in partition t >> (8 - porder); the group's first thread also writes the parameter
    const int part = tid >> (kLogT - d.porder), pbits = d.method ? 5 : 4;
    const bool first_of_part = (tid & ((1 << (kLogT - d.porder)) - 1)) == 0;
    const int k = sm.rice.kp[part];
    const int lo = (tid * n) >> kLogT, hi = ((tid + 1) * n) >> kLogT;
    long long len = first_of_part ? pbits : 0;
    for (int i = max(lo, p); i < hi; ++i) len += (long long)(u[i] >> k) + 1 + k;
    long long v = len;
    cta_scan(v, sm.wtot);
    long long pos = res + v - len;
    if (first_of_part) {
      put_bits(sm.w, pos, (unsigned)k, pbits);
      pos += pbits;
    }
    for (int i = max(lo, p); i < hi; ++i) {
      const long long q = u[i] >> k;
      put_bits(sm.w, pos + q, (1u << k) | (u[i] & ((1u << k) - 1u)), k + 1);
      pos += q + 1 + k;
    }
  }
  __syncthreads();
  // CRC-16 over the frame's first L bytes (header, subframe, zero pad): per-thread chunks, combined in order
  const int L = d.bytes - 2, C = (L + kT - 1) / kT;
  {
    unsigned c = 0;
    const int b0 = min(L, tid * C), b1 = min(L, b0 + C);
    for (int j = b0; j < b1; ++j) c = ((c << 8) & 0xFFFF) ^ sm.tab[((c >> 8) ^ get_byte(sm.w, j)) & 0xFF];
    sm.crc[tid] = c;
  }
  __syncthreads();
  if (tid == 0) {
    const unsigned xc = gf16_xpow_bytes(C);
    unsigned acc = 0;
    for (int t = 0; t < kT; ++t) {
      const int b0 = min(L, t * C), len = min(L, b0 + C) - b0;
      if (len == 0) break;
      acc = gf16_mul(acc, len == C ? xc : gf16_xpow_bytes(len)) ^ sm.crc[t];
    }
    put_bits(sm.w, 8LL * L, acc, 16);
  }
  __syncthreads();
  unsigned char* o = out + foff[blockIdx.x];
  for (int j = tid; j < d.bytes; j += kT) o[j] = (unsigned char)get_byte(sm.w, j);
}

__global__ void flac_zero_kernel(long long* p) { *p = 0; }

// workspace: the descriptors, the frame offsets and the cursor of one launch's blocks
struct Layout {
  size_t desc = 0, foff = 0, cursor = 0, roff = 0, total = 0;
};

Layout layout(int B, long long max_len) {
  const long long nb = (long long)std::min(B, kRowsPerLaunch) * blocks_of(max_len);
  Layout l;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    const size_t o = off;
    off += (bytes + 255) & ~(size_t)255;
    return o;
  };
  l.desc = take(nb * sizeof(Desc));
  l.foff = take(nb * sizeof(long long));
  l.cursor = take(sizeof(long long));
  l.roff = take((size_t)B * sizeof(long long));
  l.total = off;
  return l;
}

long long out_bound(long long n, bool header) {
  return (header ? kInfoBytes : 0) + blocks_of(n) * (kMaxHdr + 1 + 2) + 2 * n;
}

// rows [0, B) of the job in launches of 128 rows, row b lens[b] samples long (x_stride each when lens is null); row b's
// bytes land at out + row_off[b], its size in row_bytes[b]
int run(Job J, int B, const int64_t* lens, long long x_stride, char* ws, const Layout& l, unsigned char* out, long long* row_off,
        long long* row_bytes, cudaStream_t st) {
  Desc* desc = reinterpret_cast<Desc*>(ws + l.desc);
  long long* foff = reinterpret_cast<long long*>(ws + l.foff);
  long long* cursor = reinterpret_cast<long long*>(ws + l.cursor);
  flac_zero_kernel<<<1, 1, 0, st>>>(cursor);
  CK(cudaGetLastError());
  const Src src0 = J.src;
  for (int b0 = 0; b0 < B; b0 += kRowsPerLaunch) {
    const int rows = std::min(kRowsPerLaunch, B - b0);
    const RowLens<kRowsPerLaunch> L = row_lens<kRowsPerLaunch>(lens, x_stride, b0, rows);
    Rows R{};
    R.blk0[0] = 0;
    for (int i = 0; i < rows; ++i) {
      R.len[i] = L.v[i];
      R.blk0[i + 1] = R.blk0[i] + blocks_of(R.len[i]);
    }
    J.rows = rows;
    J.src.x = src0.x ? src0.x + (long long)b0 * src0.x_stride : nullptr;
    const long long nblk = R.blk0[rows];
    if (nblk > 0) {
      flac_analysis_kernel<<<(unsigned)nblk, kT, 0, st>>>(J, R, desc);
      CK(cudaGetLastError());
    }
    flac_layout_kernel<<<1, kLayT, 0, st>>>(J, R, desc, foff, cursor, out, row_off + b0, row_bytes + b0);
    CK(cudaGetLastError());
    if (nblk > 0) {
      flac_pack_kernel<<<(unsigned)nblk, kT, 0, st>>>(J, R, desc, foff, out);
      CK(cudaGetLastError());
    }
  }
  return SOPRO_OK;
}

}  // namespace

// the tail holds the carried samples [samples, samples + carried), samples emitted in frames so far being the next
// frame's number
struct SoproFlacStream {
  int sr = 0;
  chunk::Tail tail;
};

extern "C" {

int sopro_flac_sizes(int32_t B, int64_t max_len, int32_t sr, int64_t* ws_bytes, int64_t* out_bytes) {
  if (!valid_rate(sr)) return fail(SOPRO_ERR_INVALID, "sample rate %d not in [%d, %d]", sr, kMinRate, kMaxRate);
  if (B < 1 || max_len < 0 || max_len > kMaxLen)
    return fail(SOPRO_ERR_INVALID, "bad geometry: %d rows of at most %lld samples (at most %lld)", B, (long long)max_len, kMaxLen);
  if (ws_bytes) *ws_bytes = (int64_t)layout(B, max_len).total;
  if (out_bytes) *out_bytes = (int64_t)B * out_bound(max_len, true);
  return SOPRO_OK;
}

int sopro_flac_encode(const float* x, int32_t B, int64_t x_stride, const int64_t* lens_host, int32_t sr, void* ws,
                      uint8_t* out, int64_t* row_off, int64_t* row_bytes, void* stream) {
  if (!valid_rate(sr)) return fail(SOPRO_ERR_INVALID, "sample rate %d not in [%d, %d]", sr, kMinRate, kMaxRate);
  if (!ws || !out || !row_off || !row_bytes) return fail(SOPRO_ERR_INVALID, "null argument");
  long long most = 0;
  const int rc = check_rows(x, B, x_stride, lens_host, kMaxLen, &most);
  if (rc != SOPRO_OK) return rc;
  Job J{};
  J.src = Src{x, x_stride, nullptr, 0};
  J.variable = 0;
  J.num0 = 0;
  J.sr = sr;
  J.sr_code = rate_code(sr);
  J.header = 1;
  return run(J, B, lens_host, x_stride, static_cast<char*>(ws), layout(B, most), out, reinterpret_cast<long long*>(row_off),
             reinterpret_cast<long long*>(row_bytes), reinterpret_cast<cudaStream_t>(stream));
}

int sopro_flac_stream_create(int32_t sr, SoproFlacStream** out) {
  if (!out) return fail(SOPRO_ERR_INVALID, "null argument");
  *out = nullptr;
  if (!valid_rate(sr)) return fail(SOPRO_ERR_INVALID, "sample rate %d not in [%d, %d]", sr, kMinRate, kMaxRate);
  SoproFlacStream* s = new SoproFlacStream();
  s->sr = sr;
  const cudaError_t e = s->tail.alloc(kStreamMin);
  if (e != cudaSuccess) {
    sopro_flac_stream_destroy(s);
    return fail(SOPRO_ERR_CUDA, "flac stream state: %s", cudaGetErrorString(e));
  }
  *out = s;
  return SOPRO_OK;
}

int sopro_flac_stream_destroy(SoproFlacStream* s) {
  if (!s) return SOPRO_OK;
  s->tail.release();
  delete s;
  return SOPRO_OK;
}

int sopro_flac_stream_reset(SoproFlacStream* s, int32_t sr) {
  if (!s) return fail(SOPRO_ERR_INVALID, "null argument");
  if (!valid_rate(sr)) return fail(SOPRO_ERR_INVALID, "sample rate %d not in [%d, %d]", sr, kMinRate, kMaxRate);
  s->sr = sr;
  s->tail.restart(0);
  return SOPRO_OK;
}

int64_t sopro_flac_stream_carried(const SoproFlacStream* s) { return s ? s->tail.held() : -1; }

static int stream_encode(SoproFlacStream* s, const float* x, long long n, void* ws, uint8_t* out, int64_t* nbytes, bool last,
                         void* stream) {
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long total = s->tail.held() + n;
  long long keep = total % kBlock;
  if (last || keep >= kStreamMin) keep = 0;
  const long long enc = total - keep;
  char* w = static_cast<char*>(ws);
  const Layout l = layout(1, total);
  long long* roff = reinterpret_cast<long long*>(w + l.roff);
  Job J{};
  J.src = Src{x, 0, s->tail.data(), (int)s->tail.held()};
  J.variable = 1;
  J.num0 = s->tail.base;
  J.sr = s->sr;
  J.sr_code = rate_code(s->sr);
  J.header = 0;
  const int64_t lens[1] = {enc};
  const int rc = run(J, 1, lens, 0, w, l, out, roff, reinterpret_cast<long long*>(nbytes), st);
  return rc == SOPRO_OK ? s->tail.keep(s->tail.base + enc, x, n, st) : rc;
}

int sopro_flac_stream_push(SoproFlacStream* s, const float* x, int64_t n, void* ws, uint8_t* out, int64_t* nbytes, void* stream) {
  if (!s || !ws || !out || !nbytes || (!x && n > 0)) return fail(SOPRO_ERR_INVALID, "null argument");
  if (n < 0 || n > kMaxLen - s->tail.seen) return fail(SOPRO_ERR_INVALID, "push of %lld samples refused", (long long)n);
  return stream_encode(s, x, n, ws, out, nbytes, false, stream);
}

int sopro_flac_stream_finish(SoproFlacStream* s, void* ws, uint8_t* out, int64_t* nbytes, void* stream) {
  if (!s || !ws || !out || !nbytes) return fail(SOPRO_ERR_INVALID, "null argument");
  const int rc = stream_encode(s, nullptr, 0, ws, out, nbytes, true, stream);
  if (rc != SOPRO_OK) return rc;
  s->tail.restart(0);
  return SOPRO_OK;
}

}  // extern "C"
