// Word alignment: the monotonic token -> frame path through the AR step's text cross-attention weights.
// The definition (include/sopro_b200.h, oracle/align_oracle.py in float64), per utterance of L tokens and T frames:
//   A[t][l] = sum over the attention layers s ascending, then the heads h ascending, of (double) probs[t][s][b][h][l];
//   S[0][0] = A[0][0], S[0][l > 0] = -inf; S[t][l] = A[t][l] + max(S[t-1][l], S[t-1][l-1]), the stay predecessor winning
//   ties; backtrack from (T-1, L-1).  IEEE double additions and comparisons only, so the float64 restatement in the same
//   order finds the same path.
//
// align_kernel: one CTA per utterance.  The weights of TS steps are summed into a shared tile A[TS][Lp] with every load
// independent (one thread per (step, token)), then the DP walks those TS steps over S, double-buffered in shared memory,
// one thread per token and a CTA barrier per step.  Each step's back-pointer bits (1 = the path came from l - 1) are one
// ballot per warp, stored to the workspace.  The backtrack runs on one warp: per 32 steps every lane loads the two words
// its step's bit can be in (the path moves at most one token per step), then the walk reads them through shuffles.
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>
#include <vector>

#include "../../include/sopro_b200.h"
#include "common.cuh"

namespace {

constexpr int kMaxL = 2048;              // tokens of one utterance (the S buffers: 2 x 16 KB)
constexpr int kThreads = 512;
constexpr int kRowsPerLaunch = 128;      // utterances of one launch (their lengths travel as a kernel parameter)
constexpr int kTileBytes = 128 * 1024;   // the A tile
constexpr int kMaxTile = 64;             // steps of one A tile

struct AlignRows {
  int len[kRowsPerLaunch];
  int frames[kRowsPerLaunch];
};

// back-pointer words per step
inline int words_per_step(long long ld) { return (int)((std::min<long long>(ld, kMaxL) + 31) / 32); }
// tokens padded to whole warps, and the steps of one A tile
__host__ __device__ inline int padded(int L) { return (L + 31) & ~31; }
__host__ __device__ inline int tile_steps(int Lp) { return max(1, min(kMaxTile, kTileBytes / (Lp * 8))); }

// The weights of nt steps summed into the tile At[nt][Lp], every load independent (one thread per (step, token));
// step_ptr(tt) is the trace of the tile's step tt at utterance b, token 0.
template <class StepPtr>
__device__ __forceinline__ void load_tile(double* At, int Lp, int nt, int L, int n_attn, int H, long long ld, size_t s_stride,
                                          StepPtr step_ptr) {
  for (int i = threadIdx.x; i < nt * L; i += kThreads) {
    const int tt = i / L, l = i - tt * L;
    const float* src = step_ptr(tt) + l;
    double a = 0.0;
#pragma unroll 1
    for (int s = 0; s < n_attn; ++s) {
#pragma unroll 4
      for (int h = 0; h < H; ++h) a += (double)__ldg(src + s * s_stride + (size_t)h * ld);
    }
    At[(size_t)tt * Lp + l] = a;
  }
}

// One DP step: Sn = S[t] from Sp = S[t-1] and a = A[t]; for t > 0 the step's move bits go to bw[Lp / 32], one ballot
// per warp.  Whole warps: Lp is a multiple of 32.
__device__ __forceinline__ void dp_step(int t, const double* Sp, double* Sn, const double* a, int L, int Lp, unsigned* bw) {
  const int lane = threadIdx.x & 31;
  for (int l = threadIdx.x; l < Lp; l += kThreads) {
    bool mv = false;
    if (l < L) {
      if (t == 0) {
        Sn[l] = l == 0 ? a[l] : -INFINITY;
      } else {
        const double stay = Sp[l], move = l > 0 ? Sp[l - 1] : -INFINITY;
        mv = move > stay;
        Sn[l] = a[l] + (mv ? move : stay);
      }
    }
    const unsigned word = __ballot_sync(0xffffffffu, mv);
    if (lane == 0 && t > 0) bw[l >> 5] = word;
  }
}

// The backtrack on one warp (t, l and the word index are warp-uniform): from (t, l) down to step t_stop + 1, writing
// out[l] = the step at which the path moved onto token l; -> the token at step t_stop.  bits_of(τ) is step τ's move
// words.  Per 32 steps every lane loads the two words its step's bit can be in (the path moves at most one token per
// step), then the walk reads them through shuffles.
template <class BitsOf>
__device__ __forceinline__ int warp_backtrack(BitsOf bits_of, int t, int t_stop, int l, int* out) {
  const int lane = threadIdx.x & 31;
#pragma unroll 1
  while (t > t_stop) {
    const int w = l >> 5;
    const int tr = t - lane;
    unsigned hi = 0u, lo = 0u;
    if (tr > t_stop) {
      hi = __ldcg(bits_of(tr) + w);
      if (w > 0) lo = __ldcg(bits_of(tr) + w - 1);
    }
    const int n = min(32, t - t_stop);
#pragma unroll 1
    for (int j = 0; j < n; ++j) {
      const unsigned h = __shfl_sync(0xffffffffu, hi, j), lw = __shfl_sync(0xffffffffu, lo, j);
      const unsigned word = (l >> 5) == w ? h : lw;  // l >= (the l this round began with) - 31
      if (l > 0 && ((word >> (l & 31)) & 1u)) {
        if (lane == 0) out[l] = t;  // token l starts at frame t
        --l;
      }
      --t;
    }
  }
  return l;
}

__global__ void __launch_bounds__(kThreads) align_kernel(const float* __restrict__ probs, int steps, int n_attn, int B, int H,
                                                         long long ld, const __grid_constant__ AlignRows rows, int b0,
                                                         unsigned* __restrict__ bits, int W, int* __restrict__ first) {
  extern __shared__ __align__(16) double sm[];
  __shared__ int s_ok;
  const int b = b0 + blockIdx.x;
  const int L = rows.len[blockIdx.x], T = rows.frames[blockIdx.x];
  const int tid = threadIdx.x, warp = tid >> 5;
  int* out = first + (size_t)b * ld;
  if (T < L || T == 0) {  // no path
    for (long long l = tid; l < ld; l += kThreads) out[l] = -1;
    return;
  }
  const int Lp = padded(L), TS = tile_steps(Lp);
  double* S0 = sm;  // S of the even steps
  double* S1 = sm + Lp;
  double* At = sm + 2 * Lp;  // [TS][Lp]
  unsigned* bb = bits + (size_t)b * steps * W;
  const size_t s_stride = (size_t)B * H * ld, t_stride = (size_t)n_attn * s_stride;
  const float* pb = probs + (size_t)b * H * ld;
#pragma unroll 1
  for (int t0 = 0; t0 < T; t0 += TS) {
    const int nt = min(TS, T - t0);
    load_tile(At, Lp, nt, L, n_attn, H, ld, s_stride, [&](int tt) { return pb + (size_t)(t0 + tt) * t_stride; });
    __syncthreads();
#pragma unroll 1
    for (int tt = 0; tt < nt; ++tt) {
      const int t = t0 + tt;
      // S[t-1] -> S[t]
      dp_step(t, (t & 1) ? S0 : S1, (t & 1) ? S1 : S0, At + (size_t)tt * Lp, L, Lp, bb + (size_t)t * W);
      __syncthreads();  // S[t] complete, and the A tile free after its last step
    }
  }
  if (warp == 0) {
    const int l = warp_backtrack([&](int tr) { return bb + (size_t)tr * W; }, T - 1, 0, L - 1, out);
    if (tid == 0) s_ok = l == 0;
  }
  __syncthreads();
  const bool ok = s_ok != 0;
  for (long long l = tid; l < ld; l += kThreads) {
    if (!ok || l >= L) out[l] = -1;
    else if (l == 0) out[0] = 0;
  }
}

// ---- the streaming alignment (fixed-lag Viterbi with binding commits; include/sopro_b200.h)

constexpr int kStreamRows = 256;  // rows of one stream state (their push counts travel as a kernel parameter)

struct StreamRows {
  int len[kStreamRows];    // L
  int t0[kStreamRows];     // frames pushed before this push
  int n[kStreamRows];      // new frames; bit 30: the row ends after them
};
constexpr int kEndFlag = 1 << 30;

// per-row device state, rows after rows: out [rows][2 + ld] i32 ({committed frames F, committed tokens K, first[ld]}),
// then S [rows][Lpm] f64, then the move bits of the last R steps [rows][R][Wm] u32 (step τ in slot τ % R)
struct StreamGeom {
  long long ld;
  int Lpm, Wm, R, lag;
  size_t s_off, bits_off, bytes;
};

inline StreamGeom stream_geom(int rows, long long ld, int lag, int max_frames) {
  StreamGeom g{};
  g.ld = ld;
  g.Lpm = padded((int)std::min<long long>(ld, kMaxL));
  g.Wm = g.Lpm / 32;
  g.R = std::min(lag, max_frames);
  g.lag = lag;
  const size_t out = ((size_t)rows * (2 + ld) * 4 + 255) / 256 * 256;
  g.s_off = out;
  g.bits_off = g.s_off + (size_t)rows * g.Lpm * 8;
  g.bytes = g.bits_off + (size_t)rows * g.R * g.Wm * 4;
  return g;
}

__global__ void align_stream_reset_kernel(unsigned char* state, StreamGeom g, int rows) {
  const int b = blockIdx.x;
  int* out = reinterpret_cast<int*>(state) + (size_t)b * (2 + g.ld);
  for (long long i = threadIdx.x; i < 2 + g.ld; i += blockDim.x) out[i] = i < 2 ? 0 : -1;
}

// One CTA per row: the row's new frames through the DP, each step t >= lag followed by the commit of frame t - lag and
// the prune; at the row's end, the end backtrack.  S lives in shared memory for the push (loaded from and stored back
// to the row's state); the move bits of the last R steps stay in the state, read back through L1 by the ancestor walks.
__global__ void __launch_bounds__(kThreads) align_stream_kernel(const float* __restrict__ probs, int ring, int n_attn, int B,
                                                                int H, const __grid_constant__ StreamRows rows,
                                                                unsigned char* state, const StreamGeom g) {
  extern __shared__ __align__(16) double sm[];
  __shared__ double s_best[kThreads / 32];
  __shared__ int s_bl[kThreads / 32];
  __shared__ int s_kc;
  const int b = blockIdx.x;
  const int L = rows.len[b], t0 = rows.t0[b], n = rows.n[b] & ~kEndFlag;
  const bool end = (rows.n[b] & kEndFlag) != 0;
  if (n == 0 && !end) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long ld = g.ld;
  int* out = reinterpret_cast<int*>(state) + (size_t)b * (2 + ld);
  int* first = out + 2;
  double* Sg = reinterpret_cast<double*>(state + g.s_off) + (size_t)b * g.Lpm;
  unsigned* bits = reinterpret_cast<unsigned*>(state + g.bits_off) + (size_t)b * g.R * g.Wm;
  const int Lp = padded(L), W = g.Wm, R = g.R, D = g.lag;
  const int TS = tile_steps(Lp);
  auto Sb = [&](int t) { return sm + (t & 1) * Lp; };  // S of the even / odd frames
  int* anc = reinterpret_cast<int*>(sm + 2 * Lp);  // [Lp]: each state's token at the committed frame
  double* At = sm + 2 * Lp + Lp / 2;  // [TS][Lp]
  auto bits_of = [&](int tr) { return bits + (size_t)(tr % R) * W; };
  if (t0 > 0)
    for (int l = tid; l < L; l += kThreads) Sb(t0 - 1)[l] = Sg[l];
  int F = out[0], K = out[1];  // every thread reads them; thread 0 alone writes them, at the end
  const size_t s_stride = (size_t)B * H * ld, t_stride = (size_t)n_attn * s_stride;
  const float* pb = probs + (size_t)b * H * ld;
#pragma unroll 1
  for (int f0 = 0; f0 < n; f0 += TS) {
    const int nt = min(TS, n - f0);
    load_tile(At, Lp, nt, L, n_attn, H, ld, s_stride,
              [&](int tt) { return pb + (size_t)((t0 + f0 + tt) % ring) * t_stride; });
    __syncthreads();
#pragma unroll 1
    for (int tt = 0; tt < nt; ++tt) {
      const int t = t0 + f0 + tt;
      double* Sn = Sb(t);
      dp_step(t, Sb(t + 1), Sn, At + (size_t)tt * Lp, L, Lp, bits_of(t));
      __syncthreads();
      if (t >= D) {  // commit frame c = t - D, then prune
        const int c = t - D;
        // each finite state's token at frame c, and the lowest state of the largest finite S
        double bv = -INFINITY;
        int bl = INT_MAX;
        for (int l = tid; l < L; l += kThreads) {
          const double v = Sn[l];
          int k = -1;
          if (v > -INFINITY) {
            k = l;
#pragma unroll 1
            for (int tau = t; tau > c && k > 0; --tau) k -= (int)((bits_of(tau)[k >> 5] >> (k & 31)) & 1u);
            if (v > bv) bv = v, bl = l;  // l ascending: the first of equals stays
          }
          anc[l] = k;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const double ov = __shfl_down_sync(0xffffffffu, bv, o);
          const int ol = __shfl_down_sync(0xffffffffu, bl, o);
          if (ov > bv || (ov == bv && ol < bl)) bv = ov, bl = ol;
        }
        if (lane == 0) s_best[warp] = bv, s_bl[warp] = bl;
        __syncthreads();
        if (tid == 0) {
          bv = s_best[0], bl = s_bl[0];
          for (int i = 1; i < kThreads / 32; ++i)
            if (s_best[i] > bv || (s_best[i] == bv && s_bl[i] < bl)) bv = s_best[i], bl = s_bl[i];
          s_kc = bl == INT_MAX ? -1 : anc[bl];  // -1: no finite state, nothing to commit
        }
        __syncthreads();
        const int kc = s_kc;
        if (kc >= 0) {
          for (int l = tid; l < L; l += kThreads)
            if (anc[l] >= 0 && anc[l] != kc) Sn[l] = -INFINITY;
          if (tid == 0) {
            if (c == 0) first[0] = 0;
            else if (kc != K - 1) first[kc] = c;
          }
          F = c + 1;
          K = kc + 1;
        }
        __syncthreads();
      }
    }
  }
  const int T = t0 + n;
  if (end) {
    // the end state: (T-1, L-1) when finite, else the highest finite state
    const double* Sl = Sb(T - 1);
    int hi = -1;
    if (T > 0)
      for (int l = tid; l < L; l += kThreads)
        if (Sl[l] > -INFINITY) hi = l;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) hi = max(hi, __shfl_down_sync(0xffffffffu, hi, o));
    if (lane == 0) s_bl[warp] = hi;
    __syncthreads();
    if (tid == 0) {
      for (int i = 1; i < kThreads / 32; ++i) hi = max(hi, s_bl[i]);
      s_kc = hi;
    }
    __syncthreads();
    const int le = s_kc;
    if (le >= 0) {
      if (warp == 0) warp_backtrack(bits_of, T - 1, max(F - 1, 0), le, first);
      for (int l = tid; l < L; l += kThreads)
        if (l == 0) first[0] = 0;
        else if (l > le) first[l] = T;
    } else {  // no path (T == 0)
      for (int l = tid; l < L; l += kThreads) first[l] = -1;
    }
    if (tid == 0) {
      out[0] = le >= 0 ? T : 0;
      out[1] = le >= 0 ? L : 0;
    }
    return;
  }
  for (int l = tid; l < L; l += kThreads) Sg[l] = Sb(T - 1)[l];
  if (tid == 0) out[0] = F, out[1] = K;
}

}  // namespace

extern "C" {

int sopro_align_sizes(int32_t B, int32_t steps, int64_t ld, int64_t* ws_bytes) {
  if (!ws_bytes) return fail(SOPRO_ERR_INVALID, "align: null ws_bytes");
  *ws_bytes = 0;
  if (B < 1 || steps < 1 || ld < 1) return fail(SOPRO_ERR_INVALID, "align: B=%d, steps=%d, ld=%lld must be >= 1", B, steps, (long long)ld);
  *ws_bytes = (int64_t)B * steps * words_per_step(ld) * 4;
  return SOPRO_OK;
}

int sopro_align(const float* probs, int32_t steps, int32_t n_attn, int32_t B, int32_t H, int64_t ld, const int32_t* text_len_host,
                const int32_t* frames_host, void* ws, int32_t* first, void* stream) {
  if (!probs || !text_len_host || !frames_host || !ws || !first) return fail(SOPRO_ERR_INVALID, "align: null argument");
  if (B < 1 || steps < 1 || n_attn < 1 || H < 1 || ld < 1)
    return fail(SOPRO_ERR_INVALID, "align: B=%d, steps=%d, n_attn=%d, H=%d, ld=%lld must be >= 1", B, steps, n_attn, H, (long long)ld);
  if ((long long)n_attn * H > 4096) return fail(SOPRO_ERR_INVALID, "align: n_attn x H = %lld > 4096", (long long)n_attn * H);
  for (int b = 0; b < B; ++b) {
    if (text_len_host[b] < 1 || text_len_host[b] > std::min<int64_t>(ld, kMaxL))
      return fail(SOPRO_ERR_INVALID, "align: text_len[%d]=%d not in [1, min(ld=%lld, %d)]", b, text_len_host[b], (long long)ld, kMaxL);
    if (frames_host[b] < 0 || frames_host[b] > steps)
      return fail(SOPRO_ERR_INVALID, "align: frames[%d]=%d not in [0, %d]", b, frames_host[b], steps);
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int W = words_per_step(ld);
  for (int b0 = 0; b0 < B; b0 += kRowsPerLaunch) {
    const int nb = std::min(kRowsPerLaunch, B - b0);
    AlignRows rows{};
    int Lp = 32;
    for (int i = 0; i < nb; ++i) {
      rows.len[i] = text_len_host[b0 + i];
      rows.frames[i] = frames_host[b0 + i];
      Lp = std::max(Lp, padded(rows.len[i]));
    }
    // a CTA's own tile (tile_steps(own Lp) x own Lp) never exceeds this bound
    const size_t smem = (size_t)2 * Lp * 8 + std::min<size_t>((size_t)kMaxTile * Lp * 8, kTileBytes);
    CK(cudaFuncSetAttribute(align_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    align_kernel<<<nb, kThreads, smem, st>>>(probs, steps, n_attn, B, H, ld, rows, b0, static_cast<unsigned*>(ws), W, first);
    CK(cudaGetLastError());
  }
  return SOPRO_OK;
}

struct sopro_align_stream {
  int rows, max_frames;
  StreamGeom g;
  unsigned char* state;
  std::vector<int> len, t, ended;
};

static int stream_geometry_ok(int32_t rows, int64_t ld, int32_t lag, int32_t max_frames) {
  if (rows < 1 || rows > kStreamRows) return fail(SOPRO_ERR_INVALID, "align stream: rows=%d not in [1, %d]", rows, kStreamRows);
  if (ld < 1 || lag < 1 || max_frames < 1)
    return fail(SOPRO_ERR_INVALID, "align stream: ld=%lld, lag=%d, max_frames=%d must be >= 1", (long long)ld, lag, max_frames);
  return SOPRO_OK;
}

int sopro_align_stream_sizes(int32_t rows, int64_t ld, int32_t lag, int32_t max_frames, int64_t* state_bytes) {
  if (!state_bytes) return fail(SOPRO_ERR_INVALID, "align stream: null state_bytes");
  *state_bytes = 0;
  const int rc = stream_geometry_ok(rows, ld, lag, max_frames);
  if (rc != SOPRO_OK) return rc;
  *state_bytes = (int64_t)stream_geom(rows, ld, lag, max_frames).bytes;
  return SOPRO_OK;
}

int sopro_align_stream_create(int32_t rows, int64_t ld, int32_t lag, int32_t max_frames, void* state,
                              sopro_align_stream_t** out) {
  if (!out || !state) return fail(SOPRO_ERR_INVALID, "align stream: null argument");
  *out = nullptr;
  const int rc = stream_geometry_ok(rows, ld, lag, max_frames);
  if (rc != SOPRO_OK) return rc;
  auto* s = new sopro_align_stream;
  s->rows = rows;
  s->max_frames = max_frames;
  s->g = stream_geom(rows, ld, lag, max_frames);
  s->state = static_cast<unsigned char*>(state);
  s->len.assign(rows, 0);
  s->t.assign(rows, 0);
  s->ended.assign(rows, 1);
  *out = s;
  return SOPRO_OK;
}

int sopro_align_stream_destroy(sopro_align_stream_t* s) {
  delete s;
  return SOPRO_OK;
}

int sopro_align_stream_begin(sopro_align_stream_t* s, const int32_t* text_len_host, void* stream) {
  if (!s || !text_len_host) return fail(SOPRO_ERR_INVALID, "align stream: null argument");
  for (int b = 0; b < s->rows; ++b)
    if (text_len_host[b] < 1 || text_len_host[b] > std::min<int64_t>(s->g.ld, kMaxL))
      return fail(SOPRO_ERR_INVALID, "align stream: text_len[%d]=%d not in [1, min(ld=%lld, %d)]", b, text_len_host[b],
                  (long long)s->g.ld, kMaxL);
  align_stream_reset_kernel<<<s->rows, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(s->state, s->g, s->rows);
  CK(cudaGetLastError());
  for (int b = 0; b < s->rows; ++b) s->len[b] = text_len_host[b], s->t[b] = 0, s->ended[b] = 0;
  return SOPRO_OK;
}

int sopro_align_stream_push(sopro_align_stream_t* s, const float* probs, int32_t ring, int32_t n_attn, int32_t B, int32_t H,
                            int64_t ld, const int32_t* frames_host, const int32_t* end_host, void* stream) {
  if (!s || !frames_host || !end_host) return fail(SOPRO_ERR_INVALID, "align stream: null argument");
  if (B != s->rows || ld != s->g.ld)
    return fail(SOPRO_ERR_INVALID, "align stream: a trace of %d rows x ld %lld for a state of %d rows x ld %lld", B,
                (long long)ld, s->rows, (long long)s->g.ld);
  if (ring < 1 || n_attn < 1 || H < 1)
    return fail(SOPRO_ERR_INVALID, "align stream: ring=%d, n_attn=%d, H=%d must be >= 1", ring, n_attn, H);
  if ((long long)n_attn * H > 4096) return fail(SOPRO_ERR_INVALID, "align stream: n_attn x H = %lld > 4096", (long long)n_attn * H);
  StreamRows rows{};
  int Lp = 32;
  bool any = false;
  for (int b = 0; b < s->rows; ++b) {
    const int n = frames_host[b];
    if (s->ended[b] && (n != 0 || end_host[b]))
      return fail(SOPRO_ERR_INVALID, "align stream: row %d has ended; it takes no more frames until a begin", b);
    if (n < 0 || n > ring) return fail(SOPRO_ERR_INVALID, "align stream: frames[%d]=%d not in [0, ring=%d]", b, n, ring);
    if ((long long)s->t[b] + n > s->max_frames)
      return fail(SOPRO_ERR_INVALID, "align stream: row %d: %d frames after %d exceed max_frames %d", b, n, s->t[b],
                  s->max_frames);
    if (n > 0 && !probs) return fail(SOPRO_ERR_INVALID, "align stream: null probs");
    rows.len[b] = s->len[b];
    rows.t0[b] = s->t[b];
    rows.n[b] = n | (end_host[b] ? kEndFlag : 0);
    any = any || n > 0 || end_host[b];
    Lp = std::max(Lp, padded(s->len[b]));
  }
  if (any) {
    const size_t smem = (size_t)2 * Lp * 8 + (size_t)Lp * 4 + std::min<size_t>((size_t)kMaxTile * Lp * 8, kTileBytes);
    CK(cudaFuncSetAttribute(align_stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    align_stream_kernel<<<s->rows, kThreads, smem, reinterpret_cast<cudaStream_t>(stream)>>>(probs, ring, n_attn, B, H, rows,
                                                                                            s->state, s->g);
    CK(cudaGetLastError());
  }
  for (int b = 0; b < s->rows; ++b) {
    s->t[b] += frames_host[b];
    s->ended[b] = s->ended[b] || end_host[b] != 0;
  }
  return SOPRO_OK;
}

}  // extern "C"
