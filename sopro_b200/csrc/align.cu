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
#include <cmath>
#include <cstdio>

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

__global__ void __launch_bounds__(kThreads) align_kernel(const float* __restrict__ probs, int steps, int n_attn, int B, int H,
                                                         long long ld, const __grid_constant__ AlignRows rows, int b0,
                                                         unsigned* __restrict__ bits, int W, int* __restrict__ first) {
  extern __shared__ __align__(16) double sm[];
  __shared__ int s_ok;
  const int b = b0 + blockIdx.x;
  const int L = rows.len[blockIdx.x], T = rows.frames[blockIdx.x];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
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
    for (int i = tid; i < nt * L; i += kThreads) {
      const int tt = i / L, l = i - tt * L;
      const float* src = pb + (size_t)(t0 + tt) * t_stride + l;
      double a = 0.0;
#pragma unroll 1
      for (int s = 0; s < n_attn; ++s) {
#pragma unroll 4
        for (int h = 0; h < H; ++h) a += (double)__ldg(src + s * s_stride + (size_t)h * ld);
      }
      At[(size_t)tt * Lp + l] = a;
    }
    __syncthreads();
#pragma unroll 1
    for (int tt = 0; tt < nt; ++tt) {
      const int t = t0 + tt;
      const double* Sp = (t & 1) ? S0 : S1;  // S[t-1]
      double* Sn = (t & 1) ? S1 : S0;        // S[t]
      for (int l = tid; l < Lp; l += kThreads) {  // whole warps: Lp is a multiple of 32
        bool mv = false;
        if (l < L) {
          const double a = At[(size_t)tt * Lp + l];
          if (t == 0) {
            Sn[l] = l == 0 ? a : -INFINITY;
          } else {
            const double stay = Sp[l], move = l > 0 ? Sp[l - 1] : -INFINITY;
            mv = move > stay;
            Sn[l] = a + (mv ? move : stay);
          }
        }
        const unsigned word = __ballot_sync(0xffffffffu, mv);
        if (lane == 0 && t > 0) bb[(size_t)t * W + (l >> 5)] = word;
      }
      __syncthreads();  // S[t] complete, and the A tile free after its last step
    }
  }
  // ---- backtrack on warp 0 (t, l, w are warp-uniform)
  if (warp == 0) {
    int l = L - 1, t = T - 1;
#pragma unroll 1
    while (t > 0) {
      const int w = l >> 5;
      const int tr = t - lane;
      unsigned hi = 0u, lo = 0u;
      if (tr >= 1) {
        hi = __ldcg(bb + (size_t)tr * W + w);
        if (w > 0) lo = __ldcg(bb + (size_t)tr * W + w - 1);
      }
      const int n = min(32, t);
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
    if (lane == 0) s_ok = l == 0;
  }
  __syncthreads();
  const bool ok = s_ok != 0;
  for (long long l = tid; l < ld; l += kThreads) {
    if (!ok || l >= L) out[l] = -1;
    else if (l == 0) out[0] = 0;
  }
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

}  // extern "C"
