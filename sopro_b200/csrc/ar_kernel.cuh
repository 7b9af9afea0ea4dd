// Persistent autoregressive codec-token kernel for sm_90a.
//
// One launch runs up to n_steps frames for a batch of independent utterances:
// the body of SoproTTSModel.ar_stream's loop (reference model.py:265-305) —
// embedding add, 6x SSMLiteBlock.forward_step (nn/blocks.py:150-162), 3x cached
// TextXAttnBlock (nn/text.py:85-132), final RMSNorm + head (nn/generator.py:127-128),
// sample_token (sampling.py:24-93) and the anti-loop / EOS bookkeeping
// (model.py:274-305) — without returning to the host.
//
// Work decomposition (DESIGN.md §3): the grid is split into `g` TEAMS of `P`
// CTAs (one CTA per SM, co-resident: cooperative launch).  A team owns a group
// of <= 16 utterances.  Every stage of the step is a skinny GEMM
// [utterances x K] . [K x N]; inside a team the N output features are
// partitioned over the P CTAs.  Each CTA's weight slice is streamed global ->
// shared by 1-D TMA bulk copies into a ring of buffers, several stages ahead
// of its use (the weights do not depend on other CTAs), so a stage never waits
// on a weight load; the [utterances x K] activations are broadcast through L2.
// Stages are separated by a team-scoped barrier (one counter per team,
// release/acquire at gpu scope).  All arithmetic is fp32 (FMA on element pairs,
// warp-shuffle reductions); bf16 is a weight STORAGE format only.
//
// The step is written as a small INTERPRETER over a host-built stage program
// with ONE shared GEMV body: the whole per-step instruction footprint must
// stay near the SM's instruction cache (the first version, with one inlined
// specialisation per stage, was 590 KB of SASS and instruction-fetch bound).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace sopro {

constexpr int kThreads = 512;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxLayers = 16;
constexpr int kMaxTopK = 64;
constexpr int kCand = 128;  // candidate slots of the sampler's top-k
constexpr int kMaxUttPerTeam = 32;
constexpr int kMaxVocab = 8 * kThreads;
constexpr int kTapSlots = 16;     // dwconv tap rows staged per warp in the GLU stage (channels per task x utterances)
constexpr int kTimingSlots = 224;  // [0,160) stage stamps, [160,192) sampler phases, the rest spare
constexpr int kMaxStages = 6 * kMaxLayers + 2;
constexpr int kMaxTilesPerStep = 128;
constexpr int kMaxWBuf = 8;

__host__ __device__ constexpr int ilog2(int n) { return n > 1 ? 1 + ilog2(n / 2) : 0; }

// fma of an element pair, one rounding per element
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }

enum StageKind { K_GLU = 0, K_FFN1 = 1, K_FFN2 = 2, K_Q = 3, K_O = 4, K_HEAD = 5, K_ATT = 6, K_SAMPLE = 7, K_QATT = 8 };

struct LayerDev {
  const float* norm_w;
  const void* glu_w;
  const float* glu_b;
  const float* dw_w;  // [D][k]
  const float* dw_b;
  const float* ffn_norm_w;
  const void* w1;
  const float* b1;
  const void* w2;
  const float* b2;
  const float* nq_w;
  const void* wq;
  const void* wo;
  float gate_tanh;
  int has_attn;
  int attn_slot;       // index into the K/V cache
  int dil;
  int ring_len;        // (k-1)*dil + 1 (receptive field of the layer; informational)
  long long ring_off;  // float offset of this layer's conv state: [B][D][dil][KcP]
};

struct UttState {
  int len;       // tokens produced so far
  int last;      // last token (-1 = none)
  int streak;    // same-token streak (model.py:296-299)
  int recovery;  // next step samples with the recovery (top_p, temp) (model.py:274-279)
  int done;
  int pad[3];
};

struct SamplingDev {
  float top_p, temperature, rec_top_p, rec_temp, rep_pen;
  int top_k, anti_loop, loop_streak, min_gen, stop_on_first_eos;
};

// One weight tile of a CTA's slice: copied global -> shared by 1-D TMA bulk copies.
// The host builds, per team rank, the list of tiles of ONE AR step in consumption order.
struct TileDesc {
  unsigned long long src0;  // global address of part 0 (rows [row0, row0+nrows) of the matrix)
  unsigned long long src1;  // part 1: the GLU gate rows (row0 + D ...), else 0
  unsigned long long src2;  // part 2: epilogue constants. GLU: rows of the packed [D][KcE] table
                            // (dwconv taps, dwconv bias, GLU value bias, GLU gate bias); other stages:
                            // the 16-byte aligned span of the bias vector covering the tile's rows
  unsigned bytes0, bytes1, bytes2;  // multiples of 16
  int off2;                 // float index of the tile's first row inside part 2
  int row0;                 // first output feature of the tile
  int nrows;
  int pad[4];               // 64 bytes per tile: the shared-memory table is 8 KB, and the weight ring gets what it leaves
};
static_assert(sizeof(TileDesc) == 64, "the weight ring is sized around an 8 KB tile table");

// Warp task of a GEMV stage: R weight rows x TU utterances (wide) or R x TU/2 (narrow, TU >= 2).  The host picks
// the shape per stage (launch_ar); both accumulate every output in the same order, so the choice never changes a bit.
enum TaskShape { SHAPE_WIDE = 0, SHAPE_NARROW = 1 };

struct StageOp {
  unsigned char kind, layer, shape;
};

struct ArParams {
  int D, F, V, Vpad, H, Dh, Kc, KcP, KcE, n_layers, eos_id;  // KcP = Kc rounded up to 4, KcE = Kc+3 rounded up to 4
  LayerDev layer[kMaxLayers];
  StageOp prog[kMaxStages];
  int n_stage;
  const float* final_norm_w;
  const void* head_w;
  const float* head_b;
  const float* emb;  // [V+1][D]; row V = BOS
  // ---- session
  int B, steps, Lmax, noise_k;
  const float* cond;   // [B][steps][D]
  const float* noise;  // [B][steps][noise_k]
  const float* kc;     // [n_attn][B][H][Lmax][Dh]
  const float* vc;
  const int* text_len;
  float* ring;
  float* xa;      // [B][D]
  float* xb;      // [B][D]
  float* hbuf;    // [B][F]
  float* qbuf;    // [B][D]
  float* abuf;    // [B][D]
  float* logits;  // [B][Vpad]
  int* tokens;    // [B][steps]
  int* sampled;   // [B][steps]
  int* n_tokens;  // [B]
  int* done;      // [B]
  const int* forced;
  UttState* st;
  const SamplingDev* samp;
  float* trace_blocks;
  float* trace_logits;
  unsigned* tok_ll;       // [B][2] LL mode: {token | done << 30, flag}
  unsigned seq_base;      // LL mode: flags of this launch are seq_base + 1 ...
  unsigned* barrier;      // [g][32]
  const TileDesc* tiles;  // [P][kMaxTilesPerStep]
  const int* n_tiles;     // [P] tiles per step of each rank
  const unsigned char* stage_tiles;  // [P][kMaxStages] tiles of each stage
  int nbuf, wbuf_bytes, act_bytes;
  // dynamic shared-memory map [act | ring | table]: bytes from the 1024-byte aligned base (act is at 0)
  int ring_off, table_off;
  long long* timing;  // debug: [grid][kTimingSlots] clock64 stamps of step `timing_step` (null = off)
  int timing_step;
  int g, P, Bt;
  int PH;  // fused Q+attention stage: CTAs per head (P / H); rank r serves head r % H, utterances r / H + j*PH
  int t_begin, t_end;
  // word timestamps (null = off): every cross-attention weight of step t, [attn_ring][n_attn][B][H][attn_ld] fp32 in
  // step row t % attn_ring, attn_step = n_attn * B * H * attn_ld floats per step row
  float* attn_trace;
  long long attn_ld, attn_step;
  int attn_ring;
};

// ---------------------------------------------------------------------------
// small helpers
// ---------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// weights straight from global (K/V builder): read-only path, 4 consecutive k per lane
__device__ __forceinline__ float4 ldw4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 ldw4(const __nv_bfloat16* p) {
  uint2 u = __ldg(reinterpret_cast<const uint2*>(p));
  float4 r;
  r.x = __uint_as_float(u.x << 16);
  r.y = __uint_as_float(u.x & 0xffff0000u);
  r.z = __uint_as_float(u.y << 16);
  r.w = __uint_as_float(u.y & 0xffff0000u);
  return r;
}

// activations written by other CTAs: L2 only (never a stale L1 line)
__device__ __forceinline__ float4 ldcg4(const float* p) { return __ldcg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float ldcg1(const float* p) { return __ldcg(p); }

// ---------------------------------------------------------------------------
// LL ("low latency") exchange for small batches: every activation element is an 8-byte pair
// {value bits, flag}; the producer writes both with ONE 8-byte store, the consumer polls the data
// itself until the flag equals the producing stage's sequence number.  No fence, no atomic, no
// separate barrier: one L2 round trip per stage.  (Same idea as NCCL's LL protocol.)
// ---------------------------------------------------------------------------
__device__ __forceinline__ void ll_store(float* p, float v, unsigned flag) {
  asm volatile("st.volatile.global.v2.u32 [%0], {%1, %2};" ::"l"(p), "r"(__float_as_uint(v)), "r"(flag) : "memory");
}
__device__ __forceinline__ uint4 ll_load2(const float* p) {  // two consecutive elements, 16-byte aligned
  uint4 v;
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint2 ll_load1(const float* p) {
  uint2 v;
  asm volatile("ld.volatile.global.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
  return v;
}
// all threads: poll n_el (even) LL elements starting at src into dst (plain floats, shared memory).
// Four lines per thread are requested together (memory-level parallelism), then re-requested until valid.
__device__ __forceinline__ void ll_fetch(const float* __restrict__ src, int n_el, int n_valid, unsigned seq,
                                         float* __restrict__ dst) {
  constexpr int NB = 4;
  for (int base = threadIdx.x * 2; base < n_el; base += kThreads * 2 * NB) {
    uint4 v[NB];
    unsigned pending = 0;
#pragma unroll
    for (int j = 0; j < NB; ++j) {
      const int e = base + j * kThreads * 2;
      v[j] = make_uint4(0u, 0u, 0u, 0u);
      if (e < n_valid) {  // padding elements are never written: do not wait for them
        v[j] = ll_load2(src + (size_t)e * 2);
        pending |= 1u << j;
      }
    }
    while (pending) {
#pragma unroll
      for (int j = 0; j < NB; ++j) {
        if (pending & (1u << j)) {
          const int e = base + j * kThreads * 2;
          const bool second = e + 1 < n_valid;
          if (v[j].y == seq && (!second || v[j].w == seq)) pending &= ~(1u << j);
          else v[j] = ll_load2(src + (size_t)e * 2);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < NB; ++j) {
      const int e = base + j * kThreads * 2;
      if (e < n_el) {
        dst[e] = __uint_as_float(v[j].x);
        dst[e + 1] = (e + 1 < n_valid) ? __uint_as_float(v[j].z) : 0.f;
      }
    }
  }
}

struct Stamp {
  long long* buf;  // this CTA's slots, or null
  int n;
  __device__ __forceinline__ void mark() {
    if (buf && n < kTimingSlots) buf[n++] = clock64();
  }
};

// team barrier: monotonically increasing arrival counter, host zeroes it before each launch
__device__ __forceinline__ void team_barrier(unsigned* counter, unsigned P, unsigned& epoch, Stamp& ts) {
  __syncthreads();
  if (threadIdx.x == 0) {
    ts.mark();  // whole CTA finished the stage
    epoch += 1;
    const unsigned target = epoch * P;
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(counter), "r"(1u) : "memory");
    ts.mark();  // arrival posted
    unsigned v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
    } while (v < target);
    ts.mark();  // released
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------
// TMA 1-D bulk copy + mbarrier + cp.async helpers (sm_90 PTX)
// ---------------------------------------------------------------------------
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_1d(unsigned dst_smem, const void* src, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  const unsigned a = smem_u32(bar);
  unsigned ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(a), "r"(parity)
        : "memory");
  } while (!ok);
}
__device__ __forceinline__ void cp_async16(unsigned dst_smem, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst_smem), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait0() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ float lds32(unsigned a) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ float4 lds128(unsigned a) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
  return v;
}
// 4 consecutive weights at shared address a (WT = float: 16 B, bf16: 8 B)
template <typename WT>
__device__ __forceinline__ float4 ldsw4(unsigned a);
template <>
__device__ __forceinline__ float4 ldsw4<float>(unsigned a) {
  return lds128(a);
}
template <>
__device__ __forceinline__ float4 ldsw4<__nv_bfloat16>(unsigned a) {
  unsigned x, y;
  asm volatile("ld.shared.v2.b32 {%0,%1}, [%2];" : "=r"(x), "=r"(y) : "r"(a));
  float4 r;
  r.x = __uint_as_float(x << 16);
  r.y = __uint_as_float(x & 0xffff0000u);
  r.z = __uint_as_float(y << 16);
  r.w = __uint_as_float(y & 0xffff0000u);
  return r;
}

// The weight ring of a CTA: nbuf shared buffers filled by TMA in tile order.  Tile i lives in
// buffer i % nbuf and completes phase (i / nbuf) of that buffer's mbarrier.  All indices are kept
// as small wrapping counters: no integer division on the critical path.
struct WeightRing {
  unsigned long long* bars;  // [kMaxWBuf] "full" mbarriers
  unsigned base;             // shared address of buffer 0
  unsigned wbuf;             // bytes per buffer
  int nbuf;
  const TileDesc* table;     // this rank's tiles (shared-memory copy)
  int n_tiles;               // per step
  int tile;                  // table index of the next tile to consume
  int buf;                   // its buffer
  unsigned phase;            // bit b: parity to wait for on buffer b
  int itile;                 // table index of the next tile to issue
  int left;                  // tiles of this launch not yet issued
  int inflight;              // issued, not yet consumed
  __device__ __forceinline__ void issue_into(const TileDesc& td, int b) const {  // one thread
    mbar_expect_tx(&bars[b], td.bytes0 + td.bytes1 + td.bytes2);
    const unsigned dst = base + (unsigned)b * wbuf;
    tma_load_1d(dst, reinterpret_cast<const void*>(td.src0), td.bytes0, &bars[b]);
    if (td.bytes1) tma_load_1d(dst + td.bytes0, reinterpret_cast<const void*>(td.src1), td.bytes1, &bars[b]);
    if (td.bytes2)
      tma_load_1d(dst + td.bytes0 + td.bytes1, reinterpret_cast<const void*>(td.src2), td.bytes2, &bars[b]);
  }
  __device__ __forceinline__ void start(int total) {  // all threads (uniform bookkeeping)
    tile = 0;
    buf = 0;
    phase = 0;
    itile = 0;
    left = total;
    inflight = 0;
    for (int b = 0; b < nbuf && left > 0; ++b) {
      if (threadIdx.x == 0) issue_into(table[itile], b);
      if (++itile == n_tiles) itile = 0;
      --left;
      ++inflight;
    }
  }
  // all threads: wait for the next tile; returns its shared address
  __device__ __forceinline__ unsigned acquire(const TileDesc*& td) const {
    td = &table[tile];
    mbar_wait(&bars[buf], (phase >> buf) & 1u);
    return base + (unsigned)buf * wbuf;
  }
  // all threads, after the last read of the tile: recycle its buffer with the next tile to issue
  __device__ __forceinline__ void release() {
    __syncthreads();
    --inflight;
    if (left > 0) {
      if (threadIdx.x == 0) issue_into(table[itile], buf);
      if (++itile == n_tiles) itile = 0;
      --left;
      ++inflight;
    }
    phase ^= 1u << buf;
    if (++buf == nbuf) buf = 0;
    if (++tile == n_tiles) tile = 0;
  }
  // all threads: bulk copies still in flight must land before the CTA exits
  __device__ __forceinline__ void drain() {
    while (inflight > 0) {
      mbar_wait(&bars[buf], (phase >> buf) & 1u);
      phase ^= 1u << buf;
      if (++buf == nbuf) buf = 0;
      --inflight;
    }
  }
};

// ---------------------------------------------------------------------------
// warp GEMV tile, 2 rows x TU utterances: out[r][u] = sum_k W[row_r][k] * act[u][k]
// lanes split K (4 consecutive k per lane per 128-k chunk), fp32 FMA accumulation on element pairs, butterfly
// reduction (every lane ends with all totals).  Weights AND activations in shared memory.
// ---------------------------------------------------------------------------
// After the K loop the 2*TU partial sums of every lane are combined with a TRANSPOSED reduction:
// log2(2*TU) halving exchanges (each lane keeps half of the outputs and hands the other half to its
// partner) followed by plain butterflies: 2*TU - 1 + (5 - log2(2*TU)) shuffles instead of 5 * 2*TU.
// On return every lane holds the total of output o = (lane >> (5 - log2(2*TU))) & (2*TU - 1),
// with o = r * TU + u.
template <int N>
__device__ __forceinline__ float reduce_transposed(float (&v)[N], int lane) {
  int n = N;
#pragma unroll
  for (int s = 16; s >= 1; s >>= 1) {
    if (n > 1) {
      const int half = n >> 1;
      const bool up = (lane & s) != 0;
#pragma unroll
      for (int i = 0; i < N / 2; ++i) {
        if (i < half) {
          const float keep = up ? v[i + half] : v[i];
          const float send = up ? v[i] : v[i + half];
          v[i] = keep + __shfl_xor_sync(0xffffffffu, send, s);
        }
      }
      n = half;
    } else {
      v[0] += __shfl_xor_sync(0xffffffffu, v[0], s);
    }
  }
  return v[0];
}
template <>
__device__ __forceinline__ float reduce_transposed<1>(float (&v)[1], int lane) {
  return warp_sum(v[0]);
}

// UNROLL: K-loop unroll (the narrow task shape passes 1: the step's instructions must stay near the instruction cache)
template <int R, int TU, typename WT, int UNROLL = (R * TU >= 32 ? 1 : 3)>
__device__ __forceinline__ float warp_rows_s(const unsigned (&w)[R], unsigned act, int K, int lane) {
  float2 acc[R][TU];
#pragma unroll
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int u = 0; u < TU; ++u) acc[r][u] = make_float2(0.f, 0.f);
  // big register tiles (64 float2 accumulators) leave no room for unrolled loads
#pragma unroll(UNROLL)
  for (int k = lane * 4; k < K; k += 128) {
    float4 wv[R];
#pragma unroll
    for (int r = 0; r < R; ++r) wv[r] = ldsw4<WT>(w[r] + (unsigned)k * (unsigned)sizeof(WT));
#pragma unroll
    for (int u = 0; u < TU; ++u) {
      const float4 x = lds128(act + ((unsigned)u * (unsigned)K + (unsigned)k) * 4u);
#pragma unroll
      for (int r = 0; r < R; ++r) {
        acc[r][u] = ffma2(make_float2(wv[r].x, wv[r].y), make_float2(x.x, x.y), acc[r][u]);
        acc[r][u] = ffma2(make_float2(wv[r].z, wv[r].w), make_float2(x.z, x.w), acc[r][u]);
      }
    }
  }
  float v[R * TU];
#pragma unroll
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int u = 0; u < TU; ++u) v[r * TU + u] = acc[r][u].x + acc[r][u].y;
  return reduce_transposed<R * TU>(v, lane);
}

// same, weights from global memory (K/V builder only)
template <int TU, typename WT>
__device__ __forceinline__ void warp_rows_g(const WT* w0, const WT* w1, const float* __restrict__ act, int K, int lane,
                                            float (&out)[2][TU]) {
  float2 acc[2][TU];
#pragma unroll
  for (int u = 0; u < TU; ++u) acc[0][u] = acc[1][u] = make_float2(0.f, 0.f);
#pragma unroll 3
  for (int k = lane * 4; k < K; k += 128) {
    const float4 wa = ldw4(w0 + k);
    const float4 wb = ldw4(w1 + k);
#pragma unroll
    for (int u = 0; u < TU; ++u) {
      const float4 x = *reinterpret_cast<const float4*>(act + (size_t)u * K + k);
      acc[0][u] = ffma2(make_float2(wa.x, wa.y), make_float2(x.x, x.y), acc[0][u]);
      acc[0][u] = ffma2(make_float2(wa.z, wa.w), make_float2(x.z, x.w), acc[0][u]);
      acc[1][u] = ffma2(make_float2(wb.x, wb.y), make_float2(x.x, x.y), acc[1][u]);
      acc[1][u] = ffma2(make_float2(wb.z, wb.w), make_float2(x.z, x.w), acc[1][u]);
    }
  }
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int u = 0; u < TU; ++u) out[r][u] = warp_sum(acc[r][u].x + acc[r][u].y);
}

// pick element [r][u] of a register array with runtime indices without spilling
template <int TU>
__device__ __forceinline__ float pick2(const float (&a)[2][TU], int r, int u) {
  float v = a[0][0];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < TU; ++j) v = (i == r && j == u) ? a[i][j] : v;
  return v;
}

// ---------------------------------------------------------------------------
// activation staging: [nb][K] rows -> smem, optionally RMS-normalised
// (nn/blocks.py:32-37: y = (x * rsqrt(mean(x^2) + eps)) * w, two roundings).
// The whole [nb][K] block is fetched by ALL threads with one wave of 16-byte cp.async (a single
// L2 round trip, no registers); the norm weights are requested before the wait so both latencies
// overlap.  src == nullptr: the rows are already in `dst` (layer 0), normalise in place.
// ---------------------------------------------------------------------------
template <bool LL = false>
__device__ __forceinline__ void stage_rows(const float* __restrict__ src, int nb, int K, float* __restrict__ dst,
                                           const float* __restrict__ norm_w, float* __restrict__ raw_copy,
                                           unsigned seq = 0) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (src && !LL) {
    const unsigned dst_s = smem_u32(dst);
    const int total = nb * K;
    for (int e = threadIdx.x * 4; e < total; e += kThreads * 4) cp_async16(dst_s + (unsigned)e * 4u, src + e);
  }
  cp_async_commit();
  float4 nw[4];  // this lane's norm weights when K <= 512 (else they are read in the loop)
  const bool pre = norm_w != nullptr && K <= 512;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const int k = lane * 4 + c * 128;
    nw[c] = (pre && k < K) ? __ldg(reinterpret_cast<const float4*>(norm_w + k)) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (src && LL) ll_fetch(src, nb * K, nb * K, seq, dst);  // src points at LL pairs
  cp_async_wait0();
  __syncthreads();
  if (!norm_w && !raw_copy) return;
  for (int u = warp; u < nb; u += kWarps) {
    float* d = dst + (size_t)u * K;
    float ss = 0.f;
    for (int k = lane * 4; k < K; k += 128) {
      const float4 v = *reinterpret_cast<float4*>(d + k);
      if (raw_copy) *reinterpret_cast<float4*>(raw_copy + (size_t)u * K + k) = v;
      ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    }
    if (norm_w) {
      ss = warp_sum(ss);
      const float inv = 1.0f / sqrtf(ss / (float)K + 1e-6f);
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int k = lane * 4 + c * 128;
        if (pre && k < K) {
          float4 v = *reinterpret_cast<float4*>(d + k);
          v.x = (v.x * inv) * nw[c].x;
          v.y = (v.y * inv) * nw[c].y;
          v.z = (v.z * inv) * nw[c].z;
          v.w = (v.w * inv) * nw[c].w;
          *reinterpret_cast<float4*>(d + k) = v;
        }
      }
      if (!pre) {
        for (int k = lane * 4; k < K; k += 128) {
          float4 v = *reinterpret_cast<float4*>(d + k);
          const float4 w = __ldg(reinterpret_cast<const float4*>(norm_w + k));
          v.x = (v.x * inv) * w.x;
          v.y = (v.y * inv) * w.y;
          v.z = (v.z * inv) * w.z;
          v.w = (v.w * inv) * w.w;
          *reinterpret_cast<float4*>(d + k) = v;
        }
      }
    }
  }
}

__device__ __forceinline__ float sigmoid_ref(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

// Row partition of N outputs over the team's P CTAs.
__device__ __forceinline__ void slice(int N, int rank, int P, int& lo, int& hi) {
  lo = (int)(((unsigned)N * (unsigned)rank) / (unsigned)P);  // N * P < 2^32 (checked on the host)
  hi = (int)(((unsigned)N * (unsigned)(rank + 1)) / (unsigned)P);
}

struct TeamCtx {
  int team, rank, P;
  int b0, nb;  // utterances [b0, b0+nb)
};

// ---------------------------------------------------------------------------
// Cached text cross-attention core (nn/text.py:101-128): softmax(q.K^T / sqrt(Dh)) . V in fp32 over the keys
// l < text_len, ONE (utterance, head) item per GROUP of 256 threads, two items side by side in a CTA.
//   1. scores: 8 threads per key read the key row straight from L2 (the K/V caches are read-only during the launch:
//      no shared-memory staging, any text length), 3-step shuffle reduction -> sc[l] in shared memory
//   2. max / sum: every warp of the group, redundantly
//   3. output: thread (g, c) accumulates the keys l = g mod G for the float4 chunk c of the head dimension
//      (G = 256 / (Dh/4) key groups, one L2 round trip with every load in flight)
//   4. fixed-order sum over the key groups, normalise, nan_to_num (nn/text.py:128), store
// TRACE (word timestamps, p.attn_trace set): the group's first warp also stores the weights exp(sc[l] - mx) / sum after 2.
// The TRACE = false instantiations are the untraced kernels, unchanged.
// Groups synchronise with named barriers (ids 1, 2), never with the CTA barrier.
// smem per group: sc[Lp] | part[kAttG][Dh]
// ---------------------------------------------------------------------------
constexpr int kAttGroup = 256;
constexpr int kAttG = 32;  // upper bound of the key groups (Dh >= 32)
constexpr int kAttVU = 8;  // value rows per thread requested together

// word timestamps: the trace row of the step the CTA is computing (written only by the TRACE instantiations)
__shared__ int g_attn_step;

__device__ __forceinline__ void group_sync(int grp) {
  asm volatile("bar.sync %0, %1;" ::"r"(grp + 1), "r"(kAttGroup) : "memory");
}

template <bool TRACE>
__device__ __forceinline__ void attention_item(const ArParams& p, const LayerDev& L, int b, int h, const float* __restrict__ qs,
                                               float* __restrict__ sc, float* __restrict__ part, int grp, int gt, int ll,
                                               unsigned out_seq) {
  const int lane = gt & 31;
  const int Dh = p.Dh, D = p.D, H = p.H;
  const int len = p.text_len[b];
  const size_t kv_off = ((((size_t)L.attn_slot * p.B + b) * H + h) * p.Lmax) * Dh;
  const float* __restrict__ Kp = p.kc + kv_off;
  const float* __restrict__ Vp = p.vc + kv_off;
  const float scale = 1.0f / sqrtf((float)Dh);
  // Every L2 read of an item is a round trip of ~1-2k cycles on a busy GPU, and the item is on the step's critical path:
  // the key rows of two score rounds, and kAttVU value rows per thread, are requested together.  The sums keep the
  // order of one key, one value row at a time.
  // 1. scores: keys l and l + 32 of a round pair, 8 threads per key
  {
    const int sub = gt & 7;
    for (int l0 = 0; l0 < len; l0 += 2 * (kAttGroup / 8)) {
      const int la = l0 + (gt >> 3), lb = la + kAttGroup / 8;
      float sa = 0.f, sb = 0.f;
      for (int d0 = sub * 4; d0 < Dh; d0 += 4 * 32) {
        float4 ka[4], kb[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int d = d0 + 32 * i;
          ka[i] = (la < len && d < Dh) ? __ldg(reinterpret_cast<const float4*>(Kp + (size_t)la * Dh + d)) : make_float4(0.f, 0.f, 0.f, 0.f);
          kb[i] = (lb < len && d < Dh) ? __ldg(reinterpret_cast<const float4*>(Kp + (size_t)lb * Dh + d)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int d = d0 + 32 * i;
          if (d < Dh) {
            const float4 qq = *reinterpret_cast<const float4*>(qs + d);
            if (la < len) {
              const float4 kk = ka[i];
              sa += kk.x * qq.x + kk.y * qq.y + kk.z * qq.z + kk.w * qq.w;
            }
            if (lb < len) {
              const float4 kk = kb[i];
              sb += kk.x * qq.x + kk.y * qq.y + kk.z * qq.z + kk.w * qq.w;
            }
          }
        }
      }
      sa += __shfl_xor_sync(0xffffffffu, sa, 1);
      sa += __shfl_xor_sync(0xffffffffu, sa, 2);
      sa += __shfl_xor_sync(0xffffffffu, sa, 4);
      sb += __shfl_xor_sync(0xffffffffu, sb, 1);
      sb += __shfl_xor_sync(0xffffffffu, sb, 2);
      sb += __shfl_xor_sync(0xffffffffu, sb, 4);
      if (sub == 0 && la < len) sc[la] = sa * scale;
      if (sub == 0 && lb < len) sc[lb] = sb * scale;
    }
  }
  group_sync(grp);
  // 2. softmax statistics
  float mx = -INFINITY;
  for (int l = lane; l < len; l += 32) mx = fmaxf(mx, sc[l]);
  mx = warp_max(mx);
  float sum = 0.f;
  for (int l = lane; l < len; l += 32) sum += expf(sc[l] - mx);
  sum = warp_sum(sum);
  if (TRACE && gt < 32) {  // the weights the output applies (nan_to_num as in 4)
    float* row = p.attn_trace + (size_t)g_attn_step * p.attn_step + (((size_t)L.attn_slot * p.B + b) * H + h) * p.attn_ld;
    for (int l = lane; l < len; l += 32) {
      const float w = expf(sc[l] - mx) / sum;
      row[l] = isfinite(w) ? w : 0.f;
    }
  }
  // 3. partial outputs, keys l = g mod G in ascending order
  const int C4 = Dh >> 2;
  const int G = min(kAttGroup / C4, kAttG);
  {
    const int g = gt / C4, c = gt - g * C4;
    if (g < G) {
      float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int l0 = g; l0 < len; l0 += kAttVU * G) {
        float4 vr[kAttVU];
#pragma unroll
        for (int j = 0; j < kAttVU; ++j) {
          const int l = l0 + j * G;
          vr[j] = l < len ? __ldg(reinterpret_cast<const float4*>(Vp + (size_t)l * Dh + c * 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int j = 0; j < kAttVU; ++j) {
          const int l = l0 + j * G;
          if (l < len) {
            const float e = expf(sc[l] - mx);
            const float4 v = vr[j];
            o.x += e * v.x;
            o.y += e * v.y;
            o.z += e * v.z;
            o.w += e * v.w;
          }
        }
      }
      *reinterpret_cast<float4*>(part + (size_t)g * Dh + c * 4) = o;
    }
  }
  group_sync(grp);
  // 4. combine
  if (gt < Dh) {
    float acc = 0.f;
    for (int g = 0; g < G; ++g) acc += part[(size_t)g * Dh + gt];
    acc = acc / sum;
    if (!isfinite(acc)) acc = 0.f;
    const size_t aoff = (size_t)b * D + (size_t)h * Dh + gt;
    if (ll) ll_store(p.abuf + aoff * 2, acc, out_seq);
    else p.abuf[aoff] = acc;
  }
  group_sync(grp);  // sc / part are reused by the group's next item
}

// smem floats per group of the attention stages
__host__ __device__ inline int att_group_floats(int Lmax, int Dh) { return ((Lmax + 3) & ~3) + kAttG * Dh; }

// The attention stage of the un-fused program (q comes from the q stage through the exchange buffer): work items
// (utterance, head) round-robin over the team's CTAs, two items at a time per CTA.
// smem: [qs[Dh] | sc | part] x 2 groups
template <bool TRACE>
__device__ __noinline__ void stage_attention(const ArParams& p, int li, int rank, int P, int b0, int nb,
                                             float* __restrict__ smem, int ll, unsigned q_seq, unsigned out_seq) {
  const LayerDev& L = p.layer[li];
  const int tid = threadIdx.x;
  const int grp = tid / kAttGroup, gt = tid - grp * kAttGroup;
  const int H = p.H, Dh = p.Dh, D = p.D;
  const int gf = Dh + att_group_floats(p.Lmax, Dh);
  float* qs = smem + (size_t)grp * gf;
  float* sc = qs + Dh;
  float* part = sc + ((p.Lmax + 3) & ~3);
  const int n_items = nb * H;
  for (int item = rank + grp * P; item < n_items; item += 2 * P) {
    const int u = item / H, h = item % H;
    const int b = b0 + u;
    if (gt * 4 < Dh) {
      const size_t qoff = (size_t)b * D + (size_t)h * Dh + gt * 4;
      float4 q4;
      if (ll) {
        uint4 a, c;
        do {
          a = ll_load2(p.qbuf + qoff * 2);
          c = ll_load2(p.qbuf + qoff * 2 + 4);
        } while (a.y != q_seq || a.w != q_seq || c.y != q_seq || c.w != q_seq);
        q4 = make_float4(__uint_as_float(a.x), __uint_as_float(a.z), __uint_as_float(c.x), __uint_as_float(c.z));
      } else {
        q4 = ldcg4(p.qbuf + qoff);
      }
      *reinterpret_cast<float4*>(qs + gt * 4) = q4;
    }
    group_sync(grp);
    attention_item<TRACE>(p, L, b, h, qs, sc, part, grp, gt, ll, out_seq);
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------
// Sampler (sampling.py:24-93) + bookkeeping (model.py:293-305), one CTA per utterance.
// Probabilities live in shared memory; every loop over the vocabulary is a rolled loop
// (v = tid, tid+512, ...) to keep the code small.
// ---------------------------------------------------------------------------
struct SamplerSmem {
  float red_v[kWarps];
  int red_i[kWarps];
  float topv[kCand];  // unordered candidates; empty slots hold (-1, INT_MAX)
  int topi[kCand];
  float sortv[kMaxTopK];  // the best kMaxTopK of them, best first
  int sorti[kMaxTopK];
  float bc_f;
  int bc_i;
  int fallback;
  unsigned n_cand;
  // radix select (cold path)
  unsigned hist[2048];
  unsigned wtot[kWarps];
  unsigned sel_digit, sel_need;
  unsigned n_gt, n_eq, n_eq2;
};

__device__ __forceinline__ bool cand_before(float av, int ai, float bv, int bi) {
  // the device's tie contract: larger value first, ties -> lower index (torch's CPU topk / sort define no tie order)
  return av > bv || (av == bv && ai < bi);
}
__device__ __forceinline__ void warp_argmax(float& v, int& i) {
#pragma unroll 1
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (cand_before(ov, oi, v, i)) {
      v = ov;
      i = oi;
    }
  }
}

// All 512 threads order the kCand candidate slots by counting: rank(i) = #{j : slot j comes before
// slot i} (value desc, index asc); 4 threads per slot, 32 comparisons each, then the best
// kMaxTopK are scattered to sortv/sorti.  Empty slots (-1, INT_MAX) tie with each other and rank
// after every real candidate.  ~60 instructions, no single-warp serial section.
__device__ __forceinline__ void rank_order(SamplerSmem& sm) {
  const int tid = threadIdx.x;
  if (tid < kMaxTopK) {
    sm.sortv[tid] = -1.f;
    sm.sorti[tid] = 0x7fffffff;
  }
  __syncthreads();
  const int i = tid >> 2, g = tid & 3;
  const float vi = sm.topv[i];
  const int ii = sm.topi[i];
  int cnt = 0;
#pragma unroll 4
  for (int j = g * (kCand / 4); j < (g + 1) * (kCand / 4); ++j) cnt += cand_before(sm.topv[j], sm.topi[j], vi, ii) ? 1 : 0;
  cnt += __shfl_xor_sync(0xffffffffu, cnt, 1);
  cnt += __shfl_xor_sync(0xffffffffu, cnt, 2);
  if (g == 0 && cnt < kMaxTopK && ii != 0x7fffffff) {
    sm.sortv[cnt] = vi;
    sm.sorti[cnt] = ii;
  }
  __syncthreads();
}

// block-wide argmax; result valid in every thread
__device__ __forceinline__ void block_argmax(float& v, int& i, SamplerSmem& sm) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  warp_argmax(v, i);
  if (lane == 0) {
    sm.red_v[warp] = v;
    sm.red_i[warp] = i;
  }
  __syncthreads();
  if (warp == 0) {
    float bv = lane < kWarps ? sm.red_v[lane] : -INFINITY;
    int bi = lane < kWarps ? sm.red_i[lane] : 0x7fffffff;
    warp_argmax(bv, bi);
    if (lane == 0) {
      sm.bc_f = bv;
      sm.bc_i = bi;
    }
  }
  __syncthreads();
  v = sm.bc_f;
  i = sm.bc_i;
}
__device__ __forceinline__ float block_max(float v, SamplerSmem& sm) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  v = warp_max(v);
  if (lane == 0) sm.red_v[warp] = v;
  __syncthreads();
  float r = lane < kWarps ? sm.red_v[lane] : -INFINITY;
  r = warp_max(r);
  __syncthreads();
  return r;
}
__device__ __forceinline__ float block_sum(float v, SamplerSmem& sm) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  v = warp_sum(v);
  if (lane == 0) sm.red_v[warp] = v;
  __syncthreads();
  float r = lane < kWarps ? sm.red_v[lane] : 0.f;
  r = warp_sum(r);
  __syncthreads();
  return r;
}

// COLD: exact top-kk of the candidates {v : sp[v] >= t_lb} when they do not fit the 64 slots:
// MSB-first radix select on the float bits (p >= 0, so uint order == float order), 11+11+9 bits.
// Leaves the kk selected (value, index) pairs, unsorted, in sm.topv / sm.topi.
__device__ __noinline__ void topk_radix_cold(const float* __restrict__ sp, int V, int kk, float t_lb, SamplerSmem& sm) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  unsigned prefix = 0, pmask = 0, need = (unsigned)kk;
  for (int pass = 0; pass < 3; ++pass) {
    const int shift = pass == 0 ? 20 : (pass == 1 ? 9 : 0);
    const int nbits = pass == 2 ? 9 : 11;
    const int NB = 1 << nbits;
    const int PER = NB / kThreads > 0 ? NB / kThreads : 1;
    for (int i = tid; i < NB; i += kThreads) sm.hist[i] = 0;
    __syncthreads();
    for (int v = tid; v < V; v += kThreads) {
      const float q = sp[v];
      const unsigned key = __float_as_uint(q);
      if (q >= t_lb && (key & pmask) == prefix) atomicAdd(&sm.hist[(key >> shift) & (NB - 1)], 1u);
    }
    __syncthreads();
    unsigned mine = 0;
    if (tid * PER < NB)
      for (int j = 0; j < PER; ++j) mine += sm.hist[tid * PER + j];
    unsigned x = mine;  // inclusive suffix sum within the warp (bins above mine)
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned y = __shfl_down_sync(0xffffffffu, x, o);
      if (lane + o < 32) x += y;
    }
    if (lane == 0) sm.wtot[warp] = x;
    __syncthreads();
    unsigned higher = 0;
    for (int w = warp + 1; w < kWarps; ++w) higher += sm.wtot[w];
    const unsigned incl = x + higher, excl = incl - mine;
    if (excl < need && need <= incl) {  // exactly one thread
      unsigned run = excl;
      for (int j = PER - 1; j >= 0; --j) {
        const unsigned c = sm.hist[tid * PER + j];
        if (run + c >= need) {
          sm.sel_digit = (unsigned)(tid * PER + j);
          sm.sel_need = need - run;
          break;
        }
        run += c;
      }
    }
    __syncthreads();
    prefix |= sm.sel_digit << shift;
    pmask |= (unsigned)(NB - 1) << shift;
    need = sm.sel_need;
    __syncthreads();
  }
  const unsigned T = prefix;
  const int n_gt_expect = kk - (int)need;
  if (tid == 0) {
    sm.n_gt = 0;
    sm.n_eq = 0;
    sm.n_eq2 = 0;
  }
  __syncthreads();
  for (int v = tid; v < V; v += kThreads) {
    const float q = sp[v];
    const unsigned key = __float_as_uint(q);
    if (q >= t_lb && key > T) {
      const unsigned slot = atomicAdd(&sm.n_gt, 1u);
      sm.topv[slot] = q;
      sm.topi[slot] = v;
    } else if (q >= t_lb && key == T) {
      atomicAdd(&sm.n_eq, 1u);
    }
  }
  __syncthreads();
  if (sm.n_eq == need) {  // no tie straddles the cut
    for (int v = tid; v < V; v += kThreads) {
      const float q = sp[v];
      if (q >= t_lb && __float_as_uint(q) == T) {
        const unsigned slot = n_gt_expect + atomicAdd(&sm.n_eq2, 1u);
        sm.topv[slot] = q;
        sm.topi[slot] = v;
      }
    }
  } else {  // ties at the threshold: take the lowest indices, one block argmax per pick
    int taken_below = -1;  // indices <= taken_below are already taken
    for (unsigned j = 0; j < need; ++j) {
      float bv = -1.f;
      int bi = 0x7fffffff;
      for (int v = tid; v < V; v += kThreads) {
        if (v > taken_below && __float_as_uint(sp[v]) == T && sp[v] >= t_lb && bv < 0.f) {
          bv = 1.f;
          bi = v;
        }
      }
      block_argmax(bv, bi, sm);
      if (tid == 0) {
        sm.topv[n_gt_expect + j] = __uint_as_float(T);
        sm.topi[n_gt_expect + j] = bi;
      }
      taken_below = bi;
    }
  }
  __syncthreads();
}

// COLD: argmax of the penalised, temperature-scaled logits (sampling.py:65,80,90)
__device__ __noinline__ int argmax_logits_cold(const float* __restrict__ sx, int V, SamplerSmem& sm) {
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int v = threadIdx.x; v < V; v += kThreads)
    if (cand_before(sx[v], v, bv, bi)) {
      bv = sx[v];
      bi = v;
    }
  __syncthreads();
  block_argmax(bv, bi, sm);
  return bi;
}

// sx, sp: smem [Vpad] floats; flags: smem [Vpad] bytes
__device__ __noinline__ void sample_utterance(const ArParams& p, int b, int t, float* __restrict__ sx,
                                              float* __restrict__ sp, unsigned char* __restrict__ flags,
                                              SamplerSmem& sm, int ll, unsigned lg_seq, unsigned out_seq) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int V = p.V;
  long long* dbg = (p.timing && t == p.timing_step && tid == 0) ? p.timing + (size_t)blockIdx.x * kTimingSlots + 160 : nullptr;
  int dn = 0;
#define SMARK() do { if (dbg) dbg[dn++] = clock64(); } while (0)
  SMARK();
  const UttState st = p.st[b];
  const SamplingDev spar = p.samp[b];
  int* toks = p.tokens + (size_t)b * p.steps;
  if (st.done) {  // CTA-uniform
    if (ll && tid == 0) ll_store(reinterpret_cast<float*>(p.tok_ll) + (size_t)b * 2, __uint_as_float(1u << 30), out_seq);
    return;
  }
  const float top_p = st.recovery ? spar.rec_top_p : spar.top_p;
  const float temp = st.recovery ? spar.rec_temp : spar.temperature;
  const float rep = spar.rep_pen;
  const int hlen = st.len;

  // 1. repetition-penalty flags from set(hist[-50:]); logits -> nan_to_num -> /T -> penalty.
  //    The logits row is fetched with one wave of 16-byte cp.async (a single L2 round trip).
  const float* lg = p.logits + (size_t)b * p.Vpad;
  if (ll) {
    ll_fetch(p.logits + (size_t)b * p.Vpad * 2, p.Vpad, V, lg_seq, sx);
  } else {
    const unsigned sx_s = smem_u32(sx);
    for (int v = tid * 4; v < p.Vpad; v += kThreads * 4) cp_async16(sx_s + (unsigned)v * 4u, lg + v);
  }
  cp_async_commit();
  for (int v = tid; v < p.Vpad; v += kThreads) flags[v] = 0;
  if (tid < kCand) {
    sm.topv[tid] = -1.f;
    sm.topi[tid] = 0x7fffffff;
  }
  if (tid == 0) sm.n_cand = 0;
  __syncthreads();
  if (rep != 1.0f && tid < 50 && tid < hlen) {
    const int tok = toks[hlen - 1 - tid];
    if (tok >= 0 && tok < V) flags[tok] = 1;
  }
  cp_async_wait0();
  __syncthreads();
  SMARK();  // 1: state + logits fetched
  float mx = -INFINITY;
#pragma unroll 1
  for (int v = tid; v < V; v += kThreads) {
    float x = sx[v];
    if (isnan(x)) x = -1e9f;
    else if (isinf(x)) x = x > 0.f ? 1e9f : -1e9f;
    if (temp != 0.0f && temp != 1.0f) x = x / temp;
    if (flags[v]) x = (x < 0.f) ? x * rep : x / rep;
    sx[v] = x;
    mx = fmaxf(mx, x);
  }
  // 2. softmax + nan_to_num; each thread remembers its largest probability
  SMARK();  // 2: penalised logits
  mx = block_max(mx, sm);
  SMARK();  // 3: block max
  float se = 0.f;
#pragma unroll 1
  for (int v = tid; v < V; v += kThreads) {
    const float e = expf(sx[v] - mx);
    sp[v] = e;
    se += e;
  }
  se = block_sum(se, sm);
  SMARK();  // 4: exp + block sum
  float lmax = 0.f;
#pragma unroll 1
  for (int v = tid; v < V; v += kThreads) {
    float q = sp[v] / se;
    if (!isfinite(q)) q = 0.f;
    sp[v] = q;
    lmax = fmaxf(lmax, q);
  }
  const int kk = min(min(spar.top_k, V), kMaxTopK);
  SMARK();  // 5: probabilities
  // 3. top-k.  (a) a threshold from a histogram of the probabilities' float bits: 64 bins per octave, 1024 bins below the
  //    largest probability (16 octaves); the bin in which the running count (from the top) reaches kk gives the candidate
  //    set {p : bin(p) <= b} -- a superset of the kk largest, a few elements more on typical data.  (b) if the
  //    candidates fit the kCand slots, block-parallel rank ordering both selects and orders them; otherwise (extremely
  //    peaked rows whose kk-th value sits more than 16 octaves below the maximum, or massive ties) the exact radix
  //    select (cold) runs.  Order everywhere: value desc, index asc (the contract; torch's topk/sort leave ties open).
  constexpr int kBins = 1024;
  float bm;
  {
    for (int i = tid; i < kBins; i += kThreads) sm.hist[i] = 0;
    bm = block_max(lmax, sm);  // also the barrier between clearing and counting
    const int top_key = (int)(__float_as_uint(bm) >> 17);  // sign 0 | 8 exponent bits | 6 mantissa bits
#pragma unroll 1
    for (int v = tid; v < V; v += kThreads) {
      const int rel = min(top_key - (int)(__float_as_uint(sp[v]) >> 17), kBins - 1);
      atomicAdd(&sm.hist[rel], 1u);
    }
    __syncthreads();
    // inclusive scan over the bins (2 per thread), find the bin where the count reaches kk
    const unsigned c0 = sm.hist[2 * tid], c1 = sm.hist[2 * tid + 1];
    unsigned x = c0 + c1;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) sm.wtot[warp] = x;
    __syncthreads();
    unsigned before = 0;
    for (int w = 0; w < warp; ++w) before += sm.wtot[w];
    const unsigned incl = before + x, excl = incl - (c0 + c1);
    if (excl < (unsigned)kk && (unsigned)kk <= incl) {  // exactly one thread
      const bool first = excl + c0 >= (unsigned)kk;
      sm.sel_digit = (unsigned)(2 * tid + (first ? 0 : 1));
      sm.sel_need = first ? excl + c0 : incl;  // candidates down to and including that bin
    }
    __syncthreads();
  }
  const int b_sel = (int)sm.sel_digit;
  const bool fits = b_sel < kBins - 1 && sm.sel_need <= (unsigned)kCand;
  SMARK();  // 6: threshold bin
  if (fits) {
    const int top_key = (int)(__float_as_uint(bm) >> 17);
#pragma unroll 1
    for (int v = tid; v < V; v += kThreads) {
      const float q = sp[v];
      if (top_key - (int)(__float_as_uint(q) >> 17) <= b_sel) {
        const unsigned slot = atomicAdd(&sm.n_cand, 1u);
        sm.topv[slot] = q;
        sm.topi[slot] = v;
      }
    }
    __syncthreads();
  } else {
    topk_radix_cold(sp, V, kk, 0.0f, sm);
  }
  rank_order(sm);
  SMARK();  // 7: candidates compacted
  // 4. renormalise, top-p, draw: warp 0, two candidates per lane (j = lane, lane + 32)
  if (warp == 0) {
    const int j0 = lane, j1 = lane + 32;
    const float sv0 = sm.sortv[j0], sv1 = sm.sortv[j1];
    const int si0 = sm.sorti[j0], si1 = sm.sorti[j1];
    float a0 = j0 < kk ? sv0 : 0.f;
    float a1 = j1 < kk ? sv1 : 0.f;
    const int i0 = j0 < kk ? si0 : 0x7fffffff;
    const int i1 = j1 < kk ? si1 : 0x7fffffff;
    const float s1 = (float)warp_sum_d((double)a0 + (double)a1);
    int fallback = 0;
    int token = 0;
    if (s1 <= 1e-12f) {
      fallback = 1;
    } else {
      a0 = a0 / s1;
      a1 = a1 / s1;
      const float* nz = p.noise + ((size_t)b * p.steps + t) * p.noise_k;
      float r0 = 0.f, r1 = 0.f;
      int t0 = 0x7fffffff, t1 = 0x7fffffff;  // tie-break keys
      if (top_p < 1.0f) {
        // cumsum in double, rounded to float at each position (ATen CPU cumsum accumulates in
        // acc_type<float> = double); inclusive scan over lanes, first the low 32, then the high 32
        double c0 = (double)a0;
#pragma unroll 1
        for (int o = 1; o < 32; o <<= 1) {
          const double n = __shfl_up_sync(0xffffffffu, c0, o);
          if (lane >= o) c0 += n;
        }
        const double tot0 = __shfl_sync(0xffffffffu, c0, 31);
        double c1 = (double)a1;
#pragma unroll 1
        for (int o = 1; o < 32; o <<= 1) {
          const double n = __shfl_up_sync(0xffffffffu, c1, o);
          if (lane >= o) c1 += n;
        }
        c1 += tot0;
        const float cf0 = (float)c0, cf1 = (float)c1;
        // remove[j] = cum[j-1] > top_p, remove[0] = False (sampling.py:72-74)
        const float prev0 = __shfl_up_sync(0xffffffffu, cf0, 1);
        float prev1 = __shfl_up_sync(0xffffffffu, cf1, 1);
        const float last0 = __shfl_sync(0xffffffffu, cf0, 31);
        if (lane == 0) prev1 = last0;
        const bool keep0 = (lane == 0) || !(prev0 > top_p);
        const bool keep1 = !(prev1 > top_p);
        a0 = (j0 < kk && keep0) ? a0 : 0.f;
        a1 = (j1 < kk && keep1) ? a1 : 0.f;
        const float s2 = (float)warp_sum_d((double)a0 + (double)a1);
        if (s2 <= 1e-12f) {
          fallback = 1;
        } else {
          a0 = a0 / s2;
          a1 = a1 / s2;
          // multinomial == argmax(p_sorted[j] / q[j]), noise index = sorted rank (sampling.py:83-84)
          r0 = j0 < kk ? a0 / __ldg(nz + j0) : 0.f;
          r1 = j1 < kk ? a1 / __ldg(nz + j1) : 0.f;
          t0 = j0;
          t1 = j1;
        }
      } else {
        // no top-p: probs stay in vocabulary order, noise index = token id (sampling.py:88-93)
        const float s2 = (float)warp_sum_d((double)a0 + (double)a1);
        if (s2 <= 1e-12f) {
          fallback = 1;
        } else {
          a0 = a0 / s2;
          a1 = a1 / s2;
          r0 = j0 < kk ? a0 / __ldg(nz + i0) : 0.f;
          r1 = j1 < kk ? a1 / __ldg(nz + i1) : 0.f;
          t0 = i0;
          t1 = i1;
        }
      }
      if (!fallback) {
        float bv = j0 < kk ? r0 : -1.f;
        int bk = j0 < kk ? t0 : 0x7fffffff, bt = i0;
        if (j1 < kk && (r1 > bv || (r1 == bv && t1 < bk))) {
          bv = r1;
          bk = t1;
          bt = i1;
        }
#pragma unroll 1
        for (int o = 16; o > 0; o >>= 1) {
          const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
          const int ok = __shfl_xor_sync(0xffffffffu, bk, o);
          const int ot = __shfl_xor_sync(0xffffffffu, bt, o);
          if (ov > bv || (ov == bv && ok < bk)) {
            bv = ov;
            bk = ok;
            bt = ot;
          }
        }
        token = bt;
      }
    }
    if (lane == 0) {
      sm.fallback = fallback;
      sm.bc_i = token;
    }
  }
  __syncthreads();
  SMARK();  // 8: sorted, top-p, drawn
  int token = sm.bc_i;
  if (sm.fallback) token = argmax_logits_cold(sx, V, sm);
  // 5. bookkeeping: one warp (repeated_tail needs lanes 3..16)
  if (warp == 0) {
    if (lane == 0) p.sampled[(size_t)b * p.steps + t] = token;
    if (p.forced) token = p.forced[(size_t)b * p.steps + t];
    if (lane == 0) toks[t] = token;
    __syncwarp();
    const int len = hlen + 1;  // == t + 1
    // repeated_tail(hist, 16): any n in [3, min(16, len/2)] with hist[-n:] == hist[-2n:-n]
    bool rep_n = false;
    {
      const int n = lane;
      if (n >= 3 && n <= 16 && n <= len / 2) {
        rep_n = true;
        for (int i = 0; i < n; ++i) {
          const int a = (len - n + i == t) ? token : toks[len - n + i];
          const int c = toks[len - 2 * n + i];
          if (a != c) {
            rep_n = false;
            break;
          }
        }
      }
    }
    const bool any_rep = __any_sync(0xffffffffu, rep_n);
    if (lane == 0) {
      const int streak = (st.last >= 0 && token == st.last) ? st.streak + 1 : 0;
      int recovery = 0;
      if (spar.anti_loop && (any_rep || streak >= spar.loop_streak)) recovery = 1;
      const bool is_eos = token == p.eos_id;
      int done = 0;
      if (is_eos && (spar.stop_on_first_eos || len >= spar.min_gen)) done = 1;
      if (len >= p.steps) done = 1;
      UttState ns;
      ns.len = len;
      ns.last = token;
      ns.streak = streak;
      ns.recovery = recovery;
      ns.done = done;
      ns.pad[0] = ns.pad[1] = ns.pad[2] = 0;
      p.st[b] = ns;
      p.n_tokens[b] = len;
      p.done[b] = done;
      if (ll) ll_store(reinterpret_cast<float*>(p.tok_ll) + (size_t)b * 2, __uint_as_float((unsigned)token | ((unsigned)done << 30)), out_seq);
    }
  }
  SMARK();  // 9: bookkeeping
#undef SMARK
}

// ---------------------------------------------------------------------------
// Fused q projection + cached text cross-attention (nn/text.py:93-128) WITHOUT an exchange in between: rank r of a
// team serves head h = r % H for the utterances u = r / H, r / H + PH, ... (PH = P / H CTAs per head).  It computes
// q[u][h] = Wq[rows of head h] . RMSNorm_q(x[u]) itself (the head's Dh weight rows arrive through the weight ring)
// and runs the attention of its (u, h) items right away, two items side by side.  One exchange and one full GEMV
// stage fewer per attention layer than q-stage -> attention-stage.
// smem (floats): xs[MU][D] | qh[MU][Dh] | [sc | part] x 2 groups,  MU = ceil(Bt / PH)
// ---------------------------------------------------------------------------
template <typename WT, bool LL, bool TRACE>
__device__ __forceinline__ void stage_qatt(const ArParams& p, int li, const TeamCtx& tc, WeightRing& ring, int n_tiles,
                                           float* __restrict__ smem, const float* __restrict__ xsrc, unsigned x_seq,
                                           unsigned out_seq, Stamp& ts) {
  const LayerDev& L = p.layer[li];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int H = p.H, Dh = p.Dh, D = p.D, PH = p.PH;
  const int h = tc.rank % H, gi = tc.rank / H;
  const int n_my = (tc.rank < H * PH && gi < tc.nb) ? (tc.nb - gi + PH - 1) / PH : 0;
  const int MU = (p.Bt + PH - 1) / PH;
  float* xs = smem;
  float* qh = xs + (size_t)MU * D;
  if (n_my == 0) {  // no item here: only keep the weight ring in step
    ts.mark();
    ts.mark();
#pragma unroll 1
    for (int ti = n_tiles; ti > 0; --ti) {
      const TileDesc* td;
      ring.acquire(td);
      ring.release();
    }
    return;
  }
  // ---- x rows of my utterances
#pragma unroll 1
  for (int j = 0; j < n_my; ++j) {
    const int u = gi + j * PH;
    const float* src = xsrc + (size_t)(tc.b0 + u) * D * (LL ? 2 : 1);
    if (LL) {
      ll_fetch(src, D, D, x_seq, xs + (size_t)j * D);
    } else {
      for (int e = tid * 4; e < D; e += kThreads * 4) *reinterpret_cast<float4*>(xs + (size_t)j * D + e) = ldcg4(src + e);
    }
  }
  __syncthreads();
  // RMSNorm_q (nn/blocks.py:32-37), one warp per row
#pragma unroll 1
  for (int j = warp; j < n_my; j += kWarps) {
    float* d = xs + (size_t)j * D;
    float ss = 0.f;
    for (int k = lane * 4; k < D; k += 128) {
      const float4 v = *reinterpret_cast<float4*>(d + k);
      ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    }
    ss = warp_sum(ss);
    const float inv = 1.0f / sqrtf(ss / (float)D + 1e-6f);
    for (int k = lane * 4; k < D; k += 128) {
      float4 v = *reinterpret_cast<float4*>(d + k);
      const float4 w = __ldg(reinterpret_cast<const float4*>(L.nq_w + k));
      v.x = (v.x * inv) * w.x;
      v.y = (v.y * inv) * w.y;
      v.z = (v.z * inv) * w.z;
      v.w = (v.w * inv) * w.w;
      *reinterpret_cast<float4*>(d + k) = v;
    }
  }
  __syncthreads();
  ts.mark();  // activations staged
  // ---- q rows of my head: 8 rows x 2 utterances per warp task
  const unsigned xs_s = smem_u32(xs);
  const unsigned row_bytes = (unsigned)D * (unsigned)sizeof(WT);
  const int n_up = (n_my + 1) / 2;
#pragma unroll 1
  for (int ti = n_tiles; ti > 0; --ti) {
    const TileDesc* td;
    const unsigned wb = ring.acquire(td);
    const int nr = td->nrows;
    const int n_rt = (nr + 7) / 8;
#pragma unroll 1
    for (int task = warp; task < n_rt * n_up; task += kWarps) {
      const int rt = n_up == 1 ? task : task / n_up;
      const int up = task - rt * n_up;
      unsigned wr[8];
#pragma unroll
      for (int jr = 0; jr < 8; ++jr) wr[jr] = wb + (unsigned)min(rt * 8 + jr, nr - 1) * row_bytes;
      const int j0 = min(up * 2, max(n_my - 2, 0));
      const float v = warp_rows_s<8, 2, WT>(wr, xs_s + (unsigned)j0 * (unsigned)D * 4u, D, lane);
      const int o = (lane >> 1) & 15;  // after the transposed reduction: output o = row i * 2 + utterance uu
      const int i = o >> 1, uu = o & 1;
      const int ri = rt * 8 + i, j = j0 + uu;
      if ((lane & 1) == 0 && ri < nr && j >= up * 2 && j < n_my) qh[(size_t)j * Dh + (td->row0 - h * Dh) + ri] = v;
    }
    ring.release();
  }
  ts.mark();  // tiles done
  // ---- the attention of my items, two side by side
  {
    const int grp = tid / kAttGroup, gt = tid - grp * kAttGroup;
    float* sc = qh + (size_t)MU * Dh + (size_t)grp * att_group_floats(p.Lmax, Dh);
    float* part = sc + ((p.Lmax + 3) & ~3);
#pragma unroll 1
    for (int j = grp; j < n_my; j += 2) {
      const int u = gi + j * PH;
      attention_item<TRACE>(p, L, tc.b0 + u, h, qh + (size_t)j * Dh, sc, part, grp, gt, LL ? 1 : 0, out_seq);
    }
  }
}

// ---------------------------------------------------------------------------
// the persistent kernel: an interpreter over p.prog with one shared GEMV body
// ---------------------------------------------------------------------------
template <typename WT, int TU, bool LL, bool TRACE = false>
__global__ void __launch_bounds__(kThreads, 1) ar_persistent_kernel(const __grid_constant__ ArParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ SamplerSmem ssm;
  __shared__ __align__(8) unsigned long long wbars[kMaxWBuf];
  __shared__ unsigned char stage_tiles[kMaxStages];
  __shared__ int conv_phase[kMaxLayers], conv_slot[kMaxLayers];
  __shared__ int s_tok[kMaxUttPerTeam], s_done[kMaxUttPerTeam];
  constexpr int EL = LL ? 2 : 1;  // floats per activation element in the exchange buffers
  // dynamic shared memory [act | p.ring_off: ring | p.table_off: table] from a 1024-byte aligned base, so that no address
  // in the map depends on the static shared memory in front of it (the bulk copies into the ring need 16-byte alignment)
  unsigned char* const smem_base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  float* act = reinterpret_cast<float*>(smem_base);  // [nb][max(D,F)] (or 2 x [nb][D] + tap scratch)
  TeamCtx tc;
  tc.team = blockIdx.x / p.P;
  tc.rank = blockIdx.x % p.P;
  tc.P = p.P;
  if (tc.team >= p.g) return;
  tc.b0 = tc.team * p.Bt;
  tc.nb = min(p.Bt, p.B - tc.b0);
  if (tc.nb <= 0) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned* bar = p.barrier + (size_t)tc.team * 32;
  unsigned epoch = 0;
  const int D = p.D, F = p.F;
  const unsigned act_s = smem_u32(act);
  float* xraw = act + (size_t)tc.nb * D;  // second [nb][D] buffer (GLU stage only)
  const unsigned scratch_s = act_s + (unsigned)(2 * tc.nb * D) * 4u;  // GLU stage: dwconv tap rows
  // ---- weight ring: [act region][nbuf x wbuf][tile table]
  WeightRing ring;
  {
    TileDesc* tab = reinterpret_cast<TileDesc*>(smem_base + p.table_off);
    const int nt = p.n_tiles[tc.rank];
    const TileDesc* gt = p.tiles + (size_t)tc.rank * kMaxTilesPerStep;
    for (int i = threadIdx.x; i < nt; i += kThreads) tab[i] = gt[i];
    for (int i = threadIdx.x; i < p.n_stage; i += kThreads) stage_tiles[i] = p.stage_tiles[(size_t)tc.rank * kMaxStages + i];
    if (threadIdx.x == 0) {
      for (int i = 0; i < p.nbuf; ++i) mbar_init(&wbars[i], 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    ring.bars = wbars;
    ring.base = smem_u32(smem_base + p.ring_off);
    ring.wbuf = (unsigned)p.wbuf_bytes;
    ring.nbuf = p.nbuf;
    ring.table = tab;
    ring.n_tiles = nt;
    ring.start((p.t_end - p.t_begin) * nt);
  }

#pragma unroll 1
  for (int t = p.t_begin; t < p.t_end; ++t) {
    const unsigned seq0 = p.seq_base + (unsigned)((t - p.t_begin) * p.n_stage);  // stage si writes flag seq0 + si + 1
    // ---- previous tokens + done flags of the team; team-uniform early exit when every utterance finished
    if (threadIdx.x < tc.nb) {
      const int b = tc.b0 + threadIdx.x;
      int tok = 0, dn = 0;
      if (LL && t > p.t_begin) {
        uint2 w;
        do {
          w = ll_load1(reinterpret_cast<const float*>(p.tok_ll) + (size_t)b * 2);
        } while (w.y != seq0);  // written by the SAMPLE stage of step t-1 (its flag is seq0)
        tok = (int)(w.x & 0x3fffffffu);
        dn = (int)(w.x >> 30);
      } else {
        dn = __ldcg(&p.st[b].done);
        tok = (t == 0) ? 0 : __ldcg(&p.tokens[(size_t)b * p.steps + t - 1]);
      }
      s_tok[threadIdx.x] = tok;
      s_done[threadIdx.x] = dn;
    }
    if (TRACE && threadIdx.x == 0) g_attn_step = t % p.attn_ring;
    if (threadIdx.x < p.n_layers) {  // the only integer divisions of the step: one thread per layer
      const int dl = p.layer[threadIdx.x].dil;
      conv_phase[threadIdx.x] = t % dl;
      conv_slot[threadIdx.x] = (t / dl) % p.Kc;
    }
    __syncthreads();
    {
      int live = 0;
      for (int u = 0; u < tc.nb; ++u) live |= (s_done[u] == 0);
      if (!live) break;
    }
    float* cur = p.xa;
    float* nxt = p.xb;
    unsigned x_seq = 0;  // flag of the last full write of `cur`
    Stamp ts;
    ts.buf = (p.timing && t == p.timing_step && threadIdx.x == 0) ? p.timing + (size_t)blockIdx.x * kTimingSlots : nullptr;
    ts.n = 0;
    ts.mark();
#pragma unroll 1
    for (int si = 0; si < p.n_stage; ++si) {
      const int kind = p.prog[si].kind, li = p.prog[si].layer;
      const unsigned seq = seq0 + (unsigned)si + 1u;  // flag written by this stage
      if (kind <= K_HEAD) {
        const LayerDev& L = p.layer[li];
        // ---- decode the stage: y[N] = W[N][K] . act, epilogue by kind
        int N = D, K = D, ld_dst = D;
        const float* src = cur;
        unsigned src_seq = x_seq;
        const float* norm_w = nullptr;
        float* dst = cur;
        float* trace = nullptr;
        float scale = 0.f;
        if (kind == K_GLU) {          // x -> RMSNorm -> GLU -> dwconv -> + x  (nn/blocks.py:156-160)
          norm_w = L.norm_w;
          dst = nxt;
          if (li == 0) src = nullptr;
        } else if (kind == K_FFN1) {  // RMSNorm -> W1 + b1 -> GELU          (nn/blocks.py:129-131)
          norm_w = L.ffn_norm_w;
          N = F;
          dst = p.hbuf;
          ld_dst = F;
        } else if (kind == K_FFN2) {  // W2 + b2 -> + x (in place, own slice) (nn/blocks.py:132,161)
          src = p.hbuf;
          src_seq = seq - 1;
          K = F;
          if (p.trace_blocks && !L.has_attn) trace = p.trace_blocks + (((size_t)t * p.n_layers + li) * p.B) * D;
        } else if (kind == K_Q) {     // q = Wq . RMSNorm_q(x)                (nn/text.py:93-94)
          norm_w = L.nq_w;
          dst = p.qbuf;
        } else if (kind == K_O) {     // x += tanh(gate) * Wo . a            (nn/text.py:129-131)
          src = p.abuf;
          src_seq = seq - 1;
          scale = L.gate_tanh;
          if (p.trace_blocks) trace = p.trace_blocks + (((size_t)t * p.n_layers + li) * p.B) * D;
        } else {                      // logits = Wh . RMSNorm(x) + bh       (nn/generator.py:127-128)
          norm_w = p.final_norm_w;
          N = p.V;
          dst = p.logits;
          ld_dst = p.Vpad;
          if (p.trace_logits) trace = p.trace_logits + ((size_t)t * p.B) * p.V;
        }
        // ---- stage the activations
        if (src == nullptr) {  // layer 0: x = cond_ar[:, t] + emb(prev token | BOS)  (model.py:266-272)
          // cond row -> act, embedding row -> xraw (cp.async, all loads in flight together), then add
          for (int u = warp; u < tc.nb; u += kWarps) {
            const int b = tc.b0 + u;
            const float* cr = p.cond + ((size_t)b * p.steps + t) * D;
            for (int k = lane * 4; k < D; k += 128) cp_async16(act_s + (unsigned)(u * D + k) * 4u, cr + k);
            const int row = (t == 0) ? p.V : s_tok[u];
            const float* er = p.emb + (size_t)row * D;
            for (int k = lane * 4; k < D; k += 128) cp_async16(act_s + (unsigned)((tc.nb + u) * D + k) * 4u, er + k);
          }
          cp_async_commit();
          cp_async_wait0();
          __syncwarp();
          for (int u = warp; u < tc.nb; u += kWarps) {
            for (int k = lane * 4; k < D; k += 128) {
              const float4 c = *reinterpret_cast<float4*>(act + (size_t)u * D + k);
              const float4 e = *reinterpret_cast<float4*>(xraw + (size_t)u * D + k);
              const float4 x = make_float4(c.x + e.x, c.y + e.y, c.z + e.z, c.w + e.w);
              *reinterpret_cast<float4*>(act + (size_t)u * D + k) = x;
              *reinterpret_cast<float4*>(xraw + (size_t)u * D + k) = x;
            }
          }
          __syncwarp();
        }
        stage_rows<LL>(src ? src + (size_t)tc.b0 * K * EL : nullptr, tc.nb, K, act, norm_w,
                       (kind == K_GLU && src) ? xraw : nullptr, src_seq);
        __syncthreads();
        ts.mark();  // activations staged
        // ---- this CTA's rows, tile by tile from the weight ring
        const bool glu = kind == K_GLU;
        const unsigned row_bytes = (unsigned)K * (unsigned)sizeof(WT);
        float* state = p.ring + L.ring_off;
        const int dil = L.dil;
        const int phase = conv_phase[li], slot_now = conv_slot[li];
        // a task = R weight rows x tue utterances (tue = TU, or TU / 2 for a narrow stage); GLU: R/2 channels (value
        // rows, then their gate rows).  Only the K loop and its reduction are compiled once per shape.
        constexpr int R = (TU == 8) ? 4 : 2;
        constexpr int RC = R / 2;
        constexpr int TUN = TU >= 2 ? TU / 2 : TU;  // the TU = 1 instantiation has one shape
        const bool narrow = TUN != TU && p.prog[si].shape == SHAPE_NARROW;
        const int lg_tue = narrow ? ilog2(TUN) : ilog2(TU);
        const int tue = 1 << lg_tue;
        const int sh = 5 - ilog2(R) - lg_tue;  // after the transposed reduction lane L owns output (L >> sh) & (R*tue-1)
        const int n_ut = (tc.nb + tue - 1) >> lg_tue;
#pragma unroll 1
      for (int ti = stage_tiles[si]; ti > 0; --ti) {
        const TileDesc* td;
        const unsigned wb = ring.acquire(td);
        const int nr = td->nrows;
        const int n_rt = glu ? (nr + RC - 1) / RC : (nr + R - 1) / R;
        const unsigned epi_s = wb + td->bytes0 + td->bytes1;
#pragma unroll 1
        for (int task = warp; task < n_rt * n_ut; task += kWarps) {
          const int rt = n_ut == 1 ? task : (int)((unsigned)task / (unsigned)n_ut);
          const int u0 = (task - rt * n_ut) << lg_tue;
          unsigned wr[R];
#pragma unroll
          for (int jr = 0; jr < R; ++jr) {
            if (glu) {
              const int ch = min(rt * RC + (jr % RC), nr - 1);
              wr[jr] = wb + (jr < RC ? 0u : td->bytes0) + (unsigned)ch * row_bytes;
            } else {
              wr[jr] = wb + (unsigned)min(rt * R + jr, nr - 1) * row_bytes;
            }
          }
          const int ub = min(u0, max(tc.nb - tue, 0));
          const int o = (lane >> sh) & ((R << lg_tue) - 1);  // = i*tue + uu
          const int i = o >> lg_tue, uu = o & (tue - 1);
          const bool writer = (lane & ((1 << sh) - 1)) == 0;
          const int ri = glu ? rt * RC + i : rt * R + i;
          const int u = ub + uu;
          const bool mine = writer && (glu ? i < RC : true) && ri < nr && u >= u0 && u < tc.nb;
          const int r = td->row0 + ri;  // output feature (GLU: channel)
          const int b = tc.b0 + (mine ? u : 0);
          float* d = dst + ((size_t)b * ld_dst + (mine ? r : td->row0)) * EL;
          // operands of the epilogue are requested before the K loop: their latency hides under it
          float res_v = 0.f;
          float* rb = nullptr;
          // one tap row per (channel of the task, utterance): kTapSlots = 16 rows per warp (RC <= 2 channels x tue <= 8)
          const unsigned tap_w = scratch_s + (unsigned)warp * (unsigned)(kTapSlots * p.KcP * 4) +
                                 (unsigned)((i % RC) * tue + uu) * (unsigned)(p.KcP * 4);
          if (glu) {
            // conv state row of (utterance, channel, phase): [KcP] floats, see DESIGN.md §2
            rb = state + (((size_t)b * D + (mine ? r : td->row0)) * dil + phase) * p.KcP;
            if (mine)
              for (int q = 0; q < p.KcP; q += 4) cp_async16(tap_w + (unsigned)q * 4u, rb + q);
          } else if (mine && (kind == K_FFN2 || kind == K_O)) {
            res_v = ldcg1(d);  // own slice: written by this CTA at an earlier stage (value word)
          }
          cp_async_commit();
          const unsigned xa = act_s + (unsigned)ub * (unsigned)K * 4u;
          float v = narrow ? warp_rows_s<R, TUN, WT, 1>(wr, xa, K, lane) : warp_rows_s<R, TU, WT>(wr, xa, K, lane);
          // GLU: the gate total of (channel i, utterance uu) lives in the lanes of output (RC + i)*tue + uu
          const float gate_v = __shfl_sync(0xffffffffu, v, (((RC + (i % RC)) * tue + uu) << sh) & 31);
          cp_async_wait0();
          if (mine) {
            if (glu) {
              const int Kc = p.Kc;
              const unsigned er = epi_s + (unsigned)(ri * p.KcE) * 4u;  // [w0..w(Kc-1), dw_b, b_value, b_gate]
              const float a = v + lds32(er + (unsigned)(Kc + 1) * 4u);
              const float gt = gate_v + lds32(er + (unsigned)(Kc + 2) * 4u);
              const float h = a * sigmoid_ref(gt);
              rb[slot_now] = h;  // slot (t / dil) mod Kc of frame t inside its phase
              float y = 0.f;
              int pos = slot_now + 1;  // oldest tap: frame t - (Kc-1)*dil
#pragma unroll 1
              for (int j = 0; j < Kc - 1; ++j) {
                if (pos == Kc) pos = 0;
                y += lds32(tap_w + (unsigned)pos * 4u) * lds32(er + (unsigned)j * 4u);
                ++pos;
              }
              y += h * lds32(er + (unsigned)(Kc - 1) * 4u);
              y += lds32(er + (unsigned)Kc * 4u);
              v = xraw[(size_t)u * D + r] + y;
            } else {
              const float bias_v = (kind == K_Q || kind == K_O) ? 0.f : lds32(epi_s + (unsigned)(td->off2 + ri) * 4u);
              if (kind == K_FFN1) {
                v = gelu_erf(v + bias_v);
              } else if (kind == K_FFN2) {
                v = res_v + (v + bias_v);
                if (trace) trace[(size_t)b * D + r] = v;
              } else if (kind == K_O) {
                v = res_v + scale * v;
                if (trace) trace[(size_t)b * D + r] = v;
              } else if (kind == K_HEAD) {
                v += bias_v;
                if (trace) trace[(size_t)b * p.V + r] = v;
              }
            }
            if (LL) ll_store(d, v, seq);
            else *d = v;
          }
          __syncwarp();  // the tap scratch is reused by the next task of this warp
        }
        ring.release();
      }
        ts.mark();  // tiles done
        if (glu) {
          float* tmp = cur;
          cur = nxt;
          nxt = tmp;
        }
        if (kind == K_GLU || kind == K_FFN2 || kind == K_O) x_seq = seq;
      } else if (kind == K_QATT) {
        stage_qatt<WT, LL, TRACE>(p, li, tc, ring, stage_tiles[si], act, cur, x_seq, seq, ts);
      } else if (kind == K_ATT) {
        ts.mark();
        ts.mark();
        stage_attention<TRACE>(p, li, tc.rank, tc.P, tc.b0, tc.nb, act, LL ? 1 : 0, seq - 1, seq);
      } else {  // K_SAMPLE: utterances round-robin over the team's CTAs
        ts.mark();
        ts.mark();
        float* sx = act;
        float* sp = act + p.Vpad;
        unsigned char* flags = reinterpret_cast<unsigned char*>(act + 2 * p.Vpad);
        // samplers run on the team's LAST ranks, attention items on the first ones: at small batch no CTA
        // has to keep both code paths in its instruction cache
        for (int u = tc.P - 1 - tc.rank; u < tc.nb; u += tc.P) {
          sample_utterance(p, tc.b0 + u, t, sx, sp, flags, ssm, LL ? 1 : 0, seq - 1, seq);
          __syncthreads();
        }
      }
      if (LL) {
        __syncthreads();  // shared-memory reuse between stages (no team barrier in LL mode)
        ts.mark();
        ts.mark();
        ts.mark();
      } else {
        team_barrier(bar, tc.P, epoch, ts);
      }
    }
  }
  ring.drain();  // early team exit: prefetched tiles must land before the CTA exits
}

// ---------------------------------------------------------------------------
// text K/V cache builder (nn/text.py:75-83): K,V = W . RMSNorm_kv(txt) -> [slot][B][H][Lmax][Dh]
// grid = (ceil(Lmax/16), B, n_attn)
// ---------------------------------------------------------------------------
struct KvParams {
  int D, H, Dh, B, Lmax, text_stride, n_attn;
  const float* txt;  // [B][text_stride][D]
  const int* text_len;
  const float* nkv_w[kMaxLayers];
  const void* wk[kMaxLayers];
  const void* wv[kMaxLayers];
  float* kc;
  float* vc;
};

template <typename WT>
__global__ void __launch_bounds__(kThreads, 1) kv_build_kernel(const __grid_constant__ KvParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* act = reinterpret_cast<float*>(smem_raw);  // [16][D]
  constexpr int TL = 16, TU = 8;
  const int l0 = blockIdx.x * TL, b = blockIdx.y, slot = blockIdx.z;
  const int len = p.text_len[b];
  if (l0 >= len) return;
  const int nl = min(TL, len - l0);
  const int D = p.D;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // positions beyond nl: zeros, so the tiles stay in-bounds
  for (int i = threadIdx.x; i < TL * D; i += kThreads) act[i] = 0.f;
  __syncthreads();
  stage_rows(p.txt + ((size_t)b * p.text_stride + l0) * D, nl, D, act, p.nkv_w[slot], nullptr);
  __syncthreads();
  const WT* Wk = reinterpret_cast<const WT*>(p.wk[slot]);
  const WT* Wv = reinterpret_cast<const WT*>(p.wv[slot]);
  const int n_rt = (2 * D) / 2, n_ut = TL / TU;
  for (int task = warp; task < n_rt * n_ut; task += kWarps) {
    const int r0 = (task / n_ut) * 2, u0 = (task % n_ut) * TU;
    if (u0 >= nl) continue;
    const WT* w0 = (r0 < D) ? Wk + (size_t)r0 * D : Wv + (size_t)(r0 - D) * D;
    const WT* w1 = (r0 + 1 < D) ? Wk + (size_t)(r0 + 1) * D : Wv + (size_t)(r0 + 1 - D) * D;
    float out[2][TU];
    warp_rows_g<TU, WT>(w0, w1, act + (size_t)u0 * D, D, lane, out);
    const int i = lane / TU, uu = lane % TU;
    const int r = r0 + i, l = u0 + uu;
    if (lane < 2 * TU && l < nl) {
      const float v = pick2<TU>(out, i, uu);
      const int rr = r < D ? r : r - D;
      const int h = rr / p.Dh, dh = rr % p.Dh;
      float* dst = (r < D ? p.kc : p.vc) + ((((size_t)slot * p.B + b) * p.H + h) * p.Lmax + (l0 + l)) * p.Dh + dh;
      *dst = v;
    }
  }
}

}  // namespace sopro
