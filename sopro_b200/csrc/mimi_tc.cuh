// wgmma / TMA implicit GEMM for the Mimi decoder's dense blocks (sm_90a).
//
//   C[b][m][n] = epi( sum_{j<taps} sum_{ci<Cin} X[b][m + j*dil - pad][ci] * W[n][j*Cin + ci] + bias[n % bias_mod] )
//
// X is a channel-last bf16 activation [B][Min][Cin] (already passed through ELU by its producer when
// the layer wants ELU(x)), W is a bf16 weight matrix [N][K] (K = taps*Cin, K-major), accumulation is
// fp32 in registers.  This covers Linear, the causal Conv1d and the causal ConvTranspose1d of
// transformers' modeling_mimi.py (:331-351, :402-409) exactly as mimi_engine.cu's fp32 path does.
//
// One CTA computes one 128 x BN tile:
//   warp 8      TMA producer: per K chunk one 3-D box of X (rows shifted by the tap; rows outside
//               [0, Min) are zero-filled by the TMA unit == the causal left pad) and one 2-D box of W,
//               both landing swizzled in a ring of shared-memory stages, completion on mbarriers
//   warps 0-7   two consumer warpgroups, 64 tile rows each: wgmma (M=64, N=BN, K=16) from shared-memory
//               descriptors, one chunk in flight while the previous one's stage goes back to the producer;
//               then the accumulators go through the idle stage memory so that the epilogue (bias / GELU /
//               LayerScale-residual / skip, fp32 and/or bf16 out, optionally ELU'd: the next layer's operand)
//               reads and writes whole rows with 16-byte accesses
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>
#include <cstdlib>

#include "wgmma.cuh"

namespace tc {

enum { EPI_NONE = 0, EPI_GELU = 1, EPI_RES_SCALE = 2, EPI_RES = 3 };

struct TcOp {
  const float* bias;   // [bias_mod] or null
  const float* R;      // residual fp32 [B][M][N] or null
  const float* scale;  // LayerScale [N] or null
  float* out_f32;      // [B][M][N] or null
  __nv_bfloat16* out_bf16;  // [B][M][N] or null
  long long c_bs;      // batch stride of the outputs (elements)
  long long r_bs;      // batch stride of R (elements; 0 = c_bs)
  long long a_pitch;   // rows per batch item of X (0 = Min: items packed back to back)
  int M, N, K, Cin, dil, pad, bias_mod, epi, out_elu;
  int stages;          // filled in by launch()
  int tap_col[8];      // A column offset of tap j (0 everywhere for convolutions; the NAR refiner's exact three-way bf16 split
                       // pairs W's K block j with the A term it multiplies: taps over COLUMN groups of the same rows, dil = 0)
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "W_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@!p bra W_%=;\n"
      "}\n" ::"r"(bar),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* tm, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(tm)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* tm, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(tm)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// barrier of the 128 threads of one warpgroup (ids 1, 2: 0 is __syncthreads')
__device__ __forceinline__ void wg_sync(int g) { asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory"); }

__device__ __forceinline__ float elu1(float x) { return x > 0.f ? x : expm1f(x); }
// ELU whose result is rounded to bf16 right away: exp(x) - 1 with the fast exponential has an ABSOLUTE error of a few
// 1e-7 (fp32 ulps of 1; the subtraction cancels for small |x|).  That is below half a bf16 ulp of the result only for
// |x| above about 1e-4; for smaller negative x the bf16 result can be many of its own ulps off (11 at x = -1e-6,
// ~100 at -1e-7, against a correctly rounded exp), while staying ~1e-7 from the exact value.  Checks of ELU'd bf16
// outputs therefore need an absolute floor relative to the tensor's scale, not a per-element ulp bound.
__device__ __forceinline__ float elu_fast(float x) { return x > 0.f ? x : __expf(x) - 1.0f; }
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}

constexpr int kBM = 128, kBK = 64;
constexpr int kGemmThreads = 288;  // two consumer warpgroups (64 tile rows each) + one TMA producer warp
constexpr int kProducerWarp = 8;
template <int BN, int BK>
struct TileCfg {
  static constexpr int kMaxStages = BN >= 128 ? 3 : 4;
  static constexpr int kABytes = kBM * BK * 2;  // 16 KB at BK = 64
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kEpiPitch = BN + 8;                    // floats per row of the epilogue tile (conflict-free fragment stores)
  static constexpr int kEpiBytes = kBM * kEpiPitch * 4;       // the 128 x BN fp32 tile, over the stages once they are idle
  static constexpr int smem(int stages) { return (stages * kStageBytes > kEpiBytes ? stages * kStageBytes : kEpiBytes) + 1024; }
};

template <int BN, int BK>
__global__ void __launch_bounds__(kGemmThreads, BN >= 128 ? 1 : 2) igemm_tc_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                                   const __grid_constant__ CUtensorMap tmW, const TcOp op) {
  using Cfg = TileCfg<BN, BK>;
  constexpr int SM = Cfg::kMaxStages;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bars[2 * SM];
  const uint32_t tiles = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t full0 = smem_u32(&bars[0]), empty0 = smem_u32(&bars[SM]);
  const int S = op.stages;  // min(kMaxStages, K chunks): short-K layers take less shared memory -> more CTAs per SM
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * kBM, n0 = blockIdx.y * BN, b = blockIdx.z;
  const int nk = op.K / BK;

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, 2);  // one arrival per consumer warpgroup
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == kProducerWarp) {
    if (lane == 0) {
      for (int kc = 0; kc < nk; ++kc) {
        const int s = kc % S;
        const uint32_t ph = (uint32_t)(kc / S) & 1u;
        mbar_wait(empty0 + 8 * s, ph ^ 1u);
        mbar_expect_tx(full0 + 8 * s, Cfg::kStageBytes);
        const int k0 = kc * BK;
        const int j = k0 / op.Cin, ci = k0 - j * op.Cin;
        const uint32_t sa = tiles + s * Cfg::kStageBytes;
        tma_load_3d(sa, &tmA, full0 + 8 * s, ci + op.tap_col[j & 7], m0 + j * op.dil - op.pad, b);
        tma_load_2d(sa + Cfg::kABytes, &tmW, full0 + 8 * s, k0, n0);
      }
    }
    return;
  }
  const int g = warp >> 2;  // consumer warpgroup: tile rows 64g .. 64g + 63
  float d[BN / 2];
#pragma unroll 1
  for (int kc = 0; kc < nk; ++kc) {
    const int s = kc % S;
    mbar_wait(full0 + 8 * s, (uint32_t)(kc / S) & 1u);
    const uint32_t sa = tiles + s * Cfg::kStageBytes;
    const uint64_t da = wg::desc_k<BK>(sa + (uint32_t)g * (64u * BK * 2u)), db = wg::desc_k<BK>(sa + Cfg::kABytes);
    wg::fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k)  // +32 B per K=16 slice inside the swizzle atom
      wg::mma_ss<BN>(d, da + 2 * k, db + 2 * k, (kc | k) != 0);
    wg::commit();
    wg::wait<1>();  // chunk kc - 1 has completed: its stage goes back to the producer
    if (kc > 0 && (threadIdx.x & 127) == 0) mbar_arrive(empty0 + 8 * ((kc - 1) % S));
  }
  wg::wait<0>();
  wg::fence_regs(d);
  // ---- epilogue: both warpgroups are done with every stage -> the fp32 tile goes to shared memory, then each warp
  // handles whole rows (4 consecutive columns per thread)
  asm volatile("bar.sync 1, 256;" ::: "memory");
  float* et = reinterpret_cast<float*>(smem_raw + (tiles - smem_u32(smem_raw)));
  {
    const int r0 = 64 * g + 16 * (warp & 3) + (lane >> 2);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h)
        *reinterpret_cast<float2*>(et + (r0 + 8 * h) * Cfg::kEpiPitch + 8 * j + 2 * (lane & 3)) = make_float2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");
  constexpr int TPR = BN / 4, RPP = 256 / TPR;  // threads per row, rows per pass
  const int t = threadIdx.x, c = 4 * (t % TPR), n = n0 + c;
#pragma unroll 1
  for (int r = t / TPR; r < kBM; r += RPP) {
    const int m = m0 + r;
    if (m >= op.M) break;
    const size_t row = (size_t)b * (size_t)op.c_bs + (size_t)m * op.N;
    float4 v = *reinterpret_cast<const float4*>(et + r * Cfg::kEpiPitch + c);
    if (op.bias) {
      const float4 bv = __ldg(reinterpret_cast<const float4*>(op.bias + n % op.bias_mod));  // bias_mod is a multiple of 4
      v.x += bv.x;
      v.y += bv.y;
      v.z += bv.z;
      v.w += bv.w;
    }
    if (op.epi == EPI_GELU) {
      v = make_float4(gelu_erf(v.x), gelu_erf(v.y), gelu_erf(v.z), gelu_erf(v.w));
    } else if (op.epi == EPI_RES_SCALE || op.epi == EPI_RES) {
      const float4 rv = *reinterpret_cast<const float4*>(op.R + (size_t)b * (size_t)op.r_bs + (size_t)m * op.N + n);  // may alias out_f32
      if (op.epi == EPI_RES_SCALE) {
        const float4 sv = __ldg(reinterpret_cast<const float4*>(op.scale + n));
        v = make_float4(fmaf(sv.x, v.x, rv.x), fmaf(sv.y, v.y, rv.y), fmaf(sv.z, v.z, rv.z), fmaf(sv.w, v.w, rv.w));
      } else {
        v = make_float4(v.x + rv.x, v.y + rv.y, v.z + rv.z, v.w + rv.w);
      }
    }
    if (op.out_f32) *reinterpret_cast<float4*>(op.out_f32 + row + n) = v;
    if (op.out_bf16) {
      if (op.out_elu) v = make_float4(elu_fast(v.x), elu_fast(v.y), elu_fast(v.z), elu_fast(v.w));
      *reinterpret_cast<uint2*>(op.out_bf16 + row + n) = make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w));
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Fused ResnetBlock (MimiResnetBlock, modeling_mimi.py:437-451): out = z + conv1x1(ELU(conv3(ELU(z)))).
//   GEMM 1: h[128 x HID] = conv k=3 of the bf16 ELU(z) rows (3-D TMA boxes per tap), accumulators in registers
//   epilogue A: + bias, ELU, round to bf16, written swizzled into shared memory as the next A operand (each
//           warpgroup writes the 64 rows its own GEMM 2 reads)
//   GEMM 2: [128 x 2*HID] = h . W2^T (W2 loaded once per CTA), in column blocks of <= 128
//   epilogue B: through the idle stage memory (whole rows, 16-byte accesses): + bias + z (fp32 skip, read once),
//           then fp32 and/or bf16(ELU) out
// The hidden activation never touches HBM and one launch replaces two.  HID in {32, 64, 128}.
// ---------------------------------------------------------------------------------------------
struct ResOp {
  const float* bias1;  // [HID]
  const float* bias2;  // [2*HID]
  const float* Z;      // fp32 skip [B][M][2*HID], item b at Z + b * z_bs
  float* out_f32;      // [B][M][2*HID] or null, item b at b * o_bs
  __nv_bfloat16* out_bf16;  // [B][M][2*HID] or null, through ELU when out_elu
  int M, taps, pad, out_elu, stages;
  int Min;  // rows of the bf16 input X (0 = M; streaming: M + taps - 1 with pad = 0, the context rows in front)
  long long a_pitch;     // rows per batch item of X (0 = Min)
  long long z_bs, o_bs;  // batch strides of Z and of the outputs (elements; 0 = M * 2*HID)
};

template <int HID>
struct ResCfg {
  static constexpr int kCout = 2 * HID;
  static constexpr int kBKH = HID < 64 ? HID : 64;       // K chunk of the second GEMM
  static constexpr int kNK2 = HID / kBKH;
  static constexpr int kN2 = kCout < 128 ? kCout : 128;  // column block of the second GEMM
  static constexpr int kMaxStages = 3;
  static constexpr int kABytes = kBM * kBK * 2;           // 16 KB
  static constexpr int kBBytes = HID * kBK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kHBytes = kBM * HID * 2;           // hidden activation as the A operand of GEMM 2
  static constexpr int kW2Bytes = kCout * HID * 2;
  static constexpr int kEpiPitch = kN2 + 8;                  // floats per row of the epilogue tile
  static constexpr int kEpiBytes = kBM * kEpiPitch * 4;
  // the stage ring, which also holds the epilogue tile of GEMM 2 once GEMM 1 is done
  static constexpr int ring(int stages) { return stages * kStageBytes > kEpiBytes ? stages * kStageBytes : kEpiBytes; }
  static constexpr int smem(int stages) { return ring(stages) + kHBytes + kW2Bytes + 1024; }
};

template <int HID>
__global__ void __launch_bounds__(kGemmThreads, HID <= 64 ? 2 : 1) resblock_tc_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                                      const __grid_constant__ CUtensorMap tmW1,
                                                                                      const __grid_constant__ CUtensorMap tmW2,
                                                                                      const ResOp op) {
  using Cfg = ResCfg<HID>;
  constexpr int SM = Cfg::kMaxStages, COUT = Cfg::kCout, BKH = Cfg::kBKH, N2 = Cfg::kN2;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bars[2 * SM + 1];
  const int S = op.stages;
  const uint32_t tiles = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sH = tiles + Cfg::ring(S), sW2 = sH + Cfg::kHBytes;
  const uint32_t full0 = smem_u32(&bars[0]), empty0 = smem_u32(&bars[SM]), w2_full = smem_u32(&bars[2 * SM]);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * kBM, b = blockIdx.y;
  const int nk = op.taps * COUT / kBK;  // K chunks of GEMM 1 (COUT is a multiple of 64)

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, 2);
    }
    mbar_init(w2_full, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == kProducerWarp) {
    if (lane == 0) {
      mbar_expect_tx(w2_full, Cfg::kW2Bytes);
      for (int c = 0; c < Cfg::kNK2; ++c) tma_load_2d(sW2 + c * (COUT * BKH * 2), &tmW2, w2_full, c * BKH, 0);
      for (int kc = 0; kc < nk; ++kc) {
        const int s = kc % S;
        const uint32_t ph = (uint32_t)(kc / S) & 1u;
        mbar_wait(empty0 + 8 * s, ph ^ 1u);
        mbar_expect_tx(full0 + 8 * s, Cfg::kStageBytes);
        const int k0 = kc * kBK;
        const int j = k0 / COUT, ci = k0 - j * COUT;
        const uint32_t sa = tiles + s * Cfg::kStageBytes;
        tma_load_3d(sa, &tmA, full0 + 8 * s, ci, m0 + j - op.pad, b);
        tma_load_2d(sa + Cfg::kABytes, &tmW1, full0 + 8 * s, k0, 0);
      }
    }
    return;
  }
  const int g = warp >> 2;
  const int r0 = 64 * g + 16 * (warp & 3) + (lane >> 2);  // tile rows r0 and r0 + 8
  // ---- GEMM 1
  {
    float d[HID / 2];
#pragma unroll 1
    for (int kc = 0; kc < nk; ++kc) {
      const int s = kc % S;
      mbar_wait(full0 + 8 * s, (uint32_t)(kc / S) & 1u);
      const uint32_t sa = tiles + s * Cfg::kStageBytes;
      const uint64_t da = wg::desc_sw128(sa + (uint32_t)g * (64u * kBK * 2u)), db = wg::desc_sw128(sa + Cfg::kABytes);
      wg::fence();
#pragma unroll
      for (int k = 0; k < kBK / 16; ++k) wg::mma_ss<HID>(d, da + 2 * k, db + 2 * k, (kc | k) != 0);
      wg::commit();
      wg::wait<1>();
      if (kc > 0 && (threadIdx.x & 127) == 0) mbar_arrive(empty0 + 8 * ((kc - 1) % S));
    }
    wg::wait<0>();
    wg::fence_regs(d);
    // ---- epilogue A: hidden activation -> shared memory (bf16, swizzled K-major rows of BKH elements)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = r0 + 8 * h;
      const int sw = BKH == 64 ? (r & 7) : ((r >> 1) & 3);
#pragma unroll
      for (int j = 0; j < HID / 8; ++j) {
        const int c = 8 * j + 2 * (lane & 3);
        const float2 bv = __ldg(reinterpret_cast<const float2*>(op.bias1 + c));
        const uint32_t v = pack_bf16(elu_fast(d[4 * j + 2 * h] + bv.x), elu_fast(d[4 * j + 2 * h + 1] + bv.y));
        const int cb = (c % BKH) * 2;  // byte offset inside the row of K chunk c / BKH
        const uint32_t a = sH + (uint32_t)(c / BKH) * (kBM * BKH * 2) + (uint32_t)r * (BKH * 2) + (uint32_t)((((cb >> 4) ^ sw) << 4) | (cb & 15));
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(v) : "memory");
      }
    }
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy stores -> wgmma operand reads
  wg_sync(g);
  asm volatile("bar.sync 3, 256;" ::: "memory");  // both warpgroups are past GEMM 1: the stage ring is idle
  mbar_wait(w2_full, 0);
  float* et = reinterpret_cast<float*>(smem_raw + (tiles - smem_u32(smem_raw)));
  constexpr int TPR = N2 / 4, RPP = 128 / TPR;  // threads per row, rows per pass (each warpgroup: its own 64 rows)
  const int tg = threadIdx.x & 127, cl = 4 * (tg % TPR);
  // ---- GEMM 2 and epilogue B, per column block
#pragma unroll 1
  for (int nb = 0; nb < COUT / N2; ++nb) {
    float d[N2 / 2];
    wg::fence();
#pragma unroll
    for (int c = 0; c < Cfg::kNK2; ++c) {
      const uint64_t dh = wg::desc_k<BKH>(sH + c * (kBM * BKH * 2) + (uint32_t)g * (64u * BKH * 2u));
      const uint64_t dw = wg::desc_k<BKH>(sW2 + c * (COUT * BKH * 2) + nb * (N2 * BKH * 2));
#pragma unroll
      for (int k = 0; k < BKH / 16; ++k) wg::mma_ss<N2>(d, dh + 2 * k, dw + 2 * k, (c | k) != 0);
    }
    wg::commit();
    wg::wait<0>();
    wg::fence_regs(d);
#pragma unroll
    for (int j = 0; j < N2 / 8; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h)
        *reinterpret_cast<float2*>(et + (r0 + 8 * h) * Cfg::kEpiPitch + 8 * j + 2 * (lane & 3)) = make_float2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
    wg_sync(g);
    const int c = nb * N2 + cl;
#pragma unroll 1
    for (int r = 64 * g + tg / TPR; r < 64 * g + 64; r += RPP) {
      const int m = m0 + r;
      if (m >= op.M) break;
      const size_t row = (size_t)b * (size_t)op.o_bs + (size_t)m * COUT;
      const float4 a = *reinterpret_cast<const float4*>(et + r * Cfg::kEpiPitch + cl);
      const float4 zv = *reinterpret_cast<const float4*>(op.Z + (size_t)b * (size_t)op.z_bs + (size_t)m * COUT + c);
      const float4 bv = __ldg(reinterpret_cast<const float4*>(op.bias2 + c));
      float4 v = make_float4(zv.x + (a.x + bv.x), zv.y + (a.y + bv.y), zv.z + (a.z + bv.z), zv.w + (a.w + bv.w));
      if (op.out_f32) *reinterpret_cast<float4*>(op.out_f32 + row + c) = v;
      if (op.out_bf16) {
        if (op.out_elu) v = make_float4(elu_fast(v.x), elu_fast(v.y), elu_fast(v.z), elu_fast(v.w));
        *reinterpret_cast<uint2*>(op.out_bf16 + row + c) = make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w));
      }
    }
    wg_sync(g);  // the tile is read before the next column block overwrites it
  }
}

// ---------------------------------------------------------------------------------------------
// Causal sliding-window attention on the tensor cores (MimiAttention.forward, modeling_mimi.py:681-738,
// head_dim 64, window <= 257).  One CTA = 128 queries of one (batch, head), one warpgroup per 64 queries,
// over the 384 keys [q0-256, q0+128) in three blocks of 128 (blocks outside a warpgroup's band are skipped):
//   pass 1: S = Q K^T per block (M64 N128 K64, fp32 in registers) -> the exact row maximum over the valid keys
//   pass 2: S again; P = exp(S - max) rounded to bf16 stays in registers as the A operand of O += P V, with
//           V^T [d][key] tiles as the K-major B operand; the row sums add the rounded P; O / sum on the way out
// Inputs are the rotated bf16 q / k [B][T2][C] and v transposed [B][C][T2p] written by rope_pack_kernel.
// ---------------------------------------------------------------------------------------------
struct AttnOp {
  __nv_bfloat16* out;  // [B][T2][C]
  int T2, C, window;
  float scale_log2e;   // log2(e) / sqrt(head_dim)
};

constexpr int kAttnKeys = 384, kAttnDh = 64;
constexpr int kAttnThreads = 256;
constexpr int kAttnSmem = 16384 + 49152 + 49152 + 1024;  // Q, K (3 x 128 keys), V^T (6 x 64 keys), alignment slack

// S block kt of warpgroup g: 64 queries x 128 keys
__device__ __forceinline__ void attn_scores(float (&s)[64], uint32_t sQ, uint32_t sK, int g, int kt) {
  const uint64_t dq = wg::desc_sw128(sQ + (uint32_t)g * 8192u), dk = wg::desc_sw128(sK + (uint32_t)kt * 16384u);
  wg::fence();
#pragma unroll
  for (int k = 0; k < 4; ++k) wg::mma_ss<128>(s, dq + 2 * k, dk + 2 * k, k != 0);
  wg::commit();
  wg::wait<0>();
  wg::fence_regs(s);
}

static __global__ void __launch_bounds__(kAttnThreads) attn_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                                                                      const __grid_constant__ CUtensorMap tmVt, const AttnOp op) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bars[2];
  const uint32_t tiles = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sQ = tiles, sK = tiles + 16384, sV = tiles + 65536;
  const uint32_t qk_full = smem_u32(&bars[0]), v_full = smem_u32(&bars[1]);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * 128, h = blockIdx.y, b = blockIdx.z;
  const int kbase = q0 + 128 - kAttnKeys;

  if (threadIdx.x == 0) {
    mbar_init(qk_full, 1);
    mbar_init(v_full, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    mbar_expect_tx(qk_full, 65536);
    tma_load_3d(sQ, &tmQ, qk_full, h * kAttnDh, q0, b);
    for (int kt = 0; kt < 3; ++kt) tma_load_3d(sK + kt * 16384, &tmK, qk_full, h * kAttnDh, kbase + kt * 128, b);
    mbar_expect_tx(v_full, 49152);
    for (int kb = 0; kb < 6; ++kb) tma_load_3d(sV + kb * 8192, &tmVt, v_full, kbase + kb * 64, h * kAttnDh, b);
  }
  __syncthreads();

  const int g = warp >> 2;
  // this thread's query rows i[0], i[1] = i[0] + 8 and their valid key columns [clo, chi] (relative to kbase)
  int clo[2], chi[2];
  bool row_ok[2];
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int i = q0 + 64 * g + 16 * (warp & 3) + (lane >> 2) + 8 * e;
    row_ok[e] = i < op.T2;
    clo[e] = row_ok[e] ? max(0, i - op.window + 1) - kbase : 1;
    chi[e] = row_ok[e] ? i - kbase : 0;
  }
  // key blocks that hold a valid key of some row of the warpgroup (uniform over the warpgroup)
  const int i_first = q0 + 64 * g, i_last = min(i_first + 63, op.T2 - 1);
  const int wlo = max(0, i_first - op.window + 1) - kbase, whi = i_last - kbase;  // whi < wlo when the warpgroup has no rows
  auto live = [&](int kt) { return !(128 * kt + 127 < wlo || 128 * kt > whi); };
  auto valid = [&](int e, int col) { return col >= clo[e] && col <= chi[e]; };

  mbar_wait(qk_full, 0);
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll 1
  for (int kt = 0; kt < 3; ++kt) {
    if (!live(kt)) continue;
    float s[64];
    attn_scores(s, sQ, sK, g, kt);
#pragma unroll
    for (int i = 0; i < 64; ++i) {
      const int e = (i >> 1) & 1, col = 128 * kt + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
      if (valid(e, col)) mx[e] = fmaxf(mx[e], s[i]);
    }
  }
#pragma unroll
  for (int e = 0; e < 2; ++e) {  // the four lanes of a row hold its columns
    mx[e] = fmaxf(mx[e], __shfl_xor_sync(0xffffffffu, mx[e], 1));
    mx[e] = fmaxf(mx[e], __shfl_xor_sync(0xffffffffu, mx[e], 2));
  }
  const float mxs[2] = {mx[0] * op.scale_log2e, mx[1] * op.scale_log2e};
  mbar_wait(v_full, 0);
  float o[32];
  float sum[2] = {0.f, 0.f};
  uint32_t acc = 0;
#pragma unroll 1
  for (int kt = 0; kt < 3; ++kt) {
    if (!live(kt)) continue;
    float s[64];
    attn_scores(s, sQ, sK, g, kt);
    uint32_t p[32];
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
      const int e = (i >> 1) & 1, col = 128 * kt + 8 * (i >> 2) + 2 * (lane & 3);
      const float p0 = valid(e, col) ? exp2f(fmaf(s[i], op.scale_log2e, -mxs[e])) : 0.f;
      const float p1 = valid(e, col + 1) ? exp2f(fmaf(s[i + 1], op.scale_log2e, -mxs[e])) : 0.f;
      const __nv_bfloat162 hh = __floats2bfloat162_rn(p0, p1);
      sum[e] += __low2float(hh) + __high2float(hh);
      p[i >> 1] = *reinterpret_cast<const uint32_t*>(&hh);
    }
    // the accumulator layout of columns 16j .. 16j + 15 is the register A-operand layout of a K = 16 slice
    wg::fence();
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t a[4] = {p[4 * j], p[4 * j + 1], p[4 * j + 2], p[4 * j + 3]};
      wg::mma_rs<64>(o, a, wg::desc_sw128(sV + (uint32_t)(2 * kt + (j >> 2)) * 8192u) + 2 * (j & 3), acc | (uint32_t)j);
    }
    wg::commit();
    wg::wait<0>();
    wg::fence_regs(o);
    acc = 1;
  }
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    sum[e] += __shfl_xor_sync(0xffffffffu, sum[e], 1);
    sum[e] += __shfl_xor_sync(0xffffffffu, sum[e], 2);
  }
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    if (!row_ok[e]) continue;
    const int i = q0 + 64 * g + 16 * (warp & 3) + (lane >> 2) + 8 * e;
    const float inv = 1.0f / sum[e];
    __nv_bfloat16* orow = op.out + ((size_t)b * op.T2 + i) * op.C + h * kAttnDh;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<uint32_t*>(orow + 8 * j + 2 * (lane & 3)) = pack_bf16(o[4 * j + 2 * e] * inv, o[4 * j + 2 * e + 1] * inv);
  }
}


// ---------------------------------------------------------------------------------------------
// host side: tensor maps through the driver entry point (no link-time dependency on libcuda)
// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      p = nullptr;
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

// activations [B][rows][cin] bf16, item b at base + b * pitch rows (pitch 0 = rows), box = bk channels x 128 rows x
// 1 batch; rows past `rows` of an item read as zeros
inline bool make_act_map(CUtensorMap* tm, const void* base, int B, long long rows, int cin, int bk = kBK, long long pitch = 0) {
  EncodeTiledFn fn = encode_tiled_fn();
  if (!fn) return false;
  const cuuint64_t dims[3] = {(cuuint64_t)cin, (cuuint64_t)rows, (cuuint64_t)B};
  const cuuint64_t strides[2] = {(cuuint64_t)cin * 2, (cuuint64_t)(pitch > 0 ? pitch : rows) * (cuuint64_t)cin * 2};
  const cuuint32_t box[3] = {(cuuint32_t)bk, (cuuint32_t)kBM, 1};
  const cuuint32_t es[3] = {1, 1, 1};
  return fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
            bk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// weights [N][K] bf16, box = bk x BN
inline bool make_weight_map(CUtensorMap* tm, const void* base, int N, int K, int BN, int bk = kBK) {
  EncodeTiledFn fn = encode_tiled_fn();
  if (!fn) return false;
  const cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)N};
  const cuuint64_t strides[1] = {(cuuint64_t)K * 2};
  const cuuint32_t box[2] = {(cuuint32_t)bk, (cuuint32_t)BN};
  const cuuint32_t es[2] = {1, 1};
  return fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
            bk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// v transposed [B][C][T2p] bf16, box = 64 keys x 64 channels
inline bool make_vt_map(CUtensorMap* tm, const void* base, int B, int C, long long T2, long long T2p) {
  EncodeTiledFn fn = encode_tiled_fn();
  if (!fn) return false;
  const cuuint64_t dims[3] = {(cuuint64_t)T2, (cuuint64_t)C, (cuuint64_t)B};
  const cuuint64_t strides[2] = {(cuuint64_t)T2p * 2, (cuuint64_t)C * (cuuint64_t)T2p * 2};
  const cuuint32_t box[3] = {64, 64, 1};
  const cuuint32_t es[3] = {1, 1, 1};
  return fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

inline bool attn_supported(int C, int H, int window) { return H > 0 && C == H * kAttnDh && window >= 1 && window <= kAttnKeys - 127; }

// q, k: bf16 [B][T2][C] (rotated); vt: bf16 [B][C][T2p]; out: bf16 [B][T2][C]
// the dynamic shared-memory opt-in is a per-device function attribute: remember it per device
inline bool attr_needed(unsigned long long& done_mask) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return true;
  if (done_mask >> dev & 1ull) return false;
  done_mask |= 1ull << dev;
  return true;
}

inline cudaError_t launch_attn(const void* q, const void* k, const void* vt, __nv_bfloat16* out, int B, int T2, long long T2p, int C,
                               int H, int window, cudaStream_t st) {
  static unsigned long long attr_done = 0;
  if (attr_needed(attr_done)) {
    cudaError_t e = cudaFuncSetAttribute(attn_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnSmem);
    if (e != cudaSuccess) return e;
  }
  CUtensorMap tmQ, tmK, tmV;
  if (!make_act_map(&tmQ, q, B, T2, C) || !make_act_map(&tmK, k, B, T2, C) || !make_vt_map(&tmV, vt, B, C, T2, T2p))
    return cudaErrorInvalidValue;
  AttnOp op{out, T2, C, window, 1.4426950408889634f / sqrtf((float)kAttnDh)};
  dim3 grid((unsigned)((T2 + 127) / 128), (unsigned)H, (unsigned)B);
  attn_tc_kernel<<<grid, kAttnThreads, kAttnSmem, st>>>(tmQ, tmK, tmV, op);
  return cudaGetLastError();
}

inline int pick_bn(int N) { return N % 128 == 0 ? 128 : (N % 64 == 0 ? 64 : (N % 32 == 0 ? 32 : 0)); }

// ---- fused ResnetBlock launcher.  X: bf16 ELU(z) [B][M][2*hid]; W1: bf16 [hid][taps*2*hid]; W2: bf16 [2*hid][hid]
inline bool resblock_supported(int hid, int cout) { return cout == 2 * hid && (hid == 32 || hid == 64 || hid == 128); }

template <int HID>
inline cudaError_t launch_resblock_t(const void* X, const void* W1, const void* W2, ResOp op, int B, cudaStream_t st) {
  using Cfg = ResCfg<HID>;
  static unsigned long long attr_done = 0;
  if (attr_needed(attr_done)) {
    cudaError_t e = cudaFuncSetAttribute(resblock_tc_kernel<HID>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::smem(Cfg::kMaxStages));
    if (e != cudaSuccess) return e;
  }
  const int cout = Cfg::kCout, K1 = op.taps * cout, nk = K1 / kBK;
  op.stages = nk < Cfg::kMaxStages ? nk : Cfg::kMaxStages;
  if (op.z_bs == 0) op.z_bs = (long long)op.M * cout;
  if (op.o_bs == 0) op.o_bs = (long long)op.M * cout;
  CUtensorMap tmA, tmW1, tmW2;
  if (!make_act_map(&tmA, X, B, op.Min > 0 ? op.Min : op.M, cout, kBK, op.a_pitch) || !make_weight_map(&tmW1, W1, HID, K1, HID) ||
      !make_weight_map(&tmW2, W2, cout, HID, cout, Cfg::kBKH))
    return cudaErrorInvalidValue;
  dim3 grid((unsigned)((op.M + kBM - 1) / kBM), (unsigned)B);
  resblock_tc_kernel<HID><<<grid, kGemmThreads, Cfg::smem(op.stages), st>>>(tmA, tmW1, tmW2, op);
  return cudaGetLastError();
}

inline cudaError_t launch_resblock(const void* X, const void* W1, const void* W2, int hid, const ResOp& op, int B, cudaStream_t st) {
  switch (hid) {
    case 32: return launch_resblock_t<32>(X, W1, W2, op, B, st);
    case 64: return launch_resblock_t<64>(X, W1, W2, op, B, st);
    default: return launch_resblock_t<128>(X, W1, W2, op, B, st);
  }
}

// K chunk width: 64 channels (128-byte rows) when the channel count allows, else 32 (64-byte rows)
inline int pick_bk(int Cin) { return Cin % 64 == 0 ? 64 : (Cin % 32 == 0 ? 32 : 0); }

// supported when every K chunk stays inside one tap and the tile shapes divide
inline bool supported(int N, int K, int Cin) { return pick_bk(Cin) != 0 && K % Cin == 0 && pick_bn(N) != 0; }

template <int BN, int BK>
inline cudaError_t launch_bn(const CUtensorMap& tmA, const CUtensorMap& tmW, const TcOp& op, int B, cudaStream_t st) {
  using Cfg = TileCfg<BN, BK>;
  static unsigned long long attr_done = 0;
  if (attr_needed(attr_done)) {
    cudaError_t e = cudaFuncSetAttribute(igemm_tc_kernel<BN, BK>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::smem(Cfg::kMaxStages));
    if (e != cudaSuccess) return e;
  }
  TcOp o = op;
  if (o.r_bs == 0) o.r_bs = o.c_bs;
  const int nk = op.K / BK;
  o.stages = nk < Cfg::kMaxStages ? nk : Cfg::kMaxStages;
  // short-K layers are bound by their epilogues: two stages leave room for a third resident CTA per SM
  if (nk <= 4 && o.stages > 2) o.stages = 2;
  dim3 grid((unsigned)((op.M + kBM - 1) / kBM), (unsigned)(op.N / BN), (unsigned)B);
  igemm_tc_kernel<BN, BK><<<grid, kGemmThreads, Cfg::smem(o.stages), st>>>(tmA, tmW, o);
  return cudaGetLastError();
}

// X: bf16 [B][Min][a_cols] (a_cols = 0: Cin columns; larger when op.tap_col addresses column groups); W: bf16 [N][K]
inline cudaError_t launch(const void* X, long long Min, const void* W, const TcOp& op, int B, cudaStream_t st, int a_cols = 0) {
  const int BN = pick_bn(op.N), BK = pick_bk(op.Cin);
  CUtensorMap tmA, tmW;
  if (!make_act_map(&tmA, X, B, Min, a_cols > 0 ? a_cols : op.Cin, BK, op.a_pitch) || !make_weight_map(&tmW, W, op.N, op.K, BN, BK))
    return cudaErrorInvalidValue;
  if (BK == 64) {
    switch (BN) {
      case 128: return launch_bn<128, 64>(tmA, tmW, op, B, st);
      case 64: return launch_bn<64, 64>(tmA, tmW, op, B, st);
      default: return launch_bn<32, 64>(tmA, tmW, op, B, st);
    }
  }
  switch (BN) {  // narrow layers (Cin = 32)
    case 128: return launch_bn<128, 32>(tmA, tmW, op, B, st);
    case 64: return launch_bn<64, 32>(tmA, tmW, op, B, st);
    default: return launch_bn<32, 32>(tmA, tmW, op, B, st);
  }
}

}  // namespace tc
