// Micro-benchmark of the AR kernel's warp GEMV tiles in isolation (one CTA per SM, 512 threads, operands in shared
// memory, clock64 around the task loop).  Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o tile_bench tile_bench.cu
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "../../sopro_b200/csrc/ar_kernel.cuh"
using namespace sopro;


// ---- candidate (measured slower, kept as a record): k PAIRS per lane, operands of step i+1 requested before the FFMA2s of step i
template <typename WT> struct RawPair;
template <> struct RawPair<__nv_bfloat16> {
  typedef unsigned type;
  static __device__ __forceinline__ unsigned load(unsigned a) { unsigned v; asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
  static __device__ __forceinline__ float2 unpack(unsigned v) { return make_float2(__uint_as_float(v << 16), __uint_as_float(v & 0xffff0000u)); }
};
__device__ __forceinline__ float2 lds64(unsigned a) { float2 v; asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(a)); return v; }
template <int R, int TU, typename WT>
__device__ __forceinline__ float warp_rows_p(const unsigned (&w)[R], unsigned act, int K, int lane) {
  typedef typename RawPair<WT>::type Raw;
  float2 acc[R][TU];
#pragma unroll
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int u = 0; u < TU; ++u) acc[r][u] = make_float2(0.f, 0.f);
  Raw wn[R];
  float2 xn[TU];
  unsigned wa[R];
#pragma unroll
  for (int r = 0; r < R; ++r) wa[r] = w[r] + (unsigned)lane * 2u * (unsigned)sizeof(WT);
  unsigned xa = act + (unsigned)lane * 8u;
  const unsigned xrow = (unsigned)K * 4u;
#pragma unroll
  for (int r = 0; r < R; ++r) wn[r] = RawPair<WT>::load(wa[r]);
#pragma unroll
  for (int u = 0; u < TU; ++u) xn[u] = lds64(xa + (unsigned)u * xrow);
  const int steps = K >> 6;
#pragma unroll 1
  for (int it = 0; it < steps; ++it) {
    float2 wc[R], xc[TU];
#pragma unroll
    for (int r = 0; r < R; ++r) wc[r] = RawPair<WT>::unpack(wn[r]);
#pragma unroll
    for (int u = 0; u < TU; ++u) xc[u] = xn[u];
    const unsigned adv = (it + 1 < steps) ? 1u : 0u;
    xa += adv * 256u;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      wa[r] += adv * 64u * (unsigned)sizeof(WT);
      wn[r] = RawPair<WT>::load(wa[r]);
    }
#pragma unroll
    for (int u = 0; u < TU; ++u) xn[u] = lds64(xa + (unsigned)u * xrow);
#pragma unroll
    for (int u = 0; u < TU; ++u)
#pragma unroll
      for (int r = 0; r < R; ++r) acc[r][u] = ffma2(wc[r], xc[u], acc[r][u]);
  }
  float v[R * TU];
#pragma unroll
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int u = 0; u < TU; ++u) v[r * TU + u] = acc[r][u].x + acc[r][u].y;
  return reduce_transposed<R * TU>(v, lane);
}

// ---- candidate: row-packed 8 rows x 8 utterances, lanes split K one element at a time (k = lane + 32 i)
// weights in shared memory as [k][8 rows] bf16 (16 B per k), activations [k][8 utts] fp32 (32 B per k)
__device__ __forceinline__ float warp_rows_rp(unsigned wt, unsigned xt, int K, int lane) {
  float2 acc[4][8];  // [row pair][utt]: {row 2p, row 2p+1}
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int u = 0; u < 8; ++u) acc[p][u] = make_float2(0.f, 0.f);
#pragma unroll 1
  for (int k = lane; k < K; k += 32) {
    uint4 wr;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(wr.x), "=r"(wr.y), "=r"(wr.z), "=r"(wr.w) : "r"(wt + (unsigned)k * 16u));
    const float4 x0 = lds128(xt + (unsigned)k * 32u), x1 = lds128(xt + (unsigned)k * 32u + 16u);
    const float2 w0 = make_float2(__uint_as_float(wr.x << 16), __uint_as_float(wr.x & 0xffff0000u));
    const float2 w1 = make_float2(__uint_as_float(wr.y << 16), __uint_as_float(wr.y & 0xffff0000u));
    const float2 w2 = make_float2(__uint_as_float(wr.z << 16), __uint_as_float(wr.z & 0xffff0000u));
    const float2 w3 = make_float2(__uint_as_float(wr.w << 16), __uint_as_float(wr.w & 0xffff0000u));
    const float xs[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const float2 xx = make_float2(xs[u], xs[u]);
      acc[0][u] = ffma2(w0, xx, acc[0][u]);
      acc[1][u] = ffma2(w1, xx, acc[1][u]);
      acc[2][u] = ffma2(w2, xx, acc[2][u]);
      acc[3][u] = ffma2(w3, xx, acc[3][u]);
    }
  }
  float v[64];
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      v[(2 * p) * 8 + u] = acc[p][u].x;
      v[(2 * p + 1) * 8 + u] = acc[p][u].y;
    }
  // 64 outputs over 32 lanes: first fold halves, then the transposed reduction of 32
  float h[32];
  const bool up = lane & 16;
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const float keep = up ? v[i + 32] : v[i], send = up ? v[i] : v[i + 32];
    h[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
  }
  // remaining 4 levels over 32 values
  int n = 32;
#pragma unroll
  for (int s = 8; s >= 1; s >>= 1) {
    const int half = n >> 1;
    const bool u2 = (lane & s) != 0;
#pragma unroll
    for (int i = 0; i < 16; ++i)
      if (i < half) {
        const float keep = u2 ? h[i + half] : h[i], send = u2 ? h[i] : h[i + half];
        h[i] = keep + __shfl_xor_sync(0xffffffffu, send, s);
      }
    n = half;
  }
  return h[0] + h[1];
}

template <int MODE>
__global__ void __launch_bounds__(512, 1) bench(int K, int n_tasks, int rows, float* out, long long* cyc, int reps) {
  extern __shared__ __align__(128) unsigned char smem[];
  // act [8][K] fp32 | weights [rows][K] bf16
  float* act = reinterpret_cast<float*>(smem);
  __nv_bfloat16* w = reinterpret_cast<__nv_bfloat16*>(smem + (size_t)8 * K * 4);
  for (int i = threadIdx.x; i < 8 * K; i += 512) act[i] = 0.001f * (float)((i * 37) % 101);
  for (int i = threadIdx.x; i < rows * K; i += 512) w[i] = __float2bfloat16(0.01f * (float)((i * 13) % 17));
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned act_s = smem_u32(act), w_s = smem_u32(w);
  float sink = 0.f;
  __syncthreads();
  const long long t0 = clock64();
  for (int rep = 0; rep < reps; ++rep) {
    for (int task = warp; task < n_tasks; task += 16) {
      if (MODE == 0 || MODE == 1) {
        unsigned wr[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) wr[j] = w_s + (unsigned)((task * 4 + j) % rows) * (unsigned)K * 2u;
        sink += MODE == 0 ? warp_rows_s<4, 8, __nv_bfloat16>(wr, act_s, K, lane) : warp_rows_p<4, 8, __nv_bfloat16>(wr, act_s, K, lane);
      } else if (MODE == 2) {  // 8 rows x 4 utterances, k quads
        unsigned wr[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) wr[j] = w_s + (unsigned)((task * 8 + j) % rows) * (unsigned)K * 2u;
        sink += warp_rows_s<8, 4, __nv_bfloat16>(wr, act_s, K, lane);
      } else if (MODE == 3) {  // row-packed 8 x 8 (task = 8 rows)
        sink += warp_rows_rp(w_s + (unsigned)((task * 8) % rows) * 16u, act_s, K, lane);
      } else if (MODE == 4) {  // FFMA2 only: 64 accumulators, no loads (192 FFMA2 per K=384)
        float2 acc[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[i] = make_float2((float)i, (float)lane);
        float2 a = make_float2(1.0001f, 0.9999f), b = make_float2(0.5f, 0.25f);
#pragma unroll 1
        for (int k = lane * 4; k < K; k += 128) {
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            acc[i] = ffma2(a, b, acc[i]);
            acc[i] = ffma2(b, a, acc[i]);
          }
        }
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < 32; ++i) s += acc[i].x + acc[i].y;
        sink += s;
      } else if (MODE == 5) {  // loads only: the 12 LDS of a k-quad step, summed
        float s = 0.f;
#pragma unroll 1
        for (int k = lane * 4; k < K; k += 128) {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float4 q = ldsw4<__nv_bfloat16>(w_s + (unsigned)((task * 4 + j) % rows) * (unsigned)K * 2u + (unsigned)k * 2u);
            s += q.x + q.w;
          }
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            const float4 q = lds128(act_s + ((unsigned)u * (unsigned)K + (unsigned)k) * 4u);
            s += q.x + q.w;
          }
        }
        sink += s;
      }
    }
    __syncthreads();
  }
  const long long t1 = clock64();
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
  out[blockIdx.x * 512 + threadIdx.x] = sink;
}

template <int MODE>
static void run(const char* name, int K, int n_tasks, int rows, int macs_per_task) {
  int dev = 0, n_sm = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
  float* out;
  long long* cyc;
  cudaMalloc(&out, (size_t)n_sm * 512 * 4);
  cudaMalloc(&cyc, (size_t)n_sm * 8);
  const int reps = 20;
  const size_t smem = (size_t)8 * K * 4 + (size_t)rows * K * 2 + 1024;
  cudaFuncSetAttribute(bench<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  bench<MODE><<<n_sm, 512, smem>>>(K, n_tasks, rows, out, cyc, reps);
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { printf("%s: %s\n", name, cudaGetErrorString(e)); return; }
  std::vector<long long> h(n_sm);
  cudaMemcpy(h.data(), cyc, (size_t)n_sm * 8, cudaMemcpyDeviceToHost);
  long long best = h[0];
  for (auto v : h) best = v < best ? v : best;
  const double per = (double)best / reps;
  const double macs = (double)n_tasks * macs_per_task;
  printf("%-34s K=%4d tasks=%3d  %8.0f cycles/pass  %6.1f MAC/clk/SM (%4.1f%% of 128)\n", name, K, n_tasks, per, macs / per, macs / per / 1.28);
  cudaFree(out);
  cudaFree(cyc);
}

int main() {
  for (int K : {384, 1536}) {
    const int rows = K == 384 ? 88 : 24;
    for (int nt : {16, 22, 32, 6}) {
      if (K == 1536 && nt > 16) continue;
      run<0>("k-quads 4x8 (r02a)", K, nt, rows, 4 * 8 * K);
      run<1>("k-pairs 4x8 pipelined", K, nt, rows, 4 * 8 * K);
      run<2>("k-quads 8x4", K, nt, rows, 8 * 4 * K);
      run<3>("row-packed 8x8", K, nt, rows, 8 * 8 * K);
      run<4>("FFMA2 only (4x8 count)", K, nt, rows, 4 * 8 * K);
      run<5>("LDS only (4x8 k-quad pattern)", K, nt, rows, 4 * 8 * K);
    }
  }
  return 0;
}
