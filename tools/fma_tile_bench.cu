// Cost model of the grid kernel's inner loop on one SM (development aid, see tools/README.md).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o build_ab/fma_tile_bench tools/fma_tile_bench.cu
// A thread owns a U x RT register tile and runs `iters` blocks of 4 k-steps (4*U*RT FMAs), 16 warps per CTA, one CTA
// per SM.  MODE 0: operands stay in registers (pure FMA-pipe rate).  MODE 1: weights re-read from shared memory every
// block (LDS.128, warp-broadcast), activations in registers.  MODE 2: weights from shared memory AND activations from a
// 512 KB L2-resident matrix (ld.global.cg 128-bit), i.e. the real loop without the barriers.  PACK 0: scalar FFMA,
// PACK 1: pairs of utterances against one weight register (fma2_rn below: two
// scalar FFMAs on Hopper, which has no packed fp32 FMA).  Prints FMA per clock per SM.
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

// same helper as csrc/common.cuh (this tool is compiled on its own)
__device__ __forceinline__ float2 fma2_rn(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

template <int U, int RT, int PACK>
__device__ __forceinline__ void fma_block(float (&acc)[RT][U], const float4 (&w)[RT], const float (&a)[4][U]) {
#pragma unroll
  for (int r = 0; r < RT; ++r) {
    if constexpr (PACK) {
#pragma unroll
      for (int u = 0; u < U; u += 2) {
        float2 s = make_float2(acc[r][u], acc[r][u + 1]);
        s = fma2_rn(make_float2(a[0][u], a[0][u + 1]), make_float2(w[r].x, w[r].x), s);
        s = fma2_rn(make_float2(a[1][u], a[1][u + 1]), make_float2(w[r].y, w[r].y), s);
        s = fma2_rn(make_float2(a[2][u], a[2][u + 1]), make_float2(w[r].z, w[r].z), s);
        s = fma2_rn(make_float2(a[3][u], a[3][u + 1]), make_float2(w[r].w, w[r].w), s);
        acc[r][u] = s.x; acc[r][u + 1] = s.y;
      }
    } else {
#pragma unroll
      for (int u = 0; u < U; ++u) {
        acc[r][u] = fmaf(w[r].x, a[0][u], acc[r][u]);
        acc[r][u] = fmaf(w[r].y, a[1][u], acc[r][u]);
        acc[r][u] = fmaf(w[r].z, a[2][u], acc[r][u]);
        acc[r][u] = fmaf(w[r].w, a[3][u], acc[r][u]);
      }
    }
  }
}

template <int U, int RT, int PACK, int MODE>
__global__ void __launch_bounds__(512, 1) bench(const float* __restrict__ act, const float* __restrict__ wsrc, float* out,
                                                int iters, int Bp, long long* cyc) {
  extern __shared__ __align__(16) float sw[];       // [RT][4*iters] weights
  const int K4 = 128;                               // weight columns (float4) kept in shared memory, re-used cyclically
  for (int i = threadIdx.x; i < RT * K4 * 4; i += blockDim.x) sw[i] = wsrc[i];
  __syncthreads();
  float acc[RT][U];
  float a[4][U];
  float4 w[RT];
#pragma unroll
  for (int r = 0; r < RT; ++r) {
    w[r] = reinterpret_cast<const float4*>(sw)[r * K4 + (threadIdx.x & 3)];
#pragma unroll
    for (int u = 0; u < U; ++u) acc[r][u] = 0.f;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* ap = act + (size_t)(warp & 1) * 64 * Bp + lane * U;   // two k-slices, like the kernel
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int u = 0; u < U; ++u) a[k][u] = act[(k * 32 + lane) * U + u];
  long long t0 = clock64();
  auto ld_act = [&](float (&dst)[4][U], int it) {
    const float* p = ap + (size_t)((it & 63) * 4) * Bp;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if constexpr (U == 4) {
        float4 v = __ldcg(reinterpret_cast<const float4*>(p + (size_t)k * Bp));
        dst[k][0] = v.x; dst[k][1] = v.y; dst[k][2] = v.z; dst[k][3] = v.w;
      } else {
        float2 v = __ldcg(reinterpret_cast<const float2*>(p + (size_t)k * Bp));
        dst[k][0] = v.x; dst[k][1] = v.y;
      }
    }
  };
  auto ld_w = [&](int it) {
#pragma unroll
    for (int r = 0; r < RT; ++r) w[r] = reinterpret_cast<const float4*>(sw)[r * K4 + (it & (K4 - 1))];
  };
  float nb[4][U];
#pragma unroll 1
  for (int it = 0; it < iters; it += 2) {          // ping-pong register buffers like wide_accumulate_pd (PD = 1)
    if constexpr (MODE >= 2) ld_act(nb, it + 1);
    if constexpr (MODE >= 1) ld_w(it);
    fma_block<U, RT, PACK>(acc, w, a);
    if constexpr (MODE >= 2) ld_act(a, it + 2);
    if constexpr (MODE >= 1) ld_w(it + 1);
    if constexpr (MODE >= 2) fma_block<U, RT, PACK>(acc, w, nb); else fma_block<U, RT, PACK>(acc, w, a);
  }
  long long t1 = clock64();
  float s = 0.f;
#pragma unroll
  for (int r = 0; r < RT; ++r)
#pragma unroll
    for (int u = 0; u < U; ++u) s += acc[r][u];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

template <int U, int RT, int PACK, int MODE>
static void run(const char* name, int warps, const float* act, const float* w, float* out, long long* cyc, int nsm) {
  const int iters = 4096, Bp = 256;
  size_t smem = (size_t)RT * 128 * 4 * sizeof(float);
  cudaFuncSetAttribute(bench<U, RT, PACK, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  for (int rep = 0; rep < 2; ++rep) bench<U, RT, PACK, MODE><<<nsm, warps * 32, smem>>>(act, w, out, iters, Bp, cyc);
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { printf("%s: %s\n", name, cudaGetErrorString(e)); exit(1); }
  long long h[256]; cudaMemcpy(h, cyc, nsm * sizeof(long long), cudaMemcpyDeviceToHost);
  double mx = 0; for (int i = 0; i < nsm; ++i) mx = h[i] > mx ? (double)h[i] : mx;
  double fma = (double)iters * 4 * U * RT * warps * 32;
  printf("%-34s warps=%2d  %7.1f FMA/clk/SM  (%.0f cycles)\n", name, warps, fma / mx, mx);
}

int main() {
  int nsm = 128;
  float *act, *w, *out; long long* cyc;
  cudaMalloc(&act, (size_t)512 * 256 * 4 * 2); cudaMemset(act, 0, (size_t)512 * 256 * 4 * 2);
  cudaMalloc(&w, 12 * 128 * 4 * 4); cudaMemset(w, 0, 12 * 128 * 4 * 4);
  cudaMalloc(&out, 256 * 512 * 4); cudaMalloc(&cyc, 256 * 8);
  for (int warps : {16, 8, 4}) {
    run<4, 6, 0, 0>("4x6 FFMA  regs", warps, act, w, out, cyc, nsm);
    run<4, 6, 1, 0>("4x6 FFMA2 regs", warps, act, w, out, cyc, nsm);
    run<4, 6, 0, 1>("4x6 FFMA  +LDS w", warps, act, w, out, cyc, nsm);
    run<4, 6, 1, 1>("4x6 FFMA2 +LDS w", warps, act, w, out, cyc, nsm);
    run<4, 6, 0, 2>("4x6 FFMA  +LDS w +LDG act", warps, act, w, out, cyc, nsm);
    run<4, 6, 1, 2>("4x6 FFMA2 +LDS w +LDG act", warps, act, w, out, cyc, nsm);
    run<4, 12, 1, 0>("4x12 FFMA2 regs", warps, act, w, out, cyc, nsm);
    run<4, 12, 1, 2>("4x12 FFMA2 +LDS w +LDG act", warps, act, w, out, cyc, nsm);
    run<2, 12, 1, 2>("2x12 FFMA2 +LDS w +LDG act", warps, act, w, out, cyc, nsm);
    run<4, 4, 1, 2>("4x4 FFMA2 +LDS w +LDG act", warps, act, w, out, cyc, nsm);
  }
  return 0;
}
