// Development aid (tools/README.md): how fast can ONE SM pull a 256 KB image out of L2 into shared memory?
// The tensor-core step kernel (csrc/wavernn_tc.cuh) streams its activation images this way; this isolates the data path: a writer kernel leaves the buffer dirty in L2 (written by other SMs), then G
// reader CTAs stream it (a) with cp.async.bulk through a ring of 16 KB stages and mbarriers, no MMA, (b) with ld.global.cg by
// 512 threads.  Prints cycles per 256 KB and bytes per clock for G = 1, 16, 64, 128 readers.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/bulk_stream_bench.bin tools/bulk_stream_bench.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
constexpr int kStage = 16384, kStages = 16, kBytes = kStage * kStages;
__device__ __forceinline__ uint32_t s32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mb_init(unsigned long long* b, unsigned c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s32(b)), "r"(c) : "memory"); }
__device__ __forceinline__ void mb_wait(unsigned long long* b, unsigned par) {
  unsigned d = 0;
  while (!d) asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0,1,0,p;\n}\n" : "=r"(d) : "r"(s32(b)), "r"(par) : "memory");
}
__global__ void writer(uint4* buf, int n16) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += gridDim.x * blockDim.x) buf[i] = make_uint4(i, i + 1, i + 2, i + 3);
}
template <int NS>
__global__ void __launch_bounds__(128, 1) reader_bulk(const uint8_t* buf, int reps, long long* cyc) {
  extern __shared__ __align__(128) uint8_t sm[];
  __shared__ __align__(8) unsigned long long full[NS], empty[NS];
  if (threadIdx.x == 0) { for (int i = 0; i < NS; ++i) { mb_init(&full[i], 1); mb_init(&empty[i], 1); } asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
  __syncthreads();
  long long t0 = clock64();
  if (threadIdx.x == 0) {
    unsigned s = 0;
    for (int r = 0; r < reps; ++r)
      for (int k = 0; k < kStages; ++k, ++s) {
        const unsigned sl = s % NS, u = s / NS;
        mb_wait(&empty[sl], (u & 1u) ^ 1u);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(&full[sl])), "r"(kStage) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(s32(sm + sl * kStage)),
                     "l"(buf + (size_t)k * kStage), "r"(kStage), "r"(s32(&full[sl])) : "memory");
      }
  } else if (threadIdx.x == 32) {
    unsigned s = 0;
    for (int r = 0; r < reps; ++r)
      for (int k = 0; k < kStages; ++k, ++s) {
        const unsigned sl = s % NS, u = s / NS;
        mb_wait(&full[sl], u & 1u);
        asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s32(&empty[sl])) : "memory");
      }
    cyc[blockIdx.x] = clock64() - t0;
  }
}
__global__ void __launch_bounds__(512, 1) reader_ldg(const uint4* buf, int reps, long long* cyc, uint4* sink) {
  extern __shared__ __align__(128) uint8_t sm[];
  uint4* s4 = reinterpret_cast<uint4*>(sm);
  const int tid = threadIdx.x;
  long long t0 = clock64();
  for (int r = 0; r < reps; ++r)
#pragma unroll 1
    for (int k = 0; k < kStages; k += 4) {
      uint4 v[8];
#pragma unroll
      for (int j = 0; j < 4; ++j) { v[2 * j] = __ldcg(buf + (size_t)(k + j) * (kStage / 16) + tid * 2); v[2 * j + 1] = __ldcg(buf + (size_t)(k + j) * (kStage / 16) + tid * 2 + 1); }
#pragma unroll
      for (int j = 0; j < 4; ++j) { s4[((k + j) & 7) * (kStage / 16) + tid * 2] = v[2 * j]; s4[((k + j) & 7) * (kStage / 16) + tid * 2 + 1] = v[2 * j + 1]; }
    }
  __syncthreads();
  if (tid == 0) cyc[blockIdx.x] = clock64() - t0;
  if (sink && tid == 0) sink[blockIdx.x] = s4[blockIdx.x & 1023];
}
int main() {
  uint8_t* buf; long long* cyc; uint4* sink;
  cudaMalloc(&buf, kBytes); cudaMalloc(&cyc, 8 * 256); cudaMalloc(&sink, 16 * 256);
  const int reps = 50;
  const size_t smem = 8 * kStage;
  cudaFuncSetAttribute(reader_bulk<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  cudaFuncSetAttribute(reader_bulk<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  cudaFuncSetAttribute(reader_ldg, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  for (int G : {1, 16, 64, 128}) {
    for (int mode = 0; mode < 3; ++mode) {
      writer<<<64, 256>>>((uint4*)buf, kBytes / 16);
      if (mode == 0) reader_bulk<8><<<G, 128, smem>>>(buf, reps, cyc);
      else if (mode == 1) reader_bulk<4><<<G, 128, smem>>>(buf, reps, cyc);
      else reader_ldg<<<G, 512, smem>>>((const uint4*)buf, reps, cyc, sink);
      cudaError_t e = cudaDeviceSynchronize();
      if (e != cudaSuccess) { printf("error %s\n", cudaGetErrorString(e)); return 1; }
      long long h[256]; cudaMemcpy(h, cyc, 8 * G, cudaMemcpyDeviceToHost);
      long long mx = 0, mn = 1LL << 60; for (int i = 0; i < G; ++i) { mx = h[i] > mx ? h[i] : mx; mn = h[i] < mn ? h[i] : mn; }
      printf("%3d reader CTA(s), %-28s: %7.0f .. %7.0f cycles per 256 KB = %5.1f .. %5.1f bytes/clk per SM\n", G,
             mode == 0 ? "cp.async.bulk ring of 8" : (mode == 1 ? "cp.async.bulk ring of 4" : "ld.global.cg 512 threads"), (double)mn / reps, (double)mx / reps,
             kBytes / ((double)mx / reps), kBytes / ((double)mn / reps));
    }
  }
  // FRESH data: the buffer is rewritten by 64 other CTAs right before every single pass (what the step kernel's images are)
  for (int G : {16, 64}) {
    double tot = 0, mxs = 0;
    const int trials = 20;
    for (int i = 0; i < trials; ++i) {
      writer<<<64, 256>>>((uint4*)buf, kBytes / 16);
      reader_bulk<8><<<G, 128, smem>>>(buf, 1, cyc);
      cudaDeviceSynchronize();
      long long h[256]; cudaMemcpy(h, cyc, 8 * G, cudaMemcpyDeviceToHost);
      long long mx = 0; for (int k = 0; k < G; ++k) mx = h[k] > mx ? h[k] : mx;
      tot += (double)mx; mxs = mx > mxs ? (double)mx : mxs;
    }
    printf("%3d reader CTA(s), cp.async.bulk ring of 8, ONE pass over freshly written data: mean %.0f (max %.0f) cycles per 256 KB = %.1f bytes/clk per SM\n", G,
           tot / trials, mxs, kBytes / (tot / trials));
    tot = 0;
    for (int i = 0; i < trials; ++i) {
      reader_bulk<8><<<G, 128, smem>>>(buf, 1, cyc);
      cudaDeviceSynchronize();
      long long h[256]; cudaMemcpy(h, cyc, 8 * G, cudaMemcpyDeviceToHost);
      long long mx = 0; for (int k = 0; k < G; ++k) mx = h[k] > mx ? h[k] : mx;
      tot += (double)mx;
    }
    printf("%3d reader CTA(s), cp.async.bulk ring of 8, ONE pass, data NOT rewritten            : mean %.0f cycles per 256 KB = %.1f bytes/clk per SM\n", G, tot / trials,
           kBytes / (tot / trials));
  }
  return 0;
}
