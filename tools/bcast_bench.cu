// Microbenchmark: every CTA of a 128-CTA grid reads the SAME 512 KB matrix ([512 k][256 u] fp32, one layer's activations)
// from L2, the access pattern of the grid kernel.  Variants: loads in flight, traversal order, TMA bulk copies.
// Development aid.  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/bcast_bench.bin tools/bcast_bench.cu
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <cuda_runtime.h>

constexpr int N4 = 512 * 256 / 4;   // float4 elements in the matrix

template <int UNROLL, bool STAGGER>
__global__ void __launch_bounds__(256, 1) read_ldg(const float4* __restrict__ buf, int reps, float* sink) {
  float acc = 0.f;
  const int start = STAGGER ? (int)((long long)blockIdx.x * N4 / gridDim.x) : 0;
  for (int r = 0; r < reps; ++r) {
    const float4* b = buf + (size_t)(r & 3) * N4;
    for (int i = threadIdx.x; i < N4; i += 256 * UNROLL) {
      float4 v[UNROLL];
#pragma unroll
      for (int j = 0; j < UNROLL; ++j) { int idx = i + j * 256 + start; if (idx >= N4) idx -= N4; v[j] = __ldcg(b + idx); }
#pragma unroll
      for (int j = 0; j < UNROLL; ++j) acc += v[j].x + v[j].y + v[j].z + v[j].w;
    }
  }
  if (acc == 1234.5f) *sink = acc;
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, unsigned parity) {
  asm volatile(
      "{\n .reg .pred p;\n WAIT_LOOP:\n mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n @p bra DONE;\n bra WAIT_LOOP;\n DONE:\n}\n" ::"r"(
          (unsigned)__cvta_generic_to_shared(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   (unsigned)__cvta_generic_to_shared(dst)),
               "l"(src), "r"(bytes), "r"((unsigned)__cvta_generic_to_shared(bar))
               : "memory");
}

// TMA bulk ring: STAGES x CHUNK bytes; thread 0 produces, everybody consumes (reads a few words) then releases via bar.sync
template <int STAGES, int CHUNK, bool STAGGER>
__global__ void __launch_bounds__(256, 1) read_tma(const char* __restrict__ buf, int reps, float* sink) {
  extern __shared__ __align__(128) char sm[];
  __shared__ uint64_t full[STAGES];
  constexpr int NCH = 512 * 1024 / CHUNK;
  if (threadIdx.x == 0) { for (int s = 0; s < STAGES; ++s) mbar_init(&full[s], 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
  __syncthreads();
  float acc = 0.f;
  const int start = STAGGER ? (int)((long long)blockIdx.x * NCH / gridDim.x) : 0;
  const long long total = (long long)reps * NCH;
  if (threadIdx.x == 0)
    for (int p = 0; p < STAGES && p < total; ++p) {
      int ch = (int)((p + start) % NCH);
      mbar_expect_tx(&full[p], CHUNK);
      bulk_g2s(sm + (size_t)p * CHUNK, buf + (size_t)((p / NCH) & 3) * 512 * 1024 + (size_t)ch * CHUNK, CHUNK, &full[p]);
    }
  for (long long it = 0; it < total; ++it) {
    const int s = (int)(it % STAGES);
    const unsigned parity = (unsigned)((it / STAGES) & 1);
    mbar_wait(&full[s], parity);
    const float4* p = reinterpret_cast<const float4*>(sm + (size_t)s * CHUNK);
    float4 v = p[threadIdx.x % (CHUNK / 16)];
    acc += v.x + v.w;
    __syncthreads();                       // everybody done with stage s
    if (threadIdx.x == 0 && it + STAGES < total) {
      long long nx = it + STAGES;
      int ch = (int)((nx + start) % NCH);
      mbar_expect_tx(&full[s], CHUNK);
      bulk_g2s(sm + (size_t)s * CHUNK, buf + (size_t)((nx / NCH) & 3) * 512 * 1024 + (size_t)ch * CHUNK, CHUNK, &full[s]);
    }
  }
  if (acc == 1234.5f) *sink = acc;
}

template <class F>
float time_it(F launch, int reps) {
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  launch(); cudaDeviceSynchronize();
  cudaEventRecord(e0); launch(); cudaEventRecord(e1); cudaEventSynchronize(e1);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { printf("error %s\n", cudaGetErrorString(e)); return -1; }
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  return ms * 1000.f / reps;
}

int main(int argc, char** argv) {
  int reps = argc > 1 ? atoi(argv[1]) : 2000;
  char* buf; float* sink;
  cudaMalloc(&buf, 4 * 512 * 1024); cudaMemset(buf, 0, 4 * 512 * 1024); cudaMalloc(&sink, 4);
  const float4* b4 = (const float4*)buf;
  for (int ncta : {1, 16, 128, 132}) {
    printf("ncta=%d: us per 512 KB read by every CTA  (GB/s per SM)\n", ncta);
#define RUN_LDG(U, S) { float us = time_it([&] { read_ldg<U, S><<<ncta, 256>>>(b4, reps, sink); }, reps); printf("   ldg unroll=%-2d stagger=%d : %7.2f us  (%6.1f GB/s)\n", U, (int)S, us, 0.524288 / us * 1e3); }
    RUN_LDG(4, false) RUN_LDG(4, true) RUN_LDG(8, false) RUN_LDG(8, true) RUN_LDG(16, false) RUN_LDG(16, true) RUN_LDG(32, true)
#define RUN_TMA(ST, CH, S) { cudaFuncSetAttribute(read_tma<ST, CH, S>, cudaFuncAttributeMaxDynamicSharedMemorySize, ST * CH); \
      float us = time_it([&] { read_tma<ST, CH, S><<<ncta, 256, ST * CH>>>(buf, reps, sink); }, reps); \
      printf("   tma stages=%d chunk=%-5d stagger=%d : %7.2f us  (%6.1f GB/s)\n", ST, CH, (int)S, us, 0.524288 / us * 1e3); }
    RUN_TMA(4, 16384, false) RUN_TMA(4, 16384, true) RUN_TMA(8, 8192, true) RUN_TMA(4, 8192, true) RUN_TMA(8, 4096, true) RUN_TMA(16, 4096, true)
  }
  return 0;
}
