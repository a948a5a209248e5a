// Microbenchmark: cost of one grid-wide barrier for several protocols, with and without a payload
// (each CTA writes P floats before the barrier and reads 128*P floats after it, like one layer of the grid kernel).
// Development aid, not product code.   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/barrier_bench.bin tools/barrier_bench.cu
#include <cooperative_groups.h>
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
namespace cg = cooperative_groups;

__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) { unsigned v; asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ unsigned ld_relaxed(const unsigned* p) { unsigned v; asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ void red_release(unsigned* p, unsigned v) { asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void red_relaxed(unsigned* p, unsigned v) { asm volatile("red.relaxed.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void st_release(unsigned* p, unsigned v) { asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void st_relaxed(unsigned* p, unsigned v) { asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void fence_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }

template <int FLAVOR>
__device__ __forceinline__ void barrier(unsigned* ctr, unsigned* flags, unsigned epoch, unsigned ncta) {
  if (FLAVOR == 3) { cg::this_grid().sync(); return; }
  __syncthreads();
  if (FLAVOR == 0) {          // red.release + ld.acquire polling (round-1 first version)
    if (threadIdx.x == 0) { red_release(ctr, 1u); while (ld_acquire(ctr) < epoch * ncta) {} }
  } else if (FLAVOR == 1) {   // classic: fence, atomicAdd, volatile polling, fence
    if (threadIdx.x == 0) { __threadfence(); atomicAdd(ctr, 1u); while (*(volatile unsigned*)ctr < epoch * ncta) {} __threadfence(); }
  } else if (FLAVOR == 2) {   // fence + relaxed red; relaxed polling; one fence at the end
    if (threadIdx.x == 0) { fence_gpu(); red_relaxed(ctr, 1u); while (ld_relaxed(ctr) < epoch * ncta) {} fence_gpu(); }
  } else if (FLAVOR == 4) {   // flag per CTA: one release store, then warp 0 polls all flags in parallel
    if (threadIdx.x == 0) st_release(flags + blockIdx.x * 32, epoch);     // 128 B apart
    if (threadIdx.x < 32) {
      bool done;
      do {
        done = true;
        for (unsigned i = threadIdx.x; i < ncta; i += 32) done = done && (ld_relaxed(flags + i * 32) >= epoch);
        done = __all_sync(0xffffffffu, done);
      } while (!done);
      fence_gpu();
    }
  } else if (FLAVOR == 5) {   // like 4 but all flags packed in consecutive words (4 sectors for 128 CTAs)
    if (threadIdx.x == 0) st_release(flags + blockIdx.x, epoch);
    if (threadIdx.x < 32) {
      bool done;
      do {
        done = true;
        for (unsigned i = threadIdx.x; i < ncta; i += 32) done = done && (ld_relaxed(flags + i) >= epoch);
        done = __all_sync(0xffffffffu, done);
      } while (!done);
      fence_gpu();
    }
  }
  __syncthreads();
}

template <int FLAVOR>
__global__ void __launch_bounds__(256, 1) bench(unsigned* ctr, unsigned* flags, float* buf, int iters, int payload, float* sink) {
  const unsigned ncta = gridDim.x;
  float acc = 0.f;
  for (int it = 1; it <= iters; ++it) {
    float* w = buf + (size_t)(it & 1) * ncta * payload;
    for (int i = threadIdx.x; i < payload; i += blockDim.x) w[(size_t)blockIdx.x * payload + i] = (float)it + acc * 1e-20f;
    barrier<FLAVOR>(ctr, flags, (unsigned)it, ncta);
    const float4* r = reinterpret_cast<const float4*>(w);
    for (int i = threadIdx.x; i < (int)(ncta * payload / 4); i += blockDim.x) { float4 v = __ldcg(r + i); acc += v.x + v.y + v.z + v.w; }
  }
  if (acc == 12345.f) *sink = acc;
}

__global__ void chase(const unsigned* next, int iters, unsigned* out, long long* cycles) {
  unsigned p = 0;
  long long t0 = clock64();
  for (int i = 0; i < iters; ++i) p = __ldcg(next + p);
  long long t1 = clock64();
  *out = p; *cycles = t1 - t0;
}

template <int FLAVOR>
float run(int ncta, int iters, int payload, unsigned* ctr, unsigned* flags, float* buf, float* sink) {
  cudaMemset(ctr, 0, 256); cudaMemset(flags, 0, 132 * 128);
  void* args[] = {&ctr, &flags, &buf, &iters, &payload, &sink};
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0);
  cudaError_t e = cudaLaunchCooperativeKernel((const void*)bench<FLAVOR>, dim3(ncta), dim3(256), args, 0, 0);
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  if (e != cudaSuccess || cudaGetLastError() != cudaSuccess) { printf("launch failed: %s\n", cudaGetErrorString(e)); return -1; }
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  return ms * 1000.f / iters;
}

int main(int argc, char** argv) {
  int iters = argc > 1 ? atoi(argv[1]) : 20000;
  unsigned *ctr, *flags; float *buf, *sink;
  cudaMalloc(&ctr, 256); cudaMalloc(&flags, 132 * 128); cudaMalloc(&buf, 2 * 132 * 4096 * sizeof(float)); cudaMalloc(&sink, 4);
  cudaMemset(buf, 0, 2 * 132 * 4096 * sizeof(float));
  // L2 latency (pointer chase over 8 MB, stride 4 KB+)
  {
    const int n = 1 << 21; unsigned* h = (unsigned*)malloc(n * 4);
    for (int i = 0; i < n; ++i) h[i] = (unsigned)((i + 1031 * 33) % n);
    unsigned* d; cudaMalloc(&d, n * 4); cudaMemcpy(d, h, n * 4, cudaMemcpyHostToDevice);
    unsigned* o; long long* cyc; cudaMalloc(&o, 4); cudaMalloc(&cyc, 8);
    chase<<<1, 1>>>(d, 2000, o, cyc); chase<<<1, 1>>>(d, 20000, o, cyc); cudaDeviceSynchronize();
    long long c; cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost);
    printf("L2 dependent-load latency: %.1f cycles\n", (double)c / 20000);
  }
  const char* names[] = {"red.release+ld.acquire", "fence+atomicAdd+volatile+fence", "fence+red.relaxed+ld.relaxed+fence",
                         "cg::grid.sync", "flag/CTA 128B apart", "flag/CTA packed"};
  for (int ncta : {128, 132})
    for (int payload : {0, 4, 1024}) {
      printf("ncta=%d payload=%d floats/CTA:", ncta, payload);
      float r[6];
      r[0] = run<0>(ncta, iters, payload, ctr, flags, buf, sink); r[1] = run<1>(ncta, iters, payload, ctr, flags, buf, sink);
      r[2] = run<2>(ncta, iters, payload, ctr, flags, buf, sink); r[3] = run<3>(ncta, iters, payload, ctr, flags, buf, sink);
      r[4] = run<4>(ncta, iters, payload, ctr, flags, buf, sink); r[5] = run<5>(ncta, iters, payload, ctr, flags, buf, sink);
      printf("\n");
      for (int f = 0; f < 6; ++f) printf("   %-38s %.3f us/iter\n", names[f], r[f]);
    }
  return 0;
}
