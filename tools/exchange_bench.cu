// Microbenchmark of the all-to-all activation exchange of the push kernel (wavernn_push.cuh), in isolation.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o tools/exchange_bench.bin tools/exchange_bench.cu
// 128 co-resident CTAs x 512 threads.  One "exchange": every CTA publishes 4*G floats (G rows x 4 units), then every
// thread of every CTA must obtain the float4s it owns in the 128 x G x 4 vector (G/4 per thread), then a block barrier.
// Reports SM cycles per exchange for several protocols:
//   0  counter barrier (red.release.gpu + ld.acquire.gpu spin + bar) followed by plain L2 loads      [round-1 grid kernel]
//   1  flag-in-data, every thread spins on its own entries (sentinel)                                [push v1]
//   2  flag-in-data, one warp spins on row 0 of every producer, block barrier, everybody loads       [push v2]
//   3  like 2 but the canary warp spins on a HINT word per producer, replicated R times (CTA c reads replica c % R)
//   4  like 1 with __nanosleep(SLEEP) between failed rounds
// plus the cost of fence.acq_rel.gpu issued by the publishing threads once per exchange (FENCE=1).
#include <cooperative_groups.h>
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <vector>
#include <cuda_runtime.h>

constexpr int NCTA = 128, NT = 512;
constexpr uint32_t SENT = 0xFFFFFFFFu;

__device__ __forceinline__ float4 ldr4(const float* p) {
  float4 v;
  asm volatile("ld.relaxed.gpu.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint4 ldr4u(const uint32_t* p) {
  uint4 v;
  asm volatile("ld.relaxed.gpu.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void str(float* p, float v) { asm volatile("st.relaxed.gpu.global.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory"); }
__device__ __forceinline__ void stru(uint32_t* p, uint32_t v) { asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ bool ready(const float4& v) {
  return __float_as_uint(v.x) != SENT && __float_as_uint(v.y) != SENT && __float_as_uint(v.z) != SENT && __float_as_uint(v.w) != SENT;
}
__device__ __forceinline__ unsigned ldacq(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

struct Args {
  float* vec;          // [3][NCTA][G][4]  (copy it%3 written at exchange `it`, copy (it+1)%3 -- last read at it-2 -- re-armed)
  uint32_t* hint;      // [R][NCTA]
  unsigned* counter;
  long long* cycles;   // [NCTA]
  float* sink;
  int iters, proto, R, fence, sleep_ns, work;
};

template <int G>
__global__ void __launch_bounds__(NT, 1) bench(Args A) {
  constexpr int NU = (G >= 16) ? G / 2 : G, UT = G / NU, NKQ = NT / NU, NKB = 128 / NKQ, NL = NKB * UT;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, c = blockIdx.x;
  const int ul = tid % NU, kq = tid / NU;
  const bool gate = tid < 4 * G;
  const int gu = tid % G, gj = tid / G;
  const size_t vstride = (size_t)NCTA * G * 4;
  int off[NL];
#pragma unroll
  for (int i = 0; i < NKB; ++i)
#pragma unroll
    for (int j = 0; j < UT; ++j) off[i * UT + j] = ((kq + NKQ * i) * G + ul + NU * j) * 4;
  float acc = 0.f;
  unsigned nbar = 0;
  long long t0 = 0;
  for (int it = 0; it < A.iters; ++it) {
    if (it == A.iters / 4) t0 = clock64();
    const int par = it % 3;
    float* v = A.vec + par * vstride;
    float* vo = A.vec + ((it + 1) % 3) * vstride;
    // a little dependent work standing in for the gate math
    float val = (float)(it & 1023) + acc * 1e-30f;
    for (int w = 0; w < A.work; ++w) val = fmaf(val, 1.0000001f, 1e-7f);
    if (gate) {
      const size_t e = ((size_t)c * G + gu) * 4 + gj;
      if (A.proto != 0) stru(reinterpret_cast<uint32_t*>(vo) + e, SENT);   // rearm the other parity (consumed one exchange ago)
      if (A.proto == 0) v[e] = val; else str(v + e, val);
      if (A.fence) asm volatile("fence.acq_rel.gpu;" ::: "memory");
    }
    if (A.proto == 3 && warp == 0) {
      __syncwarp();
      if (lane < A.R) stru(A.hint + (size_t)lane * NCTA + c, (uint32_t)(it + 1));
    }
    float4 a[NL];
    if (A.proto == 0) {
      __syncthreads();
      if (tid == 0) {
        asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(A.counter), "r"(1u) : "memory");
        const unsigned target = (++nbar) * NCTA;
        while (ldacq(A.counter) < target) {}
      }
      __syncthreads();
#pragma unroll
      for (int i = 0; i < NL; ++i) a[i] = __ldcg(reinterpret_cast<const float4*>(v + off[i]));
    } else if (A.proto == 1 || A.proto == 4) {
#pragma unroll
      for (int i = 0; i < NL; ++i) a[i] = ldr4(v + off[i]);
      unsigned pending = 0;
#pragma unroll
      for (int i = 0; i < NL; ++i) pending |= ready(a[i]) ? 0u : (1u << i);
      while (pending) {
        if (A.proto == 4) __nanosleep(A.sleep_ns);
#pragma unroll
        for (int i = 0; i < NL; ++i)
          if (pending & (1u << i)) { a[i] = ldr4(v + off[i]); if (ready(a[i])) pending &= ~(1u << i); }
      }
    } else {
#pragma unroll
      for (int i = 0; i < NL; ++i) a[i] = ldr4(v + off[i]);
      if (warp == 15) {
        if (A.proto == 2) {
          unsigned pending = 0xF;
          while (pending)
#pragma unroll
            for (int i = 0; i < 4; ++i)
              if ((pending & (1u << i)) && ready(ldr4(v + (size_t)(lane + 32 * i) * G * 4))) pending &= ~(1u << i);
        } else {
          const uint32_t want = (uint32_t)(it + 1);
          const uint32_t* h = A.hint + (size_t)(c % A.R) * NCTA + lane * 4;
          while (true) {
            const uint4 q = ldr4u(h);
            if (q.x >= want && q.y >= want && q.z >= want && q.w >= want) break;
          }
        }
      }
      __syncthreads();
      unsigned pending = 0;
#pragma unroll
      for (int i = 0; i < NL; ++i) pending |= ready(a[i]) ? 0u : (1u << i);
      while (pending)
#pragma unroll
        for (int i = 0; i < NL; ++i)
          if (pending & (1u << i)) { a[i] = ldr4(v + off[i]); if (ready(a[i])) pending &= ~(1u << i); }
    }
#pragma unroll
    for (int i = 0; i < NL; ++i) acc += a[i].x + a[i].y + a[i].z + a[i].w;
    __syncthreads();
  }
  if (tid == 0) A.cycles[c] = clock64() - t0;
  if (acc == 123.456f) A.sink[0] = acc;
}

template <int G>
double run(Args a) {
  const size_t n = 3ull * NCTA * G * 4;
  cudaMemset(a.vec, 0xFF, n * 4);
  cudaMemset(a.hint, 0, 64 * NCTA * 4);
  cudaMemset(a.counter, 0, 4);
  void* args[] = {&a};
  cudaError_t e = cudaLaunchCooperativeKernel((const void*)bench<G>, dim3(NCTA), dim3(NT), args, 0, 0);
  if (e != cudaSuccess) { printf("launch: %s\n", cudaGetErrorString(e)); exit(1); }
  e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { printf("sync: %s\n", cudaGetErrorString(e)); exit(1); }
  std::vector<long long> h(NCTA);
  cudaMemcpy(h.data(), a.cycles, NCTA * 8, cudaMemcpyDeviceToHost);
  double s = 0;
  for (auto x : h) s += (double)x;
  return s / NCTA / (a.iters - a.iters / 4);
}

int main() {
  Args a{};
  cudaMalloc(&a.vec, 3ull * NCTA * 32 * 4 * 4);
  cudaMalloc(&a.hint, 64 * NCTA * 4);
  cudaMalloc(&a.counter, 4);
  cudaMalloc(&a.cycles, NCTA * 8);
  cudaMalloc(&a.sink, 4);
  a.iters = 20000;
  const char* names[] = {"counter barrier + loads", "all threads spin on data", "canary warp on data + bar", "canary warp on hints + bar",
                         "all spin + nanosleep"};
  for (int work : {0, 200})
    for (int fence : {0, 1})
      for (int G : {4, 8, 32}) {
        for (int proto = 0; proto < 5; ++proto) {
          for (int R : {1, 8, 32}) {
            if (proto != 3 && R != 1) continue;
            for (int sl : {50, 200}) {
              if (proto != 4 && sl != 50) continue;
              a.proto = proto; a.R = R; a.fence = fence; a.sleep_ns = sl; a.work = work;
              double cyc = G == 4 ? run<4>(a) : (G == 8 ? run<8>(a) : run<32>(a));
              printf("work=%3d fence=%d G=%2d  %-28s R=%2d sleep=%3d : %8.0f cycles/exchange\n", work, fence, G, names[proto], R, sl, cyc);
              fflush(stdout);
            }
          }
        }
      }
  return 0;
}
