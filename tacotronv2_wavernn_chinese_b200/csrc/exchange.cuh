// Flag-in-data exchange primitives shared by the grid kernels that pass activations between co-resident CTAs through L2
// (wavernn_push.cuh, wavernn_tc.cuh, taco_grid.cuh).  An exchanged value is its own flag: buffers are pre-filled with
// kPushSentinel (0xFFFFFFFF, a NaN no arithmetic here produces), a producer stores plain values, and a consumer re-polls with
// relaxed L2-coherent loads until no word carries the sentinel.  Device functions only.
#pragma once
#include "common.cuh"

namespace b200tts {

constexpr uint32_t kPushSentinel = 0xFFFFFFFFu;

// ---- L2-coherent accessors ---------------------------------------------------------------------------------------
__device__ __forceinline__ float4 ld_relaxed_f4(const float* p) {
  float4 v;
  asm volatile("ld.relaxed.gpu.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long ld_relaxed_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_f32(float* p, float v) {
  asm volatile("st.relaxed.gpu.global.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
__device__ __forceinline__ void st_relaxed_u32(float* p, uint32_t v) {
  asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_relaxed_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ bool f4_ready(const float4& v) {
  return __float_as_uint(v.x) != kPushSentinel && __float_as_uint(v.y) != kPushSentinel &&
         __float_as_uint(v.z) != kPushSentinel && __float_as_uint(v.w) != kPushSentinel;
}

// A poll gives up after ~2 s (a peer CTA is gone) or as soon as any CTA has raised the global error flag.
struct PollGuard {
  int* error;
  long long t0;
  unsigned spins;
  bool aborted;
  __device__ __forceinline__ void begin() { spins = 0; }
  __device__ __forceinline__ bool expired() {
    if ((++spins & 1023u) != 0u) return false;
    if (spins == 1024u) t0 = clock64();
    if (*reinterpret_cast<volatile int*>(error) != 0 || clock64() - t0 > 4000000000LL) {
      atomicExch(error, 1);
      aborted = true;
      return true;
    }
    return false;
  }
};

}  // namespace b200tts
