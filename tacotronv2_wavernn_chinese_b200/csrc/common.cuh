// Shared device helpers: error plumbing, Philox4x32-10, warp reductions, ordered-float packing.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include <stdexcept>

namespace b200tts {

struct Error : std::runtime_error {
  int code;
  Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

#define B200_CUDA(expr)                                                                            \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess)                                                                         \
      throw ::b200tts::Error(-2, std::string(#expr) + ": " + cudaGetErrorString(_e));              \
  } while (0)

// ---------------------------------------------------------------------------------------------
// Philox4x32-10 (Salmon et al. 2011).  counter = (step, class/4, utt_lo, utt_hi), key = seed.
// One call yields the noise of 4 consecutive classes of one (utterance, step).
// ---------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ void philox_round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
#ifdef __CUDA_ARCH__
  uint32_t hi0 = __umulhi(M0, c[0]), lo0 = M0 * c[0];
  uint32_t hi1 = __umulhi(M1, c[2]), lo1 = M1 * c[2];
#else
  uint64_t p0 = (uint64_t)M0 * c[0], p1 = (uint64_t)M1 * c[2];
  uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0, hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
#endif
  uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
  c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
}

__host__ __device__ __forceinline__ void philox4x32_10(uint32_t (&c)[4], uint64_t seed) {
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    philox_round(c, k0, k1);
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
}

// uint32 -> uniform in (0,1) -> Exp(1) sample q = -log(u).  Used by every kernel and by
// b200tts_philox_exponential so that the dumped stream is bit-identical to the one sampled from.
__device__ __forceinline__ float exp1_from_bits(uint32_t x) {
  float u = ((float)(x >> 9) + 0.5f) * (1.0f / 8388608.0f);    // 23 random bits + half: exact in fp32, in (0, 1)
  return -logf(u);
}

__device__ __forceinline__ void philox_exp4(uint64_t seed, uint64_t utt, uint32_t step, uint32_t cls4, float (&q)[4]) {
  uint32_t c[4] = {step, cls4, (uint32_t)utt, (uint32_t)(utt >> 32)};
  philox4x32_10(c, seed);
#pragma unroll
  for (int i = 0; i < 4; ++i) q[i] = exp1_from_bits(c[i]);
}

// ---------------------------------------------------------------------------------------------
// argmax packing: (ordered float bits << 32) | (0xFFFFFFFF - index)  -> max() picks the largest key and,
// among equal keys, the SMALLEST index (torch.argmax returns the first maximum).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long pack_key(float key, uint32_t idx) {
  uint32_t u = __float_as_uint(key);
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ((unsigned long long)u << 32) | (unsigned long long)(0xFFFFFFFFu - idx);
}
__device__ __forceinline__ uint32_t unpack_idx(unsigned long long p) { return 0xFFFFFFFFu - (uint32_t)p; }

__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    unsigned long long t = __shfl_xor_sync(0xffffffffu, v, o);
    v = t > v ? t : v;
  }
  return v;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float sigmoidf_acc(float x) { return 1.0f / (1.0f + expf(-x)); }

// two independent fp32 FMAs, round to nearest (the pairwise form the CUDA-core kernels are written in)
__device__ __forceinline__ float2 fma2_rn(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

// `2 * label.float() / (n_classes - 1.) - 1.` in fp32, same operation order as fatchord_version.py:235
__device__ __forceinline__ float label_to_float(int label, float ncls_m1) {
  return 2.0f * (float)label / ncls_m1 - 1.0f;
}

// ---------------------------------------------------------------------------------------------
// TMA bulk copy global -> shared (cp.async.bulk, completion through an mbarrier transaction count)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  asm volatile(
      "{\n .reg .pred p;\n B200_WAIT_%=:\n mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n @p bra B200_DONE_%=;\n"
      " bra B200_WAIT_%=;\n B200_DONE_%=:\n}\n" ::"r"((unsigned)__cvta_generic_to_shared(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   (unsigned)__cvta_generic_to_shared(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"((unsigned)__cvta_generic_to_shared(bar))
               : "memory");
}

}  // namespace b200tts
