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
// Philox4x32-10 (Salmon et al. 2011), key = seed, counter = (word 0, word 1, utt_lo, utt_hi).  Every stream keyed by the same
// (seed, utterance id) owns its own range of word 1, so no two streams ever read the same counter:
//   WaveRNN RAW noise     (step,  class/4)                              [0, 2^13)   one call = 4 consecutive classes
//   WaveRNN MOL uniforms  (step,  j = 0..2)                             [0, 3)      a model is RAW or MOL, never both
//   Tacotron keep flags   (step,  0x40000000 | layer*P/4 + unit/4)      [2^30, 2^31)
//   Griffin-Lim phase     (frame, 0x80000000 | bin/4)                   [2^31, 2^32)
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

// Tacotron prenet dropout (rate 0.5, always on): keep flag of unit `unit` of prenet layer `layer` (0 or 1, P units each) at
// decoder step `step` of utterance `utt`.  The one place the flags' counter is decided: the decoders and the masks dump call it.
__device__ __forceinline__ bool taco_keep_flag(uint64_t seed, uint64_t utt, int step, int layer, int unit, int P) {
  uint32_t c[4] = {(uint32_t)step, 0x40000000u | (uint32_t)(layer * (P >> 2) + (unit >> 2)), (uint32_t)utt, (uint32_t)(utt >> 32)};
  philox4x32_10(c, seed);
  return (c[unit & 3] >> 31) != 0;
}

// ---------------------------------------------------------------------------------------------
// Mixture-of-logistics sampling (voc_mode = 'MOL'): sample_from_discretized_mix_logistic, reference
// wavernn/utils/distribution.py:87-123, for one row.  fc3 gives p[0..29]: 10 mixture logits, 10 means, 10 log-scales.
// ---------------------------------------------------------------------------------------------
constexpr int kMolMix = 10, kMolParams = 3 * kMolMix, kMolU = kMolMix + 1;
constexpr float kMolLogScaleMin = -32.23619079589844f;   // float(np.log(1e-14)) rounded to fp32, as torch.clamp takes it

// uint32 -> uniform(1e-5, 1 - 1e-5) (the range of the reference's uniform_ calls): 24 random bits, exact in fp32
__device__ __forceinline__ float mol_uniform_from_bits(uint32_t x) {
  return __fmaf_rn((float)(x >> 8) * (1.0f / 16777216.0f), 1.0f - 2e-5f, 1e-5f);
}

// The 11 uniforms of one (utterance, step): counter (step, j, utt_lo, utt_hi), j = 0..2, gives 12 words; u[0..9] choose the
// mixture, u[10] drives the logistic, the 12th word is unused.  b200tts_philox_mol_uniform dumps the same stream.
__device__ __forceinline__ void philox_mol_u(uint64_t seed, uint64_t utt, uint32_t step, float (&u)[kMolU]) {
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    uint32_t c[4] = {step, (uint32_t)j, (uint32_t)utt, (uint32_t)(utt >> 32)};
    philox4x32_10(c, seed);
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (4 * j + i < kMolU) u[4 * j + i] = mol_uniform_from_bits(c[i]);
  }
}

// The sample x in [-1, 1] for parameters p and uniforms u, each operation rounded as torch rounds it on fp32 tensors (no
// contraction into FMAs, IEEE logf / expf):
//   k = argmax_j (p[j] - log(-log(u[j])))   (first maximum, like torch .max)
//   x = clamp(p[10+k] + exp(max(p[20+k], log(1e-14))) * (log(u[10]) - log(1 - u[10])), -1, 1)
__device__ __forceinline__ float mol_sample(const float* p, const float (&u)[kMolU]) {
  int k = 0;
  float best = __fsub_rn(p[0], logf(-logf(u[0])));
#pragma unroll
  for (int j = 1; j < kMolMix; ++j) {
    const float v = __fsub_rn(p[j], logf(-logf(u[j])));
    if (v > best) { best = v; k = j; }
  }
  const float ls = fmaxf(p[2 * kMolMix + k], kMolLogScaleMin);
  const float l = __fsub_rn(logf(u[kMolMix]), logf(__fsub_rn(1.0f, u[kMolMix])));
  const float x = __fadd_rn(p[kMolMix + k], __fmul_rn(expf(ls), l));
  return fminf(fmaxf(x, -1.0f), 1.0f);
}

// The MOL outputs of a step kernel: the sample of each step is a float, not a label.
struct MolIO {
  const float* teacher_x;     // [B][S] or null: fed back instead of the sample
  float* samples;             // [B][S]
  float* par;                 // wide grid only: [2][Bp][32] fc3 outputs of the last two steps, by step parity
};

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
