// Kernels of the Tacotron-2 decoder loop (taco_decoder_body.cuh): the batch decoder, free, forced, biased or teacher-forced,
// the memory-layer keys and the PHILOX keep flags.  The session kernel lives in its own translation unit (taco_session.cu).
#pragma once
#include "taco_decoder_body.cuh"

namespace b200tts {

// keys[b][t][:] = memory[b][t][:] . Wm      (BahdanauAttention memory_layer, attention.py:93-98; once per sentence)
__global__ void taco_keys_kernel(const float* __restrict__ memory, const float* __restrict__ Wm, int rows, int E, int A,
                                 float* __restrict__ keys) {
  int r = blockIdx.x;
  extern __shared__ float sm_row[];
  for (int e = threadIdx.x; e < E; e += blockDim.x) sm_row[e] = memory[(size_t)r * E + e];
  __syncthreads();
  for (int a = threadIdx.x; a < A; a += blockDim.x) {
    float acc = 0.f;
    for (int e = 0; e < E; ++e) acc = fmaf(sm_row[e], Wm[(size_t)e * A + a], acc);
    keys[(size_t)r * A + a] = acc;
  }
}

template <bool kTeacher>
__global__ void __launch_bounds__(kTacoThreads, 1) taco_decoder_kernel(TacoWeights W, TacoArgs A, TacoGtaArgs G) {
  taco_decoder_run<kTeacher, false>(W, A, G, nullptr);
}

// free or forced run with a per-sentence speaking-rate bias: mu_bias [B] (b200tts_taco_decode_biased)
__global__ void __launch_bounds__(kTacoThreads, 1) taco_decoder_biased_kernel(TacoWeights W, TacoArgs A, const float* mu_bias) {
  taco_decoder_run<false, true>(W, A, TacoGtaArgs{}, mu_bias);
}

// keep flags the PHILOX mode uses, [B][steps][2][P] (lets a test replay them through the oracle)
__global__ void taco_philox_masks_kernel(unsigned long long seed, unsigned long long utt0, int B, int steps, int P,
                                         unsigned char* __restrict__ masks) {
  size_t total = (size_t)B * steps * 2 * P;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    int j = (int)(e % P);
    size_t r = e / P;
    int layer = (int)(r % 2);
    r /= 2;
    int step = (int)(r % steps);
    int b = (int)(r / steps);
    masks[e] = taco_keep_flag(seed, utt0 + b, step, layer, j, P) ? 1 : 0;
  }
}

}  // namespace b200tts
