// Tacotron-2 run-once neighbours of the decoder loop, on the GPU:
//   encoder  = embedding lookup (tacotron/models/tacotron.py:44-47) -> 3 x [conv1d k5 'same' + ReLU -> BatchNorm]
//              (modules.py:168-174, :379-391, batch_norm_position='after') -> BiLSTM 2 x 256 with zoneout (modules.py:207-217)
//   postnet  = clip (tacotron.py:111-112) -> 4 x [conv k5 + tanh -> BN] + [conv k5 -> BN] (modules.py:368-376)
//              -> projection 256->80 (tacotron.py:121-123) -> residual add -> clip (:126-129)
// Every sentence is processed on its own length (zero 'same' padding at ITS ends), i.e. exactly the batch-1 graph the
// reference builds (tacotron_synthesize.py:42-43).  BatchNorm (moving stats, eps 1e-3) is folded to scale/shift in double
// on the host.
#pragma once
#include "common.cuh"
#include "taco_decoder.cuh"

namespace b200tts {

constexpr int kConvTile = 8;   // time steps per CTA

// y[b][t][co] = bn_scale[co] * act( bias[co] + sum_{j,ci} x[b][t + j - k/2][ci] * K[j][ci][co] ) + bn_shift[co]
// x is either a float tensor [B][Tmax][Cin] (optionally clipped to [lo,hi] on load) or an embedding lookup ids -> table.
struct ConvArgs {
  const float* x;          // [B][Tmax][Cin] or null
  const int* ids;          // [B][Tmax] or null (then x row = table[ids])
  const float* table;      // [V][Cin]
  const int* lengths;      // [B]
  const float* K;          // [k][Cin][Cout]
  const float* bias;       // [Cout]
  const float* bn_scale;   // [Cout]
  const float* bn_shift;   // [Cout]
  float* y;                // [B][Tmax][Cout]
  int Tmax, Cin, Cout, k, act;   // act: 0 linear, 1 relu, 2 tanh
  int clip_in;             // clip the input to [lo, hi] on load
  float lo, hi;
};

// Rows t >= lengths[b] are neither read nor written; a length outside [0, Tmax] is clamped to it, as the decoders do.
__global__ void taco_conv_bn_kernel(ConvArgs A) {
  extern __shared__ float xs[];                      // [(kConvTile + k - 1)][Cin]
  const int b = blockIdx.y, t0 = blockIdx.x * kConvTile, len = min(max(A.lengths[b], 0), A.Tmax);
  if (t0 >= len) return;
  const int half = (A.k - 1) / 2, rows = kConvTile + A.k - 1;
  for (int e = threadIdx.x; e < rows * A.Cin; e += blockDim.x) {
    const int r = e / A.Cin, ci = e % A.Cin, t = t0 + r - half;
    float v = 0.f;
    if (t >= 0 && t < len) {
      if (A.ids) v = A.table[(size_t)A.ids[(size_t)b * A.Tmax + t] * A.Cin + ci];
      else v = A.x[((size_t)b * A.Tmax + t) * A.Cin + ci];
      if (A.clip_in) v = fminf(fmaxf(v, A.lo), A.hi);
    }
    xs[e] = v;
  }
  __syncthreads();
  for (int co = threadIdx.x; co < A.Cout; co += blockDim.x) {
    float acc[kConvTile];
#pragma unroll
    for (int i = 0; i < kConvTile; ++i) acc[i] = 0.f;
    for (int j = 0; j < A.k; ++j)
      for (int ci = 0; ci < A.Cin; ++ci) {
        const float w = __ldg(A.K + ((size_t)j * A.Cin + ci) * A.Cout + co);
#pragma unroll
        for (int i = 0; i < kConvTile; ++i) acc[i] = fmaf(w, xs[(i + j) * A.Cin + ci], acc[i]);
      }
    const float bb = A.bias[co], sc = A.bn_scale[co], sh = A.bn_shift[co];
#pragma unroll
    for (int i = 0; i < kConvTile; ++i) {
      if (t0 + i < len) {
        float v = acc[i] + bb;
        if (A.act == 1) v = fmaxf(v, 0.f);
        else if (A.act == 2) v = tanhf(v);
        A.y[((size_t)b * A.Tmax + t0 + i) * A.Cout + co] = fmaf(v, sc, sh);
      }
    }
  }
}

// One CTA per (sentence, direction): zoneout LSTM over the sentence, output = un-zoned new_h  -> memory[b][t][dir*U ..]
// The sentence length is clamped to [0, Tmax] (a sentence of length 0 gives all-zero rows).
__global__ void __launch_bounds__(kTacoThreads, 1) taco_bilstm_kernel(const float* __restrict__ x /*[B][Tmax][Cin]*/,
                                                                       const int* __restrict__ lengths, int Tmax, int Cin, int U,
                                                                       const float* __restrict__ Kfw, const float* __restrict__ bfw,
                                                                       const float* __restrict__ Kbw, const float* __restrict__ bbw,
                                                                       float zoneout, float* __restrict__ memory /*[B][Tmax][2U]*/) {
  extern __shared__ __align__(1024) float sm[];   // 1024: the base these kernels were settled with (tacotron.cu)
  float* in = sm;               // [Cin + U]   x_t | h
  float* z = in + Cin + U;      // [4U]
  float* c = z + 4 * U;         // [U]
  float* part = c + U;          // [>= 4 * 4U]
  const int b = blockIdx.x, dir = blockIdx.y, len = min(max(lengths[b], 0), Tmax), tid = threadIdx.x;
  const float* K = dir ? Kbw : Kfw;
  const float* bias = dir ? bbw : bfw;
  for (int i = tid; i < U; i += kTacoThreads) { in[Cin + i] = 0.f; c[i] = 0.f; }
  __syncthreads();
  const float zk = 1.f - zoneout;
  for (int s = 0; s < len; ++s) {
    const int t = dir ? (len - 1 - s) : s;
    for (int i = tid; i < Cin; i += kTacoThreads) in[i] = x[((size_t)b * Tmax + t) * Cin + i];
    __syncthreads();
    block_matvec(K, bias, in, Cin + U, 4 * U, z, part);
    for (int j = tid; j < U; j += kTacoThreads) {
      const float i_ = z[j], j_ = z[U + j], f_ = z[2 * U + j], o_ = z[3 * U + j];
      const float cn = sigmoidf_acc(f_ + 1.0f) * c[j] + sigmoidf_acc(i_) * tanhf(j_);
      const float hn = sigmoidf_acc(o_) * tanhf(cn);
      c[j] = zk * cn + zoneout * c[j];
      in[Cin + j] = zk * hn + zoneout * in[Cin + j];
      memory[((size_t)b * Tmax + t) * (2 * U) + dir * U + j] = hn;
    }
    __syncthreads();
  }
  // rows beyond the sentence are zero (BahdanauAttention zeroes masked values; the decoder never reads them anyway)
  for (int e = tid; e < (Tmax - len) * U; e += kTacoThreads)
    memory[((size_t)b * Tmax + len + e / U) * (2 * U) + dir * U + e % U] = 0.f;
}

// mel[b][t][m] = clip( clip(dec[b][t][m]) + bias[m] + sum_c r[b][t][c] * P[c][m] )     for t < lengths[b]
__global__ void taco_postnet_proj_kernel(const float* __restrict__ dec, const float* __restrict__ r, const int* __restrict__ lengths,
                                         int Tmax, int C, int M, const float* __restrict__ P, const float* __restrict__ bias, float lo,
                                         float hi, float* __restrict__ mel) {
  const int b = blockIdx.y, t = blockIdx.x;
  if (t >= lengths[b]) return;
  extern __shared__ float rs[];
  for (int i = threadIdx.x; i < C; i += blockDim.x) rs[i] = r[((size_t)b * Tmax + t) * C + i];
  __syncthreads();
  for (int m = threadIdx.x; m < M; m += blockDim.x) {
    float acc = bias[m];
    for (int cc = 0; cc < C; ++cc) acc = fmaf(rs[cc], __ldg(P + (size_t)cc * M + m), acc);
    const float d = fminf(fmaxf(dec[((size_t)b * Tmax + t) * M + m], lo), hi);
    mel[((size_t)b * Tmax + t) * M + m] = fminf(fmaxf(d + acc, lo), hi);
  }
}

}  // namespace b200tts
