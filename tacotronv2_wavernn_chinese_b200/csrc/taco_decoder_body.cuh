// Tacotron-2 forward-attention decoder loop on the GPU: one persistent CTA per sentence runs the whole
// dynamic_decode while-loop (prenet -> 2 x zoneout LSTM -> forward location-sensitive attention -> frame / stop
// projections -> feed the frame back) until its own stop token fires.  The teacher-forced instantiation (kTeacher = true) runs
// the same step with the recorded mel fed back instead, for a fixed number of steps: ground-truth-aligned (GTA) mels.
//
// Replaces (reference paths relative to the reference root):
//   TacotronDecoderCell.__call__        tacotron/models/Architecture_wrappers.py:175-218
//   Prenet.__call__ (dropout always on) tacotron/models/modules.py:240-251
//   ZoneoutLSTMCell.__call__ (inference) tacotron/models/modules.py:114-142   (tf LSTMCell: gates i,j,f,o, forget_bias 1)
//   ForwardLocationSensitiveAttention   tacotron/models/attention.py:119-231  (+ window mode forward_attention.py:171-215)
//   FrameProjection / StopProjection    tacotron/models/modules.py:304, :334-342
//   CustomDecoder.step + TacoTestHelper tacotron/models/custom_decoder.py:105-135, helpers.py:36-66
//   TacoTrainingHelper (kTeacher)       helpers.py:111-151 (next input = targets[:, time], exactly len(targets) steps)
// Weights stay in TensorFlow's [in, out] layout: thread j of a matvec reads K[i][4j..4j+3] -- coalesced as is.
// ~6.9 MB of weights are streamed from L2 per step per CTA (first correct version; the weight-stationary multi-CTA
// form used for WaveRNN is the planned optimisation).
#pragma once
#include "common.cuh"

namespace b200tts {

constexpr int kTacoThreads = 1024;
constexpr int kTacoMaxTx = 512;

struct TacoWeights {
  const float *pre1_k, *pre1_b, *pre2_k, *pre2_b;        // [80,256],[256]; [256,256],[256]
  const float *l1_k, *l1_b, *l2_k, *l2_b;                // [1024,1024],[1024]; [512,1024],[1024]
  const float *q_k;                                      // [256,128]
  const float *loc_k, *loc_b, *locl_k;                   // [31,1,32],[32]; [32,128]
  const float *v_a, *b_a;                                // [128],[128]
  const float *mu_k, *mu_b;                              // [768,1],[1]
  const float *fr_k, *fr_b;                              // [768,80],[80]
  const float *st_k, *st_b;                              // [768,1],[1]
  const float *mem_k;                                    // [512,128] memory_layer (keys = memory . mem_k)
  int mels, P, U, E, A, NF, KW;                          // 80, 256 prenet, 256 lstm units, 512 enc, 128 attn, 32 filters, 31 taps
  float zoneout;
};

struct TacoArgs {
  const float* memory;      // [B][Tx_max][E]
  const float* keys;        // [B][Tx_max][A]   (precomputed by taco_keys_kernel)
  const int* lengths;       // [B]
  int B, Tx_max, max_steps, window;
  int rng_mode;             // 0 philox, 1 external masks
  unsigned long long seed, utt_offset;
  const unsigned char* masks;   // [B][max_steps][2][P] keep flags
  float* frames;            // [B][max_steps][mels]
  float* stop;              // [B][max_steps]
  float* align;             // [B][max_steps][Tx_max] or null
  int* nsteps;              // [B]
  // teacher forcing (parity tests): when non-null, the COMPLETE recurrent state is reloaded from here at the start of every
  // step and the stop rule is ignored (exactly max_steps steps run): [B][max_steps][taco_state_floats(Tx_max)] laid out as
  //   x[mels] | ctx[E] | c1[U] | h1[U] | c2[U] | h2[U] | mu | max_att | pos_rec | 0 | cum[Tx_max] | alpha[Tx_max]
  const float* forced;
};
// Teacher forcing from a recorded mel (GTA, wavernn_preprocess.py): its own struct, so that TacoArgs -- and with it the code of
// the free-running instantiation -- stays as it was.
struct TacoGtaArgs {
  const float* targets;         // [B][max_steps][mels]: the step-t input is targets[b][t-1] (the zero GO frame at t = 0)
  const int* target_lengths;    // [B]: steps run = clamp(target_lengths[b], 0, max_steps); no stop rule, no stop output
};
__host__ __device__ inline int taco_state_floats(int mels, int E, int U, int Tx_max) { return mels + E + 4 * U + 4 + 2 * Tx_max; }

// Decoder sessions (b200tts_taco_session_*): a free run cut into slices.  CTA u of taco_decoder_session_kernel resumes row u at
// step pos: at pos > 0 it reloads the row's state record (the layout of TacoArgs::forced, Tx_max = Tx), runs steps
// pos ... pos + n - 1 (fewer when the stop token fires), then saves the record, status[0] = its new position and status[1] =
// whether the stop fired.  Philox keys and output rows use the absolute step, so the slices of a row are its one-shot run.
constexpr int kTacoSessRows = 128;    // one wave of the H100's 132 SMs, one CTA per SM
struct TacoSessRow {
  const float* memory;      // [Tx][E]
  const float* keys;        // [Tx][A]
  float* state;             // [taco_state_floats(mels, E, U, Tx)]
  float* frames;            // [max_steps][mels], row t = step t
  float* stop;              // [max_steps]
  int* status;              // [2]
  unsigned long long seed, id;   // Philox key (seed, id) of the prenet dropout
  float mu_bias;
  int Tx, pos, n, window;
};
struct TacoSessIO {         // passed by value (an 11 KB kernel parameter)
  TacoSessRow row[kTacoSessRows];
};
// where b200tts_taco_session_outputs reads session i's frames, stop values and step count
struct TacoSessOut {
  const float* frames[kTacoSessRows];
  const float* stop[kTacoSessRows];
  int pos[kTacoSessRows];
};
// taco_session.cu: taco_decoder_session_kernel on `rows` thread blocks, and the gather of b200tts_taco_session_outputs
void launch_taco_sessions(const TacoWeights& W, const TacoSessIO& io, int rows, size_t smem, cudaStream_t st);
void launch_taco_session_outputs(const TacoSessOut& g, int n, int T_max, int M, float* frames, float* stop, int32_t* nsteps,
                                 cudaStream_t st);

// out[n] = bias[n] + sum_k in[k] * K[k][n]   (K row-major [Kdim][N], N % 4 == 0).  All threads of the CTA take part:
// N/4 column quads x KS k-slices; partial sums through `part` (>= KS_max*N floats).  Ends with the result in out[] and a
// __syncthreads().
__device__ __forceinline__ void block_matvec(const float* __restrict__ Kmat, const float* __restrict__ bias, const float* in,
                                             int Kdim, int N, float* out, float* part) {
  const int N4 = N >> 2;
  int KS = kTacoThreads / N4;
  if (KS > Kdim) KS = Kdim;
  const int tid = threadIdx.x;
  const int nq = tid % N4, ks = tid / N4;
  if (ks < KS) {
    const int per = (Kdim + KS - 1) / KS;
    const int k0 = ks * per, k1 = min(Kdim, k0 + per);
    // four interleaved accumulation chains per output (shorter fp32 chains: less rounding noise, and 4x the ILP)
    float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0, a2 = a0, a3 = a0;
    const float4* K4 = reinterpret_cast<const float4*>(Kmat) + nq;
    int k = k0;
#pragma unroll 2
    for (; k + 4 <= k1; k += 4) {
      const float4 w0 = __ldg(K4 + (size_t)k * N4), w1 = __ldg(K4 + (size_t)(k + 1) * N4);
      const float4 w2 = __ldg(K4 + (size_t)(k + 2) * N4), w3 = __ldg(K4 + (size_t)(k + 3) * N4);
      const float x0 = in[k], x1 = in[k + 1], x2 = in[k + 2], x3 = in[k + 3];
      a0.x = fmaf(x0, w0.x, a0.x); a0.y = fmaf(x0, w0.y, a0.y); a0.z = fmaf(x0, w0.z, a0.z); a0.w = fmaf(x0, w0.w, a0.w);
      a1.x = fmaf(x1, w1.x, a1.x); a1.y = fmaf(x1, w1.y, a1.y); a1.z = fmaf(x1, w1.z, a1.z); a1.w = fmaf(x1, w1.w, a1.w);
      a2.x = fmaf(x2, w2.x, a2.x); a2.y = fmaf(x2, w2.y, a2.y); a2.z = fmaf(x2, w2.z, a2.z); a2.w = fmaf(x2, w2.w, a2.w);
      a3.x = fmaf(x3, w3.x, a3.x); a3.y = fmaf(x3, w3.y, a3.y); a3.z = fmaf(x3, w3.z, a3.z); a3.w = fmaf(x3, w3.w, a3.w);
    }
    for (; k < k1; ++k) {
      const float4 w = __ldg(K4 + (size_t)k * N4);
      const float x = in[k];
      a0.x = fmaf(x, w.x, a0.x); a0.y = fmaf(x, w.y, a0.y); a0.z = fmaf(x, w.z, a0.z); a0.w = fmaf(x, w.w, a0.w);
    }
    float4 acc = make_float4((a0.x + a1.x) + (a2.x + a3.x), (a0.y + a1.y) + (a2.y + a3.y), (a0.z + a1.z) + (a2.z + a3.z),
                             (a0.w + a1.w) + (a2.w + a3.w));
    reinterpret_cast<float4*>(part + (size_t)ks * N)[nq] = acc;
  }
  __syncthreads();
  for (int n = tid; n < N; n += kTacoThreads) {
    float v = bias ? bias[n] : 0.f;
    for (int s = 0; s < KS; ++s) v += part[(size_t)s * N + n];
    out[n] = v;
  }
  __syncthreads();
}

__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = (threadIdx.x < kTacoThreads / 32) ? red[threadIdx.x] : 0.f;
  if (warp == 0) {
    t = warp_sum(t);
    if (lane == 0) red[0] = t;
  }
  __syncthreads();
  return red[0];
}
__device__ __forceinline__ float block_max(float v, float* red) {
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = (threadIdx.x < kTacoThreads / 32) ? red[threadIdx.x] : -INFINITY;
  if (warp == 0) {
    for (int o = 16; o > 0; o >>= 1) t = fmaxf(t, __shfl_xor_sync(0xffffffffu, t, o));
    if (lane == 0) red[0] = t;
  }
  __syncthreads();
  return red[0];
}

// kTeacher = false: free running (b200tts_taco_decode / _decode_forced).  kTeacher = true: GTA (b200tts_taco_decode_gta) --
// no forced-state reload, no window, no stop projection or rule, no stop / nsteps outputs (A.stop, A.nsteps unused).
// kBias (free running only): the speaking-rate bias of attention.py:163-165 -- every step's recursion uses
// mu' = clip(mu + mu_bias[b], 0, 1) instead of mu; the carried mu (s_mu, a forced record's mu) stays unbiased.
// kSess (free running, biased): session row R (TacoSessRow), whose buffers A describes as a batch of one sentence (b = 0) that runs
// steps R->pos ... A.max_steps - 1.
template <bool kTeacher, bool kBias, bool kSess = false>
__device__ __forceinline__ void taco_decoder_run(const TacoWeights& W, const TacoArgs& A, const TacoGtaArgs& G, const float* mu_bias,
                                                 const TacoSessRow* R = nullptr) {
  extern __shared__ __align__(1024) float sm[];   // 1024: the base these kernels were settled with (tacotron.cu)
  const int b = kSess ? 0 : (int)blockIdx.x, tid = threadIdx.x;
  float dmu = 0.f;
  if constexpr (kBias) dmu = mu_bias[b];
  const int Tx = min(A.lengths[b], A.Tx_max);
  if (Tx < 1) {                                        // empty sentence: nothing to attend to
    if (!kTeacher && tid == 0) A.nsteps[b] = 0;
    return;
  }
  const int P = W.P, U = W.U, E = W.E, AD = W.A, NF = W.NF, KW = W.KW, M = W.mels;
  // ---- shared memory carve-up ----
  float* x = sm;                       // [M]          previous frame
  float* p1 = x + 128;                 // [P]
  float* in1 = p1 + P;                 // [P + E + U]  prenet out | context | h1      (LSTM 1 input)
  float* in2 = in1 + (P + E + U);      // [U + U]      o1 | h2                         (LSTM 2 input)
  float* z = in2 + 2 * U;              // [4U]         LSTM pre-activations
  float* c1 = z + 4 * U;               // [U]
  float* c2 = c1 + U;                  // [U]
  float* pin = c2 + U;                 // [U + E]      o2 | context                    (projection / mu input)
  float* q = pin + (U + E);            // [AD]
  float* cum = q + AD;                 // [kTacoMaxTx]
  float* alpha = cum + kTacoMaxTx;     // [kTacoMaxTx]
  float* al = alpha + kTacoMaxTx;      // [kTacoMaxTx]
  float* fo = al + kTacoMaxTx;         // [M + 4]      frame out
  float* red = fo + 96;                // [64]
  float* lock = red + 64;              // [KW*NF]      location conv taps
  float* locl = lock + KW * NF;        // [NF*AD]      location layer
  float* part = locl + NF * AD;        // [>= 16 * 1024] split-K partials; also f[Tx][NF] during attention
  float* ctxv = in1 + P;               // context lives inside in1
  float* h1 = in1 + P + E;
  float* h2 = in2 + U;
  __shared__ float s_mu, s_stop;
  __shared__ int s_max, s_pos;

  for (int i = tid; i < KW * NF; i += kTacoThreads) lock[i] = W.loc_k[i];
  for (int i = tid; i < NF * AD; i += kTacoThreads) locl[i] = W.locl_k[i];
  for (int i = tid; i < M; i += kTacoThreads) x[i] = 0.f;                         // GO frame (helpers.py:149)
  for (int i = tid; i < P + E + U; i += kTacoThreads) in1[i] = 0.f;               // context = 0, h1 = 0
  for (int i = tid; i < 2 * U; i += kTacoThreads) in2[i] = 0.f;
  for (int i = tid; i < U; i += kTacoThreads) { c1[i] = 0.f; c2[i] = 0.f; }
  for (int i = tid; i < kTacoMaxTx; i += kTacoThreads) { cum[i] = (i == 0) ? 1.f : 0.f; alpha[i] = cum[i]; al[i] = 0.f; }
  if (tid == 0) { s_mu = 0.5f; s_max = 0; s_pos = 0; s_stop = 0.f; }
  __syncthreads();
  const float* mem = A.memory + (size_t)b * A.Tx_max * E;
  const float* keys = A.keys + (size_t)b * A.Tx_max * AD;
  const float zo = W.zoneout, zk = 1.f - W.zoneout;

  const int n_steps = kTeacher ? min(max(G.target_lengths[b], 0), A.max_steps) : A.max_steps;
  int step = 0;
  if constexpr (kSess) {                                   // resume: reload the record the last slice saved, as a forced step does
    step = R->pos;
    if (step > 0) {
      const float* st = R->state;
      for (int i = tid; i < M; i += kTacoThreads) x[i] = st[i];
      for (int i = tid; i < E; i += kTacoThreads) ctxv[i] = st[M + i];
      for (int i = tid; i < U; i += kTacoThreads) {
        c1[i] = st[M + E + i]; h1[i] = st[M + E + U + i]; c2[i] = st[M + E + 2 * U + i]; h2[i] = st[M + E + 3 * U + i];
      }
      const float* tail = st + M + E + 4 * U;
      if (tid == 0) { s_mu = tail[0]; s_max = (int)tail[1]; s_pos = (int)tail[2]; }
      for (int i = tid; i < A.Tx_max; i += kTacoThreads) { cum[i] = tail[4 + i]; alpha[i] = tail[4 + A.Tx_max + i]; }
      __syncthreads();
    }
  }
  for (; step < n_steps; ++step) {
    if (!kTeacher && A.forced) {                                        // teacher forcing: reload the whole state (see TacoArgs::forced)
      const float* st = A.forced + ((size_t)b * A.max_steps + step) * taco_state_floats(M, E, U, A.Tx_max);
      for (int i = tid; i < M; i += kTacoThreads) x[i] = st[i];
      for (int i = tid; i < E; i += kTacoThreads) ctxv[i] = st[M + i];
      for (int i = tid; i < U; i += kTacoThreads) {
        c1[i] = st[M + E + i]; h1[i] = st[M + E + U + i]; c2[i] = st[M + E + 2 * U + i]; h2[i] = st[M + E + 3 * U + i];
      }
      const float* tail = st + M + E + 4 * U;
      if (tid == 0) { s_mu = tail[0]; s_max = (int)tail[1]; s_pos = (int)tail[2]; }
      for (int i = tid; i < A.Tx_max; i += kTacoThreads) { cum[i] = tail[4 + i]; alpha[i] = tail[4 + A.Tx_max + i]; }
      __syncthreads();
    }
    // ---------------- prenet (2 x dense + relu + dropout 0.5, always on) ----------------
    block_matvec(W.pre1_k, W.pre1_b, x, M, P, p1, part);
    for (int j = tid; j < P; j += kTacoThreads) {
      float keep;
      if (A.rng_mode == 0) {
        keep = taco_keep_flag(A.seed, A.utt_offset + b, step, 0, j, P) ? 1.f : 0.f;
      } else {
        keep = A.masks[(((size_t)b * A.max_steps + step) * 2 + 0) * P + j] ? 1.f : 0.f;
      }
      p1[j] = fmaxf(p1[j], 0.f) * keep * 2.0f;
    }
    __syncthreads();
    block_matvec(W.pre2_k, W.pre2_b, p1, P, P, in1, part);
    for (int j = tid; j < P; j += kTacoThreads) {
      float keep;
      if (A.rng_mode == 0) {
        keep = taco_keep_flag(A.seed, A.utt_offset + b, step, 1, j, P) ? 1.f : 0.f;
      } else {
        keep = A.masks[(((size_t)b * A.max_steps + step) * 2 + 1) * P + j] ? 1.f : 0.f;
      }
      in1[j] = fmaxf(in1[j], 0.f) * keep * 2.0f;
    }
    __syncthreads();
    // ---------------- LSTM 1: [prenet | context | h1] . K1 ----------------
    block_matvec(W.l1_k, W.l1_b, in1, P + E + U, 4 * U, z, part);
    for (int j = tid; j < U; j += kTacoThreads) {
      const float i_ = z[j], j_ = z[U + j], f_ = z[2 * U + j], o_ = z[3 * U + j];
      const float cn = sigmoidf_acc(f_ + 1.0f) * c1[j] + sigmoidf_acc(i_) * tanhf(j_);
      const float hn = sigmoidf_acc(o_) * tanhf(cn);
      c1[j] = zk * cn + zo * c1[j];                       // zoneout at inference, modules.py:137-138
      const float hprev = h1[j];
      h1[j] = zk * hn + zo * hprev;
      in2[j] = hn;                                        // the cell OUTPUT is the un-zoned new_h (:118,:142)
    }
    __syncthreads();
    // ---------------- LSTM 2: [o1 | h2] . K2 ----------------
    block_matvec(W.l2_k, W.l2_b, in2, 2 * U, 4 * U, z, part);
    for (int j = tid; j < U; j += kTacoThreads) {
      const float i_ = z[j], j_ = z[U + j], f_ = z[2 * U + j], o_ = z[3 * U + j];
      const float cn = sigmoidf_acc(f_ + 1.0f) * c2[j] + sigmoidf_acc(i_) * tanhf(j_);
      const float hn = sigmoidf_acc(o_) * tanhf(cn);
      c2[j] = zk * cn + zo * c2[j];
      const float hprev = h2[j];
      h2[j] = zk * hn + zo * hprev;
      pin[j] = hn;                                        // o2 = query and first part of the projection input
    }
    __syncthreads();
    // ---------------- attention ----------------
    block_matvec(W.q_k, nullptr, pin, U, AD, q, part);    // processed query (no bias)
    // location convolution on the cumulated alignments: f[t][c] ('same', cross-correlation)  -> part[t*NF + c]
    float* f = part;
    for (int e = tid; e < Tx * NF; e += kTacoThreads) {
      const int t = e / NF, c = e % NF;
      float acc = W.loc_b[c];
      for (int k = 0; k < KW; ++k) {
        const int tt = t + k - (KW - 1) / 2;
        if (tt >= 0 && tt < Tx) acc = fmaf(lock[k * NF + c], cum[tt], acc);
      }
      f[e] = acc;
    }
    __syncthreads();
    // energy[t] = sum_d v[d] * tanh(keys[t][d] + q[d] + (f[t] . Wl)[d] + b_a[d]) : one warp per t
    {
      const int lane = tid & 31, warp = tid >> 5;
      for (int t = warp; t < Tx; t += kTacoThreads / 32) {
        float e = 0.f;
        for (int d = lane; d < AD; d += 32) {
          float loc = 0.f;
          for (int c = 0; c < NF; ++c) loc = fmaf(f[t * NF + c], locl[c * AD + d], loc);
          e += W.v_a[d] * tanhf(keys[(size_t)t * AD + d] + q[d] + loc + W.b_a[d]);
        }
        e = warp_sum(e);
        if (lane == 0) al[t] = e;
      }
    }
    __syncthreads();
    // softmax over t < Tx, cumulate (pre-modulation), forward recursion, normalise
    float ev = -INFINITY;
    for (int t = tid; t < Tx; t += kTacoThreads) ev = fmaxf(ev, al[t]);
    const float emax = block_max(ev, red);
    float es = 0.f;
    for (int t = tid; t < Tx; t += kTacoThreads) { const float e = expf(al[t] - emax); al[t] = e; es += e; }
    const float esum = block_sum(es, red);
    float mu = s_mu;
    if constexpr (kBias) mu = fmaxf(fminf(__fadd_rn(mu, dmu), 1.f), 0.f);   // tf.clip_by_value(mu + delta, 0, 1): min, then max
    float fs = 0.f;
    for (int t = tid; t < Tx; t += kTacoThreads) {
      const float a = al[t] / esum;
      cum[t] += a;                                                             // attention.py:154
      const float sh = t > 0 ? alpha[t - 1] : 0.f;
      const float v = ((1.f - mu) * alpha[t] + mu * sh + 1e-10f) * a;          // attention.py:167
      al[t] = v;
      fs += v;
    }
    __syncthreads();
    if (!kTeacher && A.window) {                                               // forward_attention.py:171-215
      if (tid == 0) {
        int am = 0; float best = al[0];
        for (int t = 1; t < Tx; ++t) if (al[t] > best) { best = al[t]; am = t; }
        int nm = (am <= s_max) ? s_max : s_max + 1;
        if (s_pos < 5 && 2 < nm) nm = s_max;
        int pr = (nm == s_max) ? s_pos + 1 : 1;
        if (!(pr < 10)) { nm = nm + 1; pr = 1; }                               // :191-195
        s_max = nm; s_pos = pr;
      }
      __syncthreads();
      const int nm = s_max;
      float ws = 0.f;
      for (int t = tid; t < Tx; t += kTacoThreads) {
        if (!(t >= nm - 2 && t < nm + 3)) al[t] = 0.f;
        ws += al[t];
      }
      const float wsum = block_sum(ws, red);
      if (tid == 0) { const int pk = min(max(nm, 0), Tx - 1); al[pk] = (wsum < 1e-10f ? 1.0f : wsum) * 2.0f; }   // :209-215
      __syncthreads();
      fs = 0.f;
      for (int t = tid; t < Tx; t += kTacoThreads) fs += al[t];
    }
    const float fsum = block_sum(fs, red);
    for (int t = tid; t < Tx; t += kTacoThreads) {
      const float v = al[t] / fsum;                                            // attention.py:220
      al[t] = v;
      alpha[t] = v;
      if (A.align) A.align[((size_t)b * A.max_steps + step) * A.Tx_max + t] = v;
    }
    __syncthreads();
    // context = al . memory  -> ctxv (in1) and pin[U..]   : E/4 column quads x t-slices
    {
      const int E4 = E >> 2;
      int TS = kTacoThreads / E4;
      const int nq = tid % E4, ts = tid / E4;
      if (ts < TS) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int t = ts; t < Tx; t += TS) {
          const float a = al[t];
          const float4 m = __ldg(reinterpret_cast<const float4*>(mem + (size_t)t * E) + nq);
          acc.x = fmaf(a, m.x, acc.x); acc.y = fmaf(a, m.y, acc.y); acc.z = fmaf(a, m.z, acc.z); acc.w = fmaf(a, m.w, acc.w);
        }
        reinterpret_cast<float4*>(part + (size_t)ts * E)[nq] = acc;
      }
      __syncthreads();
      for (int e = tid; e < E; e += kTacoThreads) {
        float v = 0.f;
        for (int s = 0; s < TS; ++s) v += part[(size_t)s * E + e];
        ctxv[e] = v;
        pin[U + e] = v;
      }
      __syncthreads();
    }
    // mu' = sigmoid([context | query_in] . Wmu + b)   (attention.py:229: concat order is [context, query])
    // stop = sigmoid([o2 | context] . Ws + b)          (Architecture_wrappers.py:196-199)
    if constexpr (kTeacher) {
      float pm = 0.f;
      for (int i = tid; i < U + E; i += kTacoThreads) {
        const int mi = (i < U) ? (E + i) : (i - U);
        pm = fmaf(pin[i], W.mu_k[mi], pm);
      }
      const float sm_ = block_sum(pm, red);
      if (tid == 0) s_mu = sigmoidf_acc(sm_ + W.mu_b[0]);
    } else {
      float pm = 0.f, ps = 0.f;
      for (int i = tid; i < U + E; i += kTacoThreads) {
        const float vin = pin[i];                       // i < U: o2[i] ; else context[i-U]
        ps = fmaf(vin, W.st_k[i], ps);
        const int mi = (i < U) ? (E + i) : (i - U);     // position in [context | query]
        pm = fmaf(vin, W.mu_k[mi], pm);
      }
      const float sm_ = block_sum(pm, red);
      const float ss_ = block_sum(ps, red);
      if (tid == 0) { s_mu = sigmoidf_acc(sm_ + W.mu_b[0]); s_stop = sigmoidf_acc(ss_ + W.st_b[0]); }
    }
    // frame = [o2 | context] . Wf + b
    block_matvec(W.fr_k, W.fr_b, pin, U + E, M, fo, part);
    for (int i = tid; i < M; i += kTacoThreads) {
      const float v = fo[i];
      A.frames[((size_t)b * A.max_steps + step) * M + i] = v;
      if constexpr (kTeacher)
        x[i] = G.targets[((size_t)b * A.max_steps + step) * M + i];   // next input = the recorded frame (helpers.py:142)
      else
        x[i] = v;                                        // next input = this frame (r = 1, helpers.py:64)
    }
    if constexpr (!kTeacher) {
      if (tid == 0) A.stop[(size_t)b * A.max_steps + step] = s_stop;
    }
    __syncthreads();
    if constexpr (!kTeacher) {
      if (s_stop > 0.5f && !A.forced) { ++step; break; }   // finished = round(stop) (half-to-even -> strictly > 0.5)
    }
  }
  if constexpr (!kTeacher) {
    if (tid == 0) A.nsteps[b] = step;
  }
  if constexpr (kSess) {                                   // save the record for the next slice (A.nsteps = R->status)
    float* st = R->state;
    for (int i = tid; i < M; i += kTacoThreads) st[i] = x[i];
    for (int i = tid; i < E; i += kTacoThreads) st[M + i] = ctxv[i];
    for (int i = tid; i < U; i += kTacoThreads) {
      st[M + E + i] = c1[i]; st[M + E + U + i] = h1[i]; st[M + E + 2 * U + i] = c2[i]; st[M + E + 3 * U + i] = h2[i];
    }
    float* tail = st + M + E + 4 * U;
    if (tid == 0) { tail[0] = s_mu; tail[1] = (float)s_max; tail[2] = (float)s_pos; tail[3] = 0.f; R->status[1] = s_stop > 0.5f; }
    for (int i = tid; i < A.Tx_max; i += kTacoThreads) { tail[4 + i] = cum[i]; tail[4 + A.Tx_max + i] = alpha[i]; }
  }
}

}  // namespace b200tts
