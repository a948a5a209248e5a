// Tacotron-2 forward-attention decoder loop, WEIGHT-STATIONARY over 128 thread blocks (one sentence; BASELINE config 4).
//
// taco_decoder_kernel (taco_decoder.cuh) runs a sentence in ONE block and re-streams the 6.9 MB of decoder weights from L2
// every step.  Here the weights are resident chip-wide, the way the WaveRNN grid is:
// block c of 128 (cooperative launch, 512 threads) keeps in shared memory the columns that produce
//     prenet units 2c, 2c+1 (both layers)   .   LSTM-1 and LSTM-2 units 2c, 2c+1 (all four gates)   .   attention dimension c
//     context columns 4c ... 4c+3           .   mel column c (c < 80)
// and the six vectors a step needs from everybody travel through L2 as FLAG-IN-DATA records (exchange.cuh: the
// value is the flag, a sentinel NaN marks "not yet", parity copies re-armed one step ahead):
//     P1, P2  prenet layer outputs (dropout applied)           L1  LSTM-1 output o1 | zoned h1          L2  o2 | zoned h2
//     EN      per-dimension partial energies e_c[t] = v_c tanh(keys[t][c] + q_c + loc_c[t] + b_c)        CTX context
// Partitioning the attention by DIMENSION keeps the query layer local (q_c needs column c of W_q only) and costs one
// tanh per position and block; every block then adds the 128 partial energies of each position in producer order and runs
// softmax / cumulation / forward recursion / window redundantly, so alignments and stop decisions agree bit for bit everywhere.
// The frame that is fed back never travels: prenet layer 1 consumes [o2 | context] through W_f . W_1 folded on the host in
// float64 (a forced previous frame, teacher forcing, takes the plain W_1 path).
//
// Replaces the same reference code as taco_decoder.cuh (Architecture_wrappers.py:175-218, attention.py:119-231,
// forward_attention.py:171-215, modules.py:114-142,240-251,304,334-342, custom_decoder.py:105-135, helpers.py:36-66).
#pragma once
#include "common.cuh"
#include "taco_decoder.cuh"
#include "exchange.cuh"

namespace b200tts {

constexpr int kTgThreads = 512;
constexpr int kTgWarps = kTgThreads / 32;
constexpr int kTgCtas = 128;

struct TacoGridModel {        // one block's weight blob (offsets in floats)
  int oW1, oB1;               // [M][2], [2]                 prenet layer 1 columns (forced / GO frame path)
  int oWfold, oBfold;         // [U+E][2], [2]               (W_f . W_1) columns: prenet layer 1 from [o2 | context]
  int oW2, oB2;               // [P][2], [2]
  int oK1, oBk1;              // [P+E+U][8], [8]             LSTM-1 columns gate*2 + unit (gates i, j, f, o)
  int oK2, oBk2;              // [2U][8], [8]
  int oWq;                    // [U]                         column c of the query layer
  int oFloc;                  // [KW] + 4                    folded location filter of dimension c | (b_loc . W_l + b_a)[c] | v_a[c] | 1 - zoneout | zoneout
  int oProj;                  // [U+E][4] + [4]              (mu gate, stop token, mel column c, 0) in [o2 | context] order, biases
  int blob;
  int M, P, U, E, KW;
};

struct TacoGridArgs {
  const float* wblob;         // [128][blob]
  float* vec;                 // [2][copy]   exchange buffers, copy = 2048 + 128 * Txp floats
  int* error;
  const float* memory;        // [Tx][E]
  const float* keys;          // [Tx][AD]
  const int* lengths;         // [1] true sentence length (<= Tx)
  int Tx, Txp, max_steps, window;     // Tx = padded length of the caller's buffers
  int rng_mode;
  unsigned long long seed, utt;
  const unsigned char* masks; // [max_steps][2][P]
  const float* forced;        // [max_steps][taco_state_floats]  (Tx_max = Tx_alloc)
  int Tx_alloc;               // Tx_max of the caller's buffers (align rows, forced records)
  float* frames;              // [max_steps][M]
  float* stop;                // [max_steps]
  float* align;               // [max_steps][Tx_alloc] or null
  int* nsteps;
};

enum { TG_P1 = 0, TG_P2 = 256, TG_L1 = 512, TG_L2 = 1024, TG_CTX = 1536, TG_EN = 2048 };

// ---- block-wide helpers (512 threads) ---------------------------------------------------------------------------------
// out[c] = bias[c] + sum_k in[k] * W[k*NC + c]; partial sums: warp shuffle tree, then the 16 warps in order.
template <int NC>
__device__ __forceinline__ void tg_matvec(const float* __restrict__ W, const float* __restrict__ bias, const float* in, int K, float* out,
                                          float* part) {
  float acc[NC];
#pragma unroll
  for (int c = 0; c < NC; ++c) acc[c] = 0.f;
  for (int k = threadIdx.x; k < K; k += kTgThreads) {
    const float x = in[k];
    if constexpr (NC % 4 == 0) {
#pragma unroll
      for (int c4 = 0; c4 < NC / 4; ++c4) {
        const float4 w = reinterpret_cast<const float4*>(W + (size_t)k * NC)[c4];
        acc[c4 * 4 + 0] = fmaf(x, w.x, acc[c4 * 4 + 0]); acc[c4 * 4 + 1] = fmaf(x, w.y, acc[c4 * 4 + 1]);
        acc[c4 * 4 + 2] = fmaf(x, w.z, acc[c4 * 4 + 2]); acc[c4 * 4 + 3] = fmaf(x, w.w, acc[c4 * 4 + 3]);
      }
    } else {
#pragma unroll
      for (int c = 0; c < NC; ++c) acc[c] = fmaf(x, W[(size_t)k * NC + c], acc[c]);
    }
  }
#pragma unroll
  for (int c = 0; c < NC; ++c) acc[c] = warp_sum(acc[c]);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
#pragma unroll
    for (int c = 0; c < NC; ++c) part[warp * NC + c] = acc[c];
  }
  __syncthreads();
  if (threadIdx.x < NC) {
    float v = bias ? bias[threadIdx.x] : 0.f;
#pragma unroll
    for (int w = 0; w < kTgWarps; ++w) v += part[w * NC + threadIdx.x];
    out[threadIdx.x] = v;
  }
  __syncthreads();
}
__device__ __forceinline__ float tg_block_sum(float v, float* red) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < kTgWarps; ++w) t += red[w];
  return t;
}
__device__ __forceinline__ float tg_block_max(float v, float* red) {
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = -INFINITY;
#pragma unroll
  for (int w = 0; w < kTgWarps; ++w) t = fmaxf(t, red[w]);
  return t;
}

// polls `n4` float4 records starting at src and hands each to `sink(index, value)`; every thread takes records tid, tid+512, ...
template <class Sink>
__device__ __forceinline__ void tg_gather(const float* src, int n4, PollGuard& pg, Sink sink) {
  for (int i = threadIdx.x; i < n4; i += kTgThreads) {
    float4 v = ld_relaxed_f4(src + (size_t)i * 4);
    if (!f4_ready(v)) {
      pg.begin();
      while (!pg.aborted) {
        v = ld_relaxed_f4(src + (size_t)i * 4);
        if (f4_ready(v) || pg.expired()) break;
      }
    }
    sink(i, v);
  }
}

// kBias: the speaking-rate bias of attention.py:163-165 (see taco_decoder_run); every block applies the same mu_bias[0]
// redundantly, so alignments and stop decisions still agree bit for bit everywhere.
template <bool kBias>
__device__ __forceinline__ void taco_grid_run(const TacoGridModel& Md, const TacoGridArgs& A, const float* mu_bias) {
  extern __shared__ __align__(1024) float sm[];   // 1024: the base these kernels were settled with (tacotron.cu)
  const int tid = threadIdx.x, c = blockIdx.x;
  float dmu = 0.f;
  if constexpr (kBias) dmu = mu_bias[0];
  const int M = Md.M, P = Md.P, U = Md.U, E = Md.E, KW = Md.KW;
  const int Tx = min(A.lengths[0], A.Tx), Txp = A.Txp;
  if (Tx < 1) {                                        // empty sentence: nothing to attend to
    if (threadIdx.x == 0 && blockIdx.x == 0) A.nsteps[0] = 0;
    return;
  }
  float* Wb = sm;
  float* in1 = sm + Md.blob;             // [P + E + U]   prenet-2 out | context | h1
  float* in2 = in1 + (P + E + U);        // [2U]          o1 | h2
  float* pin = in2 + 2 * U;              // [U + E]       o2 | context
  float* p1 = pin + (U + E);             // [P]
  float* xbuf = p1 + P;                  // [128]         forced previous frame
  float* cum = xbuf + 128;               // [Txp]
  float* alpha = cum + Txp;              // [Txp]
  float* al = alpha + Txp;               // [Txp]
  float* keyc = al + Txp;                // [Txp]         keys[t][c]
  float* memc = keyc + Txp;              // [Txp][4]      memory[t][4c .. 4c+3]
  float* part = memc + 4 * Txp;          // [16 * 8 + 64]
  float* outv = part + 16 * 8;           // [16] matvec results
  float* red = outv + 16;                // [32]
  float* epart = red + 32;               // [16][Txp]     partial energy sums of 8 producers each
  __shared__ float s_mu, s_stop, s_c1[2], s_c2[2], s_h1[2], s_h2[2];
  __shared__ int s_max, s_pos;

  {   // weights: TMA bulk copies signalled through an mbarrier
    __shared__ __align__(8) unsigned long long wbar;
    const char* src = reinterpret_cast<const char*>(A.wblob + (size_t)c * Md.blob);
    const unsigned total = (unsigned)Md.blob * 4u;
    if (tid == 0) mbar_init(&wbar, 1);
    __syncthreads();
    if (tid == 0) {
      mbar_expect_tx(&wbar, total);
      for (unsigned off = 0; off < total; off += 32768u)
        tma_bulk_g2s(reinterpret_cast<char*>(Wb) + off, src + off, min(32768u, total - off), &wbar);
    }
    mbar_wait(&wbar, 0);
  }
  for (int i = tid; i < P + E + U; i += kTgThreads) in1[i] = 0.f;                 // context = 0, h1 = 0
  for (int i = tid; i < 2 * U; i += kTgThreads) in2[i] = 0.f;
  for (int i = tid; i < U + E; i += kTgThreads) pin[i] = 0.f;
  for (int i = tid; i < 128; i += kTgThreads) xbuf[i] = 0.f;                       // GO frame (helpers.py:149)
  for (int i = tid; i < Txp; i += kTgThreads) {
    cum[i] = (i == 0) ? 1.f : 0.f; alpha[i] = cum[i]; al[i] = 0.f;                 // attention.py:112-117
    keyc[i] = i < Tx ? A.keys[(size_t)i * 128 + c] : 0.f;
  }
  for (int i = tid; i < 4 * Txp; i += kTgThreads) memc[i] = (i >> 2) < Tx ? A.memory[(size_t)(i >> 2) * E + 4 * c + (i & 3)] : 0.f;
  if (tid == 0) { s_mu = 0.5f; s_max = 0; s_pos = 0; s_stop = 0.f; s_c1[0] = s_c1[1] = s_c2[0] = s_c2[1] = 0.f; s_h1[0] = s_h1[1] = s_h2[0] = s_h2[1] = 0.f; }
  __syncthreads();

  PollGuard pg{A.error, 0, 0, false};
  const size_t copy = (size_t)2048 + (size_t)kTgCtas * Txp;
  const float* wfloc = Wb + Md.oFloc;
  const float bloc = wfloc[KW], v_c = wfloc[KW + 1], zk = wfloc[KW + 2], zr = wfloc[KW + 3];   // 1 - zoneout, zoneout

  int step = 0;
  for (; step < A.max_steps; ++step) {
    const int par = step & 1;
    float* vw = A.vec + (size_t)par * copy;            // this step's copy
    float* vo = A.vec + (size_t)(par ^ 1) * copy;      // last step's copy: re-armed below for step + 1
    bool use_x = (step == 0);
    if (A.forced) {                                    // teacher forcing: reload the whole recurrent state (TacoArgs::forced)
      const float* st = A.forced + (size_t)step * taco_state_floats(M, E, U, A.Tx_alloc);
      for (int i = tid; i < M; i += kTgThreads) xbuf[i] = st[i];
      for (int i = tid; i < E; i += kTgThreads) { in1[P + i] = st[M + i]; pin[U + i] = st[M + i]; }
      for (int i = tid; i < U; i += kTgThreads) { in1[P + E + i] = st[M + E + U + i]; in2[U + i] = st[M + E + 3 * U + i]; }
      const float* tail = st + M + E + 4 * U;
      if (tid == 0) {
        s_mu = tail[0]; s_max = (int)tail[1]; s_pos = (int)tail[2];
        s_c1[0] = st[M + E + 2 * c]; s_c1[1] = st[M + E + 2 * c + 1];
        s_h1[0] = st[M + E + U + 2 * c]; s_h1[1] = st[M + E + U + 2 * c + 1];
        s_c2[0] = st[M + E + 2 * U + 2 * c]; s_c2[1] = st[M + E + 2 * U + 2 * c + 1];
        s_h2[0] = st[M + E + 3 * U + 2 * c]; s_h2[1] = st[M + E + 3 * U + 2 * c + 1];
      }
      for (int i = tid; i < Txp; i += kTgThreads) {
        cum[i] = i < Tx ? tail[4 + i] : 0.f;
        alpha[i] = i < Tx ? tail[4 + A.Tx_alloc + i] : 0.f;
      }
      use_x = true;
      __syncthreads();
    }
    // ---------------- S1: prenet layer 1 (dense + relu + dropout 0.5, always on: modules.py:240-251) ----------------
    if (use_x) tg_matvec<2>(Wb + Md.oW1, Wb + Md.oB1, xbuf, M, outv, part);
    else tg_matvec<2>(Wb + Md.oWfold, Wb + Md.oBfold, pin, U + E, outv, part);
    if (tid < 2) {
      const int j = 2 * c + tid;
      float keep;
      if (A.rng_mode == 0) {
        keep = taco_keep_flag(A.seed, A.utt, step, 0, j, P) ? 1.f : 0.f;
      } else {
        keep = A.masks[((size_t)step * 2 + 0) * P + j] ? 1.f : 0.f;
      }
      st_relaxed_f32(vw + TG_P1 + j, fmaxf(outv[tid], 0.f) * keep * 2.0f);
    }
    // ---------------- E1 + S2: prenet layer 2 ----------------
    tg_gather(vw + TG_P1, P / 4, pg, [&](int i, float4 v) { reinterpret_cast<float4*>(p1)[i] = v; });
    if (__syncthreads_or(pg.aborted ? 1 : 0)) return;
    // REARM: every block's P1 of this step has been seen, so every block is past all its reads of the PREVIOUS step's
    // vectors (a block publishes P1(step) after its last read of step-1 data): last step's copy can take the sentinel
    // again.  Nobody polls that copy for step+1 before it has seen this block's CTX of this step, published after this fence.
    {
      if (tid < 2) { st_relaxed_u32(vo + TG_P1 + 2 * c + tid, kPushSentinel); st_relaxed_u32(vo + TG_P2 + 2 * c + tid, kPushSentinel); }
      if (tid < 4) { st_relaxed_u32(vo + TG_L1 + 4 * c + tid, kPushSentinel); st_relaxed_u32(vo + TG_L2 + 4 * c + tid, kPushSentinel);
                     st_relaxed_u32(vo + TG_CTX + 4 * c + tid, kPushSentinel); }
      for (int i = tid; i < Txp; i += kTgThreads) st_relaxed_u32(vo + TG_EN + (size_t)c * Txp + i, kPushSentinel);
      if (tid < Txp || tid < 4) asm volatile("fence.acq_rel.gpu;" ::: "memory");
    }
    tg_matvec<2>(Wb + Md.oW2, Wb + Md.oB2, p1, P, outv, part);
    if (tid < 2) {
      const int j = 2 * c + tid;
      float keep;
      if (A.rng_mode == 0) {
        keep = taco_keep_flag(A.seed, A.utt, step, 1, j, P) ? 1.f : 0.f;
      } else {
        keep = A.masks[((size_t)step * 2 + 1) * P + j] ? 1.f : 0.f;
      }
      st_relaxed_f32(vw + TG_P2 + j, fmaxf(outv[tid], 0.f) * keep * 2.0f);
    }
    // ---------------- E2 + S3: LSTM 1 on [prenet | context | h1] ----------------
    tg_gather(vw + TG_P2, P / 4, pg, [&](int i, float4 v) { reinterpret_cast<float4*>(in1)[i] = v; });
    if (__syncthreads_or(pg.aborted ? 1 : 0)) return;
    tg_matvec<8>(Wb + Md.oK1, Wb + Md.oBk1, in1, P + E + U, outv, part);
    if (tid < 2) {
      const float i_ = outv[tid], j_ = outv[2 + tid], f_ = outv[4 + tid], o_ = outv[6 + tid];
      const float cn = sigmoidf_acc(f_ + 1.0f) * s_c1[tid] + sigmoidf_acc(i_) * tanhf(j_);
      const float hn = sigmoidf_acc(o_) * tanhf(cn);
      s_c1[tid] = zk * cn + zr * s_c1[tid];                 // zoneout at inference, modules.py:137-138
      const float hz = zk * hn + zr * s_h1[tid];
      s_h1[tid] = hz;
      st_relaxed_f32(vw + TG_L1 + 4 * c + tid, hn);          // the cell OUTPUT is the un-zoned new_h (:118,:142)
      st_relaxed_f32(vw + TG_L1 + 4 * c + 2 + tid, hz);
    }
    // ---------------- E3 + S4: LSTM 2 on [o1 | h2] ----------------
    tg_gather(vw + TG_L1, U / 2, pg, [&](int i, float4 v) {
      in2[2 * i] = v.x; in2[2 * i + 1] = v.y;               // o1 of units 2i, 2i+1
      in1[P + E + 2 * i] = v.z; in1[P + E + 2 * i + 1] = v.w;   // zoned h1 for the next step
    });
    if (__syncthreads_or(pg.aborted ? 1 : 0)) return;
    tg_matvec<8>(Wb + Md.oK2, Wb + Md.oBk2, in2, 2 * U, outv, part);
    if (tid < 2) {
      const float i_ = outv[tid], j_ = outv[2 + tid], f_ = outv[4 + tid], o_ = outv[6 + tid];
      const float cn = sigmoidf_acc(f_ + 1.0f) * s_c2[tid] + sigmoidf_acc(i_) * tanhf(j_);
      const float hn = sigmoidf_acc(o_) * tanhf(cn);
      s_c2[tid] = zk * cn + zr * s_c2[tid];
      const float hz = zk * hn + zr * s_h2[tid];
      s_h2[tid] = hz;
      st_relaxed_f32(vw + TG_L2 + 4 * c + tid, hn);
      st_relaxed_f32(vw + TG_L2 + 4 * c + 2 + tid, hz);
    }
    // ---------------- E4 + S5: query dimension c, partial energies of every position ----------------
    tg_gather(vw + TG_L2, U / 2, pg, [&](int i, float4 v) {
      pin[2 * i] = v.x; pin[2 * i + 1] = v.y;               // o2 = query and first part of the projection input
      in2[U + 2 * i] = v.z; in2[U + 2 * i + 1] = v.w;       // zoned h2 for the next step
    });
    if (__syncthreads_or(pg.aborted ? 1 : 0)) return;
    tg_matvec<1>(Wb + Md.oWq, nullptr, pin, U, outv, part);
    {
      const float q_c = outv[0];
      for (int t = tid; t < Txp; t += kTgThreads) {
        float e = 0.f;
        if (t < Tx) {
          float loc = bloc;                                  // location features of dimension c: folded conv (31 taps) . W_l, 'same'
          for (int k = 0; k < KW; ++k) {
            const int tt = t + k - (KW - 1) / 2;
            if (tt >= 0 && tt < Tx) loc = fmaf(wfloc[k], cum[tt], loc);
          }
          e = v_c * tanhf(keyc[t] + q_c + loc);
        }
        st_relaxed_f32(vw + TG_EN + (size_t)c * Txp + t, e);
      }
    }
    // ---------------- E6 + S6: energies = sum over the 128 dimensions (producer order), softmax, forward recursion ----------------
    {
      const int n4 = Txp / 4;                                // float4 columns per producer
      const int q = tid / n4, col = tid - q * n4;            // 16 producer queues of 8 producers each
      if (q < 16 && n4 <= 32) {
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float* src = vw + TG_EN + (size_t)(q * 8 + i) * Txp + col * 4;
          float4 v = ld_relaxed_f4(src);
          if (!f4_ready(v)) {
            pg.begin();
            while (!pg.aborted) { v = ld_relaxed_f4(src); if (f4_ready(v) || pg.expired()) break; }
          }
          s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
        }
        reinterpret_cast<float4*>(epart + (size_t)q * Txp)[col] = s;
      } else if (n4 > 32) {                                  // long inputs: every thread walks several (queue, column) pairs
        for (int it = tid; it < 16 * n4; it += kTgThreads) {
          const int qq = it / n4, cc4 = it - qq * n4;
          float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
          for (int i = 0; i < 8; ++i) {
            const float* src = vw + TG_EN + (size_t)(qq * 8 + i) * Txp + cc4 * 4;
            float4 v = ld_relaxed_f4(src);
            if (!f4_ready(v)) {
              pg.begin();
              while (!pg.aborted) { v = ld_relaxed_f4(src); if (f4_ready(v) || pg.expired()) break; }
            }
            s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
          }
          reinterpret_cast<float4*>(epart + (size_t)qq * Txp)[cc4] = s;
        }
      }
    }
    if (__syncthreads_or(pg.aborted ? 1 : 0)) return;
    float ev = -INFINITY;
    for (int t = tid; t < Tx; t += kTgThreads) {
      float e = 0.f;
#pragma unroll
      for (int q = 0; q < 16; ++q) e += epart[(size_t)q * Txp + t];
      al[t] = e;
      ev = fmaxf(ev, e);
    }
    const float emax = tg_block_max(ev, red);
    float es = 0.f;
    for (int t = tid; t < Tx; t += kTgThreads) { const float e = expf(al[t] - emax); al[t] = e; es += e; }
    const float esum = tg_block_sum(es, red);
    float mu = s_mu;
    if constexpr (kBias) mu = fmaxf(fminf(__fadd_rn(mu, dmu), 1.f), 0.f);   // tf.clip_by_value(mu + delta, 0, 1): min, then max
    __syncthreads();
    float fs = 0.f;
    for (int t = tid; t < Tx; t += kTgThreads) {
      const float a = al[t] / esum;
      cum[t] += a;                                                             // attention.py:154
      const float sh = t > 0 ? alpha[t - 1] : 0.f;
      const float v = ((1.f - mu) * alpha[t] + mu * sh + 1e-10f) * a;          // attention.py:167
      al[t] = v;
      fs += v;
    }
    __syncthreads();
    if (A.window) {                                                            // forward_attention.py:171-215
      if (tid == 0) {
        int am = 0; float best = al[0];
        for (int t = 1; t < Tx; ++t) if (al[t] > best) { best = al[t]; am = t; }
        int nm = (am <= s_max) ? s_max : s_max + 1;
        if (s_pos < 5 && 2 < nm) nm = s_max;
        int pr = (nm == s_max) ? s_pos + 1 : 1;
        if (!(pr < 10)) { nm = nm + 1; pr = 1; }
        s_max = nm; s_pos = pr;
      }
      __syncthreads();
      const int nm = s_max;
      float ws = 0.f;
      for (int t = tid; t < Tx; t += kTgThreads) {
        if (!(t >= nm - 2 && t < nm + 3)) al[t] = 0.f;
        ws += al[t];
      }
      const float wsum = tg_block_sum(ws, red);
      __syncthreads();
      if (tid == 0) { const int pk = min(max(nm, 0), Tx - 1); al[pk] = (wsum < 1e-10f ? 1.0f : wsum) * 2.0f; }
      __syncthreads();
      fs = 0.f;
      for (int t = tid; t < Tx; t += kTgThreads) fs += al[t];
    }
    const float fsum = tg_block_sum(fs, red);
    float cx[4] = {0.f, 0.f, 0.f, 0.f};
    for (int t = tid; t < Tx; t += kTgThreads) {
      const float v = al[t] / fsum;                                            // attention.py:220
      alpha[t] = v;
      if (A.align && c == 0) A.align[(size_t)step * A.Tx_alloc + t] = v;
      const float4 m = reinterpret_cast<const float4*>(memc)[t];
      cx[0] = fmaf(v, m.x, cx[0]); cx[1] = fmaf(v, m.y, cx[1]); cx[2] = fmaf(v, m.z, cx[2]); cx[3] = fmaf(v, m.w, cx[3]);
    }
    // context columns 4c ... 4c+3 = al . memory (attention.py:222): shuffle tree, then the 16 warps in order
#pragma unroll
    for (int j = 0; j < 4; ++j) cx[j] = warp_sum(cx[j]);
    __syncthreads();
    if ((tid & 31) == 0) {
#pragma unroll
      for (int j = 0; j < 4; ++j) part[(tid >> 5) * 4 + j] = cx[j];
    }
    __syncthreads();
    if (tid < 4) {
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < kTgWarps; ++w) v += part[w * 4 + tid];
      st_relaxed_f32(vw + TG_CTX + 4 * c + tid, v);
    }
    // ---------------- E8 + S7: context everywhere; mu gate, stop token, mel column ----------------
    tg_gather(vw + TG_CTX, E / 4, pg, [&](int i, float4 v) {
      reinterpret_cast<float4*>(in1 + P)[i] = v;
      reinterpret_cast<float4*>(pin + U)[i] = v;
    });
    if (__syncthreads_or(pg.aborted ? 1 : 0)) return;
    tg_matvec<4>(Wb + Md.oProj, Wb + Md.oProj + 4 * (U + E), pin, U + E, outv, part);
    if (tid == 0) {
      s_mu = sigmoidf_acc(outv[0]);                                           // attention.py:229
      s_stop = sigmoidf_acc(outv[1]);                                         // Architecture_wrappers.py:196-199
      if (c < M) A.frames[(size_t)step * M + c] = outv[2];
      if (c == 0) A.stop[step] = s_stop;
    }
    __syncthreads();
    if (s_stop > 0.5f && !A.forced) { ++step; break; }     // finished = round(stop) (half-to-even -> strictly > 0.5)
  }
  if (tid == 0 && c == 0) A.nsteps[0] = step;
}

__global__ void __launch_bounds__(kTgThreads, 1) taco_grid_kernel(TacoGridModel Md, TacoGridArgs A) {
  taco_grid_run<false>(Md, A, nullptr);
}

// one sentence with a speaking-rate bias: mu_bias [1] (b200tts_taco_decode_biased)
__global__ void __launch_bounds__(kTgThreads, 1) taco_grid_biased_kernel(TacoGridModel Md, TacoGridArgs A, const float* mu_bias) {
  taco_grid_run<true>(Md, A, mu_bias);
}

// a poll that timed out leaves the outputs half written: mark the sentence as failed instead of returning a plausible step count
__global__ void taco_grid_finish_kernel(const int* __restrict__ error, int* __restrict__ nsteps) {
  if (*error) nsteps[0] = -1;
}

// dynamic shared memory of taco_grid_kernel for a sentence buffer of Txp (Tx rounded up to 4) positions
inline size_t taco_grid_smem_bytes(const TacoGridModel& g, int Txp) {
  const size_t fl = (size_t)g.blob + (size_t)(g.P + g.E + g.U) + 2 * g.U + (g.U + g.E) + g.P + 128 + 24 * (size_t)Txp + 176;
  return fl * sizeof(float);
}

// ---- host: the per-block weight blobs [128][blob], cut from the batch decoder's weights in their original layouts (`w` points
//      to host memory).  Fills the layout `g`; the blobs are empty when the model or device cannot run this kernel. -----------
inline std::vector<float> pack_taco_grid_model(const TacoWeights& w, int sm_count, bool coop, TacoGridModel& g) {
  const int M = w.mels, P = w.P, U = w.U, E = w.E, AD = w.A, NF = w.NF, KW = w.KW;
  g = TacoGridModel{};
  if (!(coop && sm_count >= kTgCtas && P == 256 && U == 256 && E == 512 && AD == 128 && M <= 96 && KW <= 64)) return {};
  g.M = M; g.P = P; g.U = U; g.E = E; g.KW = KW;
  int off = 0;
  auto take = [&](int n) { int o0 = off; off += (n + 3) & ~3; return o0; };
  g.oW1 = take(M * 2); g.oB1 = take(2);
  g.oWfold = take((U + E) * 2); g.oBfold = take(2);
  g.oW2 = take(P * 2); g.oB2 = take(2);
  g.oK1 = take((P + E + U) * 8); g.oBk1 = take(8);
  g.oK2 = take(2 * U * 8); g.oBk2 = take(8);
  g.oWq = take(U);
  g.oFloc = take(KW + 4);
  g.oProj = take((U + E) * 4 + 4);
  g.blob = off;
  const float *W1 = w.pre1_k, *b1 = w.pre1_b, *W2 = w.pre2_k, *b2 = w.pre2_b, *K1 = w.l1_k, *bk1 = w.l1_b, *K2 = w.l2_k,
              *bk2 = w.l2_b, *Wq = w.q_k, *lock = w.loc_k, *locb = w.loc_b, *locl = w.locl_k, *va = w.v_a, *ba = w.b_a,
              *muk = w.mu_k, *mub = w.mu_b, *frk = w.fr_k, *frb = w.fr_b, *stk = w.st_k, *stb = w.st_b;
  // W_f . W_1 and b_f . W_1 + b_1 in float64
  std::vector<double> fold((size_t)(U + E) * P), bfold(P);
  for (int i = 0; i < U + E; ++i)
    for (int p2 = 0; p2 < P; ++p2) {
      double a = 0;
      for (int m = 0; m < M; ++m) a += (double)frk[(size_t)i * M + m] * (double)W1[(size_t)m * P + p2];
      fold[(size_t)i * P + p2] = a;
    }
  for (int p2 = 0; p2 < P; ++p2) {
    double a = b1[p2];
    for (int m = 0; m < M; ++m) a += (double)frb[m] * (double)W1[(size_t)m * P + p2];
    bfold[p2] = a;
  }
  std::vector<float> hb((size_t)kTgCtas * g.blob, 0.f);
  for (int c2 = 0; c2 < kTgCtas; ++c2) {
    float* d = &hb[(size_t)c2 * g.blob];
    for (int j = 0; j < 2; ++j) {
      const int col = 2 * c2 + j;
      for (int m = 0; m < M; ++m) d[g.oW1 + m * 2 + j] = W1[(size_t)m * P + col];
      d[g.oB1 + j] = b1[col];
      for (int i = 0; i < U + E; ++i) d[g.oWfold + i * 2 + j] = (float)fold[(size_t)i * P + col];
      d[g.oBfold + j] = (float)bfold[col];
      for (int k = 0; k < P; ++k) d[g.oW2 + k * 2 + j] = W2[(size_t)k * P + col];
      d[g.oB2 + j] = b2[col];
      for (int gate = 0; gate < 4; ++gate) {
        const int src = gate * U + col, dst = gate * 2 + j;
        for (int k = 0; k < P + E + U; ++k) d[g.oK1 + k * 8 + dst] = K1[(size_t)k * 4 * U + src];
        d[g.oBk1 + dst] = bk1[src];
        for (int k = 0; k < 2 * U; ++k) d[g.oK2 + k * 8 + dst] = K2[(size_t)k * 4 * U + src];
        d[g.oBk2 + dst] = bk2[src];
      }
    }
    for (int u = 0; u < U; ++u) d[g.oWq + u] = Wq[(size_t)u * AD + c2];
    double bl = ba[c2];
    for (int f = 0; f < NF; ++f) bl += (double)locb[f] * (double)locl[(size_t)f * AD + c2];
    for (int k = 0; k < KW; ++k) {
      double a = 0;
      for (int f = 0; f < NF; ++f) a += (double)lock[(size_t)k * NF + f] * (double)locl[(size_t)f * AD + c2];
      d[g.oFloc + k] = (float)a;
    }
    d[g.oFloc + KW] = (float)bl;
    d[g.oFloc + KW + 1] = va[c2];
    d[g.oFloc + KW + 2] = 1.0f - w.zoneout;
    d[g.oFloc + KW + 3] = w.zoneout;
    for (int i = 0; i < U + E; ++i) {
      d[g.oProj + i * 4 + 0] = muk[i < U ? E + i : i - U];          // attention.py:229 concatenates [context, query]
      d[g.oProj + i * 4 + 1] = stk[i];
      d[g.oProj + i * 4 + 2] = c2 < M ? frk[(size_t)i * M + c2] : 0.f;
    }
    d[g.oProj + (U + E) * 4 + 0] = mub[0];
    d[g.oProj + (U + E) * 4 + 1] = stb[0];
    d[g.oProj + (U + E) * 4 + 2] = c2 < M ? frb[c2] : 0.f;
  }
  return hb;
}

}  // namespace b200tts
