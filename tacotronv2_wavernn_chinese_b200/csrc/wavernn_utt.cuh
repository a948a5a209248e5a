// WaveRNN per-sample recurrence, "utterance" kernel: one persistent CTA owns G utterances for the whole
// sequence; the 17.4 MB of fp32 step weights are streamed from L2 every step (they do not fit one SM).
//
// Replaces the hot loop of WaveRNN.generate, reference wavernn/models/fatchord_version.py:201-237:
//   I (:208-209) -> GRUCell rnn1 (:210) -> +res (:212) -> GRUCell rnn2 (:213-214) -> +res (:216)
//   -> relu fc1 (:217-218) -> relu fc2 (:220-221) -> fc3 (:223) -> softmax + Categorical.sample (:232-235)
//   -> x = 2*label/1023 - 1 (:235-237); or, for MOL models, sample_from_discretized_mix_logistic (:225-229).
// This kernel keeps the reference's operation structure one to one (no algebraic folding), takes the debug
// options (teacher forcing, logits dump) and serves as the on-device cross-check of the grid kernel.
#pragma once
#include "common.cuh"

namespace b200tts {

struct StepWeights {          // original row-major layouts (rows padded to a multiple of 4 floats where noted)
  const float* I_w;           // [R][ldI]   ldI = roundup4(1 + feat + aux)
  const float* I_b;           // [R]
  const float* ih1_w;         // [3R][R]
  const float* hh1_w;         // [3R][R]
  const float* ih1_b;         // [3R]
  const float* hh1_b;         // [3R]
  const float* ih2_w;         // [3R][R + aux]
  const float* hh2_w;         // [3R][R]
  const float* ih2_b;
  const float* hh2_b;
  const float* fc1_w;         // [F][R + aux]
  const float* fc1_b;
  const float* fc2_w;         // [F][F + aux]
  const float* fc2_b;
  const float* fc3_w;         // [NC][F]
  const float* fc3_b;
  int R, F, aux, feat, NC, ldI;
};

struct GenArgs {
  const float* mels_up;       // [B][S][feat]
  const float* aux_frames;    // [B][T][4*aux]
  int B, S, T, hop;
  int steps;                  // number of steps to run (<= S)
  int rng_mode;
  unsigned long long seed, utt_offset;
  const unsigned long long* utt_ids;   // optional [B]: global utterance index of every row (overrides utt_offset + row)
  const float* q;             // [S][B][NC] (EXT_EXPONENTIAL); [S][B][11] uniforms (EXT_UNIFORM, MOL)
  const int16_t* teacher;     // [B][S] or null
  float* logits_out;          // [S][B][NC] or null
  int16_t* labels;            // [B][S]
};

constexpr int kUttThreads = 512;

// dot products of NR weight rows with G smem vectors; the warp cooperates, lanes stride over float4 columns.
template <int NR, int G>
__device__ __forceinline__ void warp_rows_dot(const float* __restrict__ W, int ldw, const int (&rows)[NR], const float* x,
                                              int ldx, int K4, int lane, float (&out)[NR][G]) {
  float acc[NR][G];
#pragma unroll
  for (int r = 0; r < NR; ++r)
#pragma unroll
    for (int g = 0; g < G; ++g) acc[r][g] = 0.f;
  for (int k4 = lane; k4 < K4; k4 += 32) {
    float4 xv[G];
#pragma unroll
    for (int g = 0; g < G; ++g) xv[g] = reinterpret_cast<const float4*>(x + (size_t)g * ldx)[k4];
#pragma unroll
    for (int r = 0; r < NR; ++r) {
      float4 w = __ldg(reinterpret_cast<const float4*>(W + (size_t)rows[r] * ldw) + k4);
#pragma unroll
      for (int g = 0; g < G; ++g) {
        acc[r][g] = fmaf(w.x, xv[g].x, acc[r][g]);
        acc[r][g] = fmaf(w.y, xv[g].y, acc[r][g]);
        acc[r][g] = fmaf(w.z, xv[g].z, acc[r][g]);
        acc[r][g] = fmaf(w.w, xv[g].w, acc[r][g]);
      }
    }
  }
#pragma unroll
  for (int r = 0; r < NR; ++r)
#pragma unroll
    for (int g = 0; g < G; ++g) out[r][g] = warp_sum(acc[r][g]);
}

// Host side: the floats of dynamic shared memory utt_run<G, *> carves up below, buffer by buffer.
inline size_t utt_smem_floats(const StepWeights& W, int G) {
  const int KX = W.R + W.aux, KF = W.F + W.aux;
  return (size_t)G * (W.ldI + W.R + 2 * W.R + 2 * W.R + KX + KX + KF + W.F + W.NC);
}

// Host side: whether G rows per CTA fit the 227 KB of shared memory a CTA may have, the static `red` array of utt_run included.
inline bool utt_fits(const StepWeights& W, int G) {
  return utt_smem_floats(W, G) * sizeof(float) + (size_t)G * (kUttThreads / 32) * sizeof(unsigned long long) <= 227 * 1024;
}

// The whole loop; MOL selects the sampler (fc3 then has NC = 32 rows, the 30 parameters padded to whole quads).
template <int G, bool MOL>
__device__ __forceinline__ void utt_run(StepWeights W, GenArgs A, MolIO M) {
  extern __shared__ __align__(16) float sm[];
  const int R = W.R, F = W.F, AUX = W.aux, NC = W.NC, ldI = W.ldI;
  const int KX = R + AUX;                       // 544
  // ---- shared memory carve-up (all row strides multiples of 4 floats) ----
  float* xin = sm;                              // [G][ldI]     x | m_t | a1
  float* xi = xin + G * ldI;                    // [G][R]       I output
  float* h1 = xi + G * R;                       // [2][G][R]
  float* h2 = h1 + 2 * G * R;                   // [2][G][R]
  float* in2 = h2 + 2 * G * R;                  // [G][KX]      (xi + h1') | a2
  float* in3 = in2 + G * KX;                    // [G][KX]      (.. + h2') | a3
  const int KF = F + AUX;
  float* in4 = in3 + G * KX;                    // [G][KF]      relu fc1  | a4
  float* f2 = in4 + G * KF;                     // [G][F]
  float* lg = f2 + G * F;                       // [G][NC]
  __shared__ unsigned long long red[G][kUttThreads / 32];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, NW = kUttThreads / 32;
  const int b0 = blockIdx.x * G;
  const float ncls_m1 = (float)(NC - 1);

  for (int e = tid; e < G * ldI; e += kUttThreads) xin[e] = 0.f;
  for (int e = tid; e < 2 * G * R; e += kUttThreads) { h1[e] = 0.f; h2[e] = 0.f; }
  __syncthreads();

  int cur = 0;
  for (int i = 0; i < A.steps; ++i) {
    // ---- conditioning of this step: m_t -> xin[1..feat], a1 -> xin[1+feat..], a2/a3/a4 -> tails ----
    const int fr = i / A.hop;
    for (int e = tid; e < G * (W.feat + 4 * AUX); e += kUttThreads) {
      int g = e / (W.feat + 4 * AUX), c = e % (W.feat + 4 * AUX);
      int b = b0 + g;
      float v = 0.f;
      if (b < A.B) {
        v = (c < W.feat) ? A.mels_up[((size_t)b * A.S + i) * W.feat + c]
                         : A.aux_frames[((size_t)b * A.T + fr) * (4 * AUX) + (c - W.feat)];
      }
      if (c < W.feat + AUX) xin[g * ldI + 1 + c] = v;
      else if (c < W.feat + 2 * AUX) in2[g * KX + R + (c - W.feat - AUX)] = v;
      else if (c < W.feat + 3 * AUX) in3[g * KX + R + (c - W.feat - 2 * AUX)] = v;
      else in4[g * KF + F + (c - W.feat - 3 * AUX)] = v;
    }
    __syncthreads();
    // ---- I: R rows x ldI ----
    for (int r0 = warp * 4; r0 < R; r0 += NW * 4) {
      int rows[4] = {r0, r0 + 1, r0 + 2, r0 + 3};
      float o[4][G];
      warp_rows_dot<4, G>(W.I_w, ldI, rows, xin, ldI, ldI / 4, lane, o);
      if (lane == 0) {
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int g = 0; g < G; ++g) xi[g * R + r0 + r] = o[r][g] + W.I_b[r0 + r];
      }
    }
    __syncthreads();
    // ---- GRU 1 (torch GRUCell, gate rows r,z,n) ----
    {
      const float* hc = h1 + cur * G * R;
      float* hn = h1 + (cur ^ 1) * G * R;
      for (int j = warp; j < R; j += NW) {
        int rows[3] = {j, R + j, 2 * R + j};
        float gi[3][G], gh[3][G];
        warp_rows_dot<3, G>(W.ih1_w, R, rows, xi, R, R / 4, lane, gi);
        warp_rows_dot<3, G>(W.hh1_w, R, rows, hc, R, R / 4, lane, gh);
        if (lane == 0) {
#pragma unroll
          for (int g = 0; g < G; ++g) {
            float r = sigmoidf_acc((gi[0][g] + W.ih1_b[j]) + (gh[0][g] + W.hh1_b[j]));
            float z = sigmoidf_acc((gi[1][g] + W.ih1_b[R + j]) + (gh[1][g] + W.hh1_b[R + j]));
            float n = tanhf((gi[2][g] + W.ih1_b[2 * R + j]) + r * (gh[2][g] + W.hh1_b[2 * R + j]));
            float h = (1.0f - z) * n + z * hc[g * R + j];
            hn[g * R + j] = h;
            in2[g * KX + j] = xi[g * R + j] + h;
          }
        }
      }
    }
    __syncthreads();
    // ---- GRU 2 ----
    {
      const float* hc = h2 + cur * G * R;
      float* hn = h2 + (cur ^ 1) * G * R;
      for (int j = warp; j < R; j += NW) {
        int rows[3] = {j, R + j, 2 * R + j};
        float gi[3][G], gh[3][G];
        warp_rows_dot<3, G>(W.ih2_w, KX, rows, in2, KX, KX / 4, lane, gi);
        warp_rows_dot<3, G>(W.hh2_w, R, rows, hc, R, R / 4, lane, gh);
        if (lane == 0) {
#pragma unroll
          for (int g = 0; g < G; ++g) {
            float r = sigmoidf_acc((gi[0][g] + W.ih2_b[j]) + (gh[0][g] + W.hh2_b[j]));
            float z = sigmoidf_acc((gi[1][g] + W.ih2_b[R + j]) + (gh[1][g] + W.hh2_b[R + j]));
            float n = tanhf((gi[2][g] + W.ih2_b[2 * R + j]) + r * (gh[2][g] + W.hh2_b[2 * R + j]));
            float h = (1.0f - z) * n + z * hc[g * R + j];
            hn[g * R + j] = h;
            in3[g * KX + j] = in2[g * KX + j] + h;
          }
        }
      }
    }
    __syncthreads();
    // ---- fc1 / fc2 (relu) ----
    for (int r0 = warp * 4; r0 < F; r0 += NW * 4) {
      int rows[4] = {r0, r0 + 1, r0 + 2, r0 + 3};
      float o[4][G];
      warp_rows_dot<4, G>(W.fc1_w, KX, rows, in3, KX, KX / 4, lane, o);
      if (lane == 0) {
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int g = 0; g < G; ++g) in4[g * KF + r0 + r] = fmaxf(o[r][g] + W.fc1_b[r0 + r], 0.f);
      }
    }
    __syncthreads();
    for (int r0 = warp * 4; r0 < F; r0 += NW * 4) {
      int rows[4] = {r0, r0 + 1, r0 + 2, r0 + 3};
      float o[4][G];
      warp_rows_dot<4, G>(W.fc2_w, KF, rows, in4, KF, KF / 4, lane, o);
      if (lane == 0) {
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int g = 0; g < G; ++g) f2[g * F + r0 + r] = fmaxf(o[r][g] + W.fc2_b[r0 + r], 0.f);
      }
    }
    __syncthreads();
    // ---- fc3 -> logits ----
    for (int r0 = warp * 4; r0 < NC; r0 += NW * 4) {
      int rows[4] = {r0, r0 + 1, r0 + 2, r0 + 3};
      float o[4][G];
      warp_rows_dot<4, G>(W.fc3_w, F, rows, f2, F, F / 4, lane, o);
      if (lane == 0) {
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int g = 0; g < G; ++g) lg[g * NC + r0 + r] = o[r][g] + W.fc3_b[r0 + r];
      }
    }
    __syncthreads();
    if constexpr (MOL) {
      // ---- sample_from_discretized_mix_logistic, one thread per row (distribution.py:87-123, fatchord_version.py:225-229) ----
      if (tid < G && b0 + tid < A.B) {
        const int g = tid, b = b0 + g;
        float u[kMolU];
        if (A.rng_mode == 0) {
          philox_mol_u(A.seed, A.utt_ids ? A.utt_ids[b] : A.utt_offset + (unsigned long long)b, (uint32_t)i, u);
        } else {
#pragma unroll
          for (int j = 0; j < kMolU; ++j) u[j] = A.q[((size_t)i * A.B + b) * kMolU + j];
        }
        const float* p = lg + g * NC;
        if (A.logits_out)
          for (int j = 0; j < kMolParams; ++j) A.logits_out[((size_t)i * A.B + b) * kMolParams + j] = p[j];
        const float x = mol_sample(p, u);
        M.samples[(size_t)b * A.S + i] = x;
        xin[g * ldI] = M.teacher_x ? M.teacher_x[(size_t)b * A.S + i] : x;
      }
    } else {
      // ---- sample: argmax_c (logit_c - log q_c), q ~ Exp(1)  == Categorical(softmax(logits)).sample() ----
#pragma unroll
      for (int g = 0; g < G; ++g) {
        const int b = b0 + g;
        unsigned long long best = 0ull;
        if (b < A.B) {
          for (int c4 = tid; c4 < NC / 4; c4 += kUttThreads) {
            float q[4];
            if (A.rng_mode == 0) {
              philox_exp4(A.seed, A.utt_ids ? A.utt_ids[b] : A.utt_offset + (unsigned long long)b, (uint32_t)i, (uint32_t)c4, q);
            } else {
              float4 qv = *reinterpret_cast<const float4*>(A.q + ((size_t)i * A.B + b) * NC + c4 * 4);
              q[0] = qv.x; q[1] = qv.y; q[2] = qv.z; q[3] = qv.w;
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              float l = lg[g * NC + c4 * 4 + u];
              if (A.logits_out) A.logits_out[((size_t)i * A.B + b) * NC + c4 * 4 + u] = l;
              unsigned long long p = pack_key(l - logf(q[u]), (uint32_t)(c4 * 4 + u));
              best = p > best ? p : best;
            }
          }
        }
        best = warp_max_u64(best);
        if (lane == 0) red[g][warp] = best;
      }
      __syncthreads();
      if (warp == 0) {
#pragma unroll
        for (int g = 0; g < G; ++g) {
          unsigned long long v = lane < NW ? red[g][lane] : 0ull;
          v = warp_max_u64(v);
          if (lane == 0) {
            const int b = b0 + g;
            int label = (int)unpack_idx(v);
            if (b < A.B) {
              A.labels[(size_t)b * A.S + i] = (int16_t)label;
              int fb = A.teacher ? (int)A.teacher[(size_t)b * A.S + i] : label;
              xin[g * ldI] = label_to_float(fb, ncls_m1);
            }
          }
        }
      }
    }
    cur ^= 1;
    __syncthreads();
  }
}

template <int G>
__global__ void __launch_bounds__(kUttThreads, 1) wavernn_utt_kernel(StepWeights W, GenArgs A) {
  utt_run<G, false>(W, A, MolIO{});
}

template <int G>
__global__ void __launch_bounds__(kUttThreads, 1) wavernn_utt_mol_kernel(StepWeights W, GenArgs A, MolIO M) {
  utt_run<G, true>(W, A, M);
}

}  // namespace b200tts
