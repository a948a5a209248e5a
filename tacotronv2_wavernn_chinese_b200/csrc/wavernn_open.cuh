// Batched, ragged open of generation sessions (b200tts_wavernn_session_open_batch): n mels of their own frame counts become n
// sessions' conditioning tables in three launches, whatever n is.
//   session_mel_prep_kernel        each row's mel in [0, 1], zero-padded to the session's T = max(frames, 21), packed
//                                  back to back ([feat][T] per row, row r from frame f0[r]);
//   melresnet_ragged_kernel<FT>    MelResNet over every row's tiles (melresnet_tile, as melresnet_kernel runs one row);
//   push_cond_table_ragged_kernel  every row's [T+1][ncta][52] table (push_cond_table_tile), into the session's memory.
// A tile of either ragged kernel finds its row by a binary search over the prefix sums of tiles per row, then computes exactly
// what melresnet_kernel / push_cond_table_kernel compute for that tile of a one-row launch: same statements, same operands.
#pragma once
#include "wavernn_push.cuh"
#include "wavernn_upsample.cuh"

namespace b200tts {

constexpr int kOpenMaxRows = 256;   // kTcSessRows: the most sessions one run takes
constexpr int kOpenFT = 8;          // frames per CTA of MelResNet and the tables, as one-shot generation launches them

struct OpenRows {                   // passed by value (6 KB of kernel parameters)
  int n;
  int frames[kOpenMaxRows];         // frames of row r's mel as given (1..T_max)
  int T[kOpenMaxRows];              // frames of its session, max(frames, 21)
  int f0[kOpenMaxRows + 1];         // first frame of row r in the packed mel [feat][T] and aux [T][O] buffers
  int res0[kOpenMaxRows + 1];       // first MelResNet tile of row r: prefix sums of ceil(T / FT)
  int tab0[kOpenMaxRows + 1];       // first table tile of row r: prefix sums of ceil((T + 1) / FT)
  float* tab[kOpenMaxRows];         // row r's session table [T+1][ncta][52]
};

// The row whose tiles [start[r], start[r + 1]) hold tile x.
__device__ __forceinline__ int open_row(const int* start, int n, int x) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (start[mid] <= x) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// layout 0: src [n][feat][T_max], already in [0, 1].  layout 1: src [n][T_max][feat], the Tacotron postnet output, mapped with
// the float32 statements of Synthesizer.mels: m = clip(m, -a, a), then clip((m + a) / (2a), 0, 1).  Frames past the row's own
// count are zero in the [0, 1] domain.  Grid (x, n).
__global__ void session_mel_prep_kernel(const float* __restrict__ src, int layout, int T_max, int feat, float max_abs, OpenRows R,
                                        float* __restrict__ dst) {
  const int r = blockIdx.y, T = R.T[r], nf = R.frames[r];
  float* d = dst + (size_t)R.f0[r] * feat;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < feat * T; e += gridDim.x * blockDim.x) {
    const int k = e / T, t = e % T;
    float v = 0.f;
    if (t < nf) {
      if (layout == 0) {
        v = src[((size_t)r * feat + k) * T_max + t];
      } else {
        const float m = fminf(fmaxf(src[((size_t)r * T_max + t) * feat + k], -max_abs), max_abs);
        v = fminf(fmaxf(__fdiv_rn(__fadd_rn(m, max_abs), __fmul_rn(2.f, max_abs)), 0.f), 1.f);
      }
    }
    d[e] = v;
  }
}

template <int FT>
__global__ void melresnet_ragged_kernel(ResnetParams P, const float* __restrict__ mel /*packed [feat][T] rows*/, OpenRows R,
                                        float* __restrict__ aux_frames /*packed [T][O] rows*/) {
  const int r = open_row(R.res0, R.n, blockIdx.x);
  melresnet_tile<FT>(P, mel + (size_t)R.f0[r] * P.feat, R.T[r], 0, (blockIdx.x - R.res0[r]) * FT,
                     aux_frames + (size_t)R.f0[r] * P.O);
}

template <int FT>
__global__ void push_cond_table_ragged_kernel(PushCondW W, const float* __restrict__ mel, const float* __restrict__ aux_frames,
                                              OpenRows R) {
  const int r = open_row(R.tab0, R.n, blockIdx.x);
  push_cond_table_tile<FT>(W, mel + (size_t)R.f0[r] * W.feat, aux_frames + (size_t)R.f0[r] * 4 * W.aux, 1, R.T[r], 0,
                           (blockIdx.x - R.tab0[r]) * FT, R.tab[r]);
}

}  // namespace b200tts
