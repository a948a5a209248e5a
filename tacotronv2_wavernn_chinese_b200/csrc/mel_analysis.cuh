// Mel analysis: the reference's feature extraction (tacotron/datasets/preprocessor.py:52-121 _process_utterance_v1, and
// tacotron/datasets/audio.py:71-77 trim_silence (librosa 0.7.2 effects.trim), :47-50 preemphasis, :95-102 melspectrogram,
// :203-207 _stft, :250-254 _linear_to_mel, :273-275 _amp_to_db, :283-295 _normalize).  Four kernels:
//   ma_trim_power_kernel  one warp per (row, trim frame): mean square of the reflect-padded 2048-sample frame, fp64
//   ma_bounds_kernel      one CTA per row: loudest trim frame, threshold, first / last non-silent frame -> [s, e); then the
//                         peaks max|wav[s:e]| and max|preemphasis(wav[s:e])| the rescale divides by; frame count T
//   ma_frame_kernel       one CTA per (row, frame): gather the frame's win_size windowed samples of the (pre-emphasised,
//                         rescaled) trimmed signal, 2048-point rfft, |X|^p, mel projection, dB, symmetric normalisation
//   ma_audio_kernel       the rescaled trimmed wav zero-padded to T * hop samples (the training audio `out`)
// Pre-emphasis is never materialised: p[n] = x[n] + (-k) x[n-1] (x[-1] = 0) is recomputed in fp64 where it is needed, with
// the roundings scipy's lfilter makes, so the STFT input equals the reference's float64 signal until the gathered frame is
// rounded to fp32.  The FFT is fft2048.cuh's.  No atomics: every value depends on its own row only.
#pragma once
#include <climits>

#include "common.cuh"
#include "fft2048.cuh"

namespace b200tts {

constexpr int kMaThreads = 256;
constexpr int kMaBoundsThreads = 1024;
constexpr int kMaTrimWarps = kMaThreads / 32;      // trim frames per CTA of ma_trim_power_kernel
constexpr int kMaMaxMels = 128;                     // the mel bands Griffin-Lim can invert (kGlMaxMels)

enum : int { kMaTrim = 1, kMaPreemphasis = 2, kMaRescale = 4 };

struct MaRow {          // per-row results of ma_bounds_kernel
  int s, len, T, pad;   // trimmed signal wav[s, s + len), T frames
  float wav_peak;       // max |wav[s:e]| (0: no rescale)
  float pad2;
  double pre_peak;      // max |p[n]| over the trimmed signal (0: no rescale)
};

struct MaArgs {
  const float* wav;     // [B][Lmax]
  const int* len;       // [B]
  int Lmax, flags;
  // trim
  int trim_n, trim_hop;
  double trim_top_db;
  double* ms;           // [B][1 + Lmax / trim_hop] mean squares
  MaRow* rows;          // [B]
  int* frames;          // [B]
  int* bounds;          // optional [B][2]
  // stft / mel
  int hop, win_len, M, Tmax;
  double preemph, rescale_max_d;
  float rescale_max_f;
  const double* win;    // [win_len] periodic Hann, fp64
  const float2* tw;     // [kGlHalf / 2]
  const float2* tws;    // [kGlHalf / 2 + 1]
  const float* basis;   // [M][kGlBins] fp32 Slaney filterbank
  const int2* band;     // [M] non-zero bin range [lo, hi) of each band
  float mag_power;
  double min_level, min_db, ref_db, max_abs;
  float* mel;           // [B][Tmax][M]
  float* audio;         // optional [B][Tmax * hop]
};

__device__ __forceinline__ int ma_row_len(const MaArgs& A, int b) {
  const int L = A.len[b];
  return L < 0 ? 0 : (L > A.Lmax ? A.Lmax : L);
}

// Pre-emphasised sample n of the signal x (x[-1] = 0): lfilter([1, -k], [1], x) as scipy computes it in float64.
__device__ __forceinline__ double ma_preemph(const float* __restrict__ x, int n, double negk) {
  const double cur = (double)__ldg(x + n);
  return n > 0 ? __dadd_rn(cur, __dmul_rn(negk, (double)__ldg(x + n - 1))) : cur;
}

__device__ __forceinline__ double ma_signal(const MaArgs& A, const float* __restrict__ x, int n) {
  return (A.flags & kMaPreemphasis) ? ma_preemph(x, n, -A.preemph) : (double)__ldg(x + n);
}

// Mean square of every trim frame (librosa feature.rms(center=True, pad_mode='reflect') squared): frame f covers the
// samples f * hop - N/2 .. f * hop + N/2 - 1, reflected at both ends.  Lane i sums samples i, i + 32, ... in fp64, then a
// fixed butterfly adds the lanes.
__global__ void __launch_bounds__(kMaThreads) ma_trim_power_kernel(MaArgs A) {
  const int b = blockIdx.y;
  const int f = blockIdx.x * kMaTrimWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int L = ma_row_len(A, b);
  if (L < A.trim_n || f > L / A.trim_hop) return;
  const float* __restrict__ x = A.wav + (size_t)b * A.Lmax;
  const int n0 = f * A.trim_hop - A.trim_n / 2;
  double acc = 0.0;
  for (int j = lane; j < A.trim_n; j += 32) {
    int n = n0 + j;
    n = n < 0 ? -n : (n >= L ? 2 * (L - 1) - n : n);
    const double v = (double)__ldg(x + n);
    acc = fma(v, v, acc);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) A.ms[(size_t)b * (A.Lmax / A.trim_hop + 1) + f] = acc / A.trim_n;
}

__device__ __forceinline__ double ma_db10(double p) { return 10.0 * log10(fmax(1e-10, p)); }   // power_to_db, amin 1e-10

__global__ void __launch_bounds__(kMaBoundsThreads) ma_bounds_kernel(MaArgs A) {
  __shared__ double red_d[kMaBoundsThreads / 32];
  __shared__ int red_lo[kMaBoundsThreads / 32], red_hi[kMaBoundsThreads / 32];
  __shared__ float red_f[kMaBoundsThreads / 32];
  __shared__ int s_lo, s_hi;
  __shared__ double s_max;
  const int b = blockIdx.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int L = ma_row_len(A, b);
  int s = 0, e = L;
  if (A.flags & kMaTrim) {
    if (L < A.trim_n) {
      e = 0;
    } else {
      const int F = L / A.trim_hop + 1;
      const double* ms = A.ms + (size_t)b * (A.Lmax / A.trim_hop + 1);
      double mx = 0.0;
      for (int f = threadIdx.x; f < F; f += kMaBoundsThreads) mx = fmax(mx, ms[f]);
      for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      if (lane == 0) red_d[wid] = mx;
      __syncthreads();
      if (threadIdx.x == 0) {
        double m = 0.0;
        for (int w = 0; w < kMaBoundsThreads / 32; ++w) m = fmax(m, red_d[w]);
        s_max = m;
      }
      __syncthreads();
      const double ref = ma_db10(s_max);
      int lo = INT_MAX, hi = -1;
      if (s_max > 0.0) {           // an all-zero row has no non-silent frame (the reference would go on to divide by 0)
        for (int f = threadIdx.x; f < F; f += kMaBoundsThreads)
          if (ma_db10(ms[f]) - ref > -A.trim_top_db) { lo = min(lo, f); hi = max(hi, f); }
      }
      for (int o = 16; o > 0; o >>= 1) {
        lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
        hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
      }
      if (lane == 0) { red_lo[wid] = lo; red_hi[wid] = hi; }
      __syncthreads();
      if (threadIdx.x == 0) {
        int a = INT_MAX, c = -1;
        for (int w = 0; w < kMaBoundsThreads / 32; ++w) { a = min(a, red_lo[w]); c = max(c, red_hi[w]); }
        s_lo = a; s_hi = c;
      }
      __syncthreads();
      if (s_hi < 0) {
        e = 0;
      } else {
        s = s_lo * A.trim_hop;                              // frames_to_samples
        e = min(L, (s_hi + 1) * A.trim_hop);
      }
    }
  }
  const int n = e > s ? e - s : 0;
  if (n == 0) s = 0;
  // peaks of the trimmed wav and of its pre-emphasis (max is order-free: any reduction order gives the same value)
  const float* __restrict__ x = A.wav + (size_t)b * A.Lmax + s;
  float wp = 0.f;
  double pp = 0.0;
  if (A.flags & kMaRescale) {
    for (int i = threadIdx.x; i < n; i += kMaBoundsThreads) {
      wp = fmaxf(wp, fabsf(__ldg(x + i)));
      pp = fmax(pp, fabs(ma_signal(A, x, i)));
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    wp = fmaxf(wp, __shfl_xor_sync(0xffffffffu, wp, o));
    pp = fmax(pp, __shfl_xor_sync(0xffffffffu, pp, o));
  }
  __syncthreads();
  if (lane == 0) { red_f[wid] = wp; red_d[wid] = pp; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 0; w < kMaBoundsThreads / 32; ++w) { wp = fmaxf(wp, red_f[w]); pp = fmax(pp, red_d[w]); }
    MaRow r{};
    r.s = s;
    r.len = n;
    r.T = n > 0 ? 1 + n / A.hop : 0;
    r.wav_peak = wp;
    r.pre_peak = pp;
    A.rows[b] = r;
    A.frames[b] = r.T;
    if (A.bounds) { A.bounds[2 * b] = s; A.bounds[2 * b + 1] = s + n; }
  }
}

// One CTA per (row, frame t): frame t of librosa's stft (center=True, constant padding) covers samples t * hop - n_fft/2 ..
// t * hop + n_fft/2 - 1 of the trimmed signal; only the win_len samples under the centred window are non-zero.
__global__ void __launch_bounds__(kMaThreads) ma_frame_kernel(MaArgs A) {
  __shared__ __align__(16) float2 buf[2][kGlHalf];
  const int t = blockIdx.x, b = blockIdx.y;
  const MaRow r = A.rows[b];
  float* __restrict__ out = A.mel + ((size_t)b * A.Tmax + t) * A.M;
  if (t >= r.T) {
    for (int m = threadIdx.x; m < A.M; m += kMaThreads) out[m] = 0.f;
    return;
  }
  const float* __restrict__ x = A.wav + (size_t)b * A.Lmax + r.s;
  const bool rescale = (A.flags & kMaRescale) && r.pre_peak > 0.0;
  const int lpad = (kGlN - A.win_len) / 2;
  float* xs = reinterpret_cast<float*>(buf[0]);
  for (int i = threadIdx.x; i < kGlN; i += kMaThreads) {
    float v = 0.f;
    const int j = i - lpad, n = t * A.hop - kGlN / 2 + i;
    if (j >= 0 && j < A.win_len && n >= 0 && n < r.len) {
      double p = ma_signal(A, x, n);
      if (rescale) p = __dmul_rn(__ddiv_rn(p, r.pre_peak), A.rescale_max_d);
      v = (float)(p * __ldg(A.win + j));
    }
    xs[i] = v;
  }
  __syncthreads();
  gl_fft1024<false>(buf[0], buf[1], A.tw);                         // 10 stages: result back in buf[0]
  float* pw = reinterpret_cast<float*>(buf[1]);                    // |X[k]|^p, k = 0..1024
  for (int k = threadIdx.x; k <= kGlHalf / 2; k += kMaThreads) {
    float2 X0, X1;
    gl_forward_split(buf[0][k], buf[0][(kGlHalf - k) & (kGlHalf - 1)], __ldg(A.tws + k), &X0, &X1);
    const float r0 = hypotf(X0.x, X0.y), r1 = hypotf(X1.x, X1.y);
    pw[k] = A.mag_power == 2.f ? r0 * r0 : powf(r0, A.mag_power);
    pw[kGlHalf - k] = A.mag_power == 2.f ? r1 * r1 : powf(r1, A.mag_power);
  }
  __syncthreads();
  for (int m = threadIdx.x; m < A.M; m += kMaThreads) {
    const int2 rg = __ldg(A.band + m);
    const float* __restrict__ row = A.basis + (size_t)m * kGlBins;
    float acc = 0.f;
    for (int k = rg.x; k < rg.y; ++k) acc = fmaf(__ldg(row + k), pw[k], acc);      // ascending bins
    const double db = 20.0 * log10(fmax(A.min_level, (double)acc)) - A.ref_db;       // _amp_to_db - ref_level_db
    const double v = (2.0 * A.max_abs) * ((db - A.min_db) / (-A.min_db)) - A.max_abs; // _normalize, symmetric
    out[m] = (float)fmin(fmax(v, -A.max_abs), A.max_abs);
  }
}

// out[n] = wav[s + n] / max|wav[s:e]| * rescaling_max (fp32, as numpy computes it) for n < e - s, zero up to Tmax * hop.
__global__ void __launch_bounds__(kMaThreads) ma_audio_kernel(MaArgs A) {
  const int b = blockIdx.y;
  const MaRow r = A.rows[b];
  const size_t Lout = (size_t)A.Tmax * A.hop;
  const float* __restrict__ x = A.wav + (size_t)b * A.Lmax + r.s;
  float* __restrict__ y = A.audio + (size_t)b * Lout;
  const bool rescale = (A.flags & kMaRescale) && r.wav_peak > 0.f;
  for (size_t n = (size_t)blockIdx.x * kMaThreads + threadIdx.x; n < Lout; n += (size_t)gridDim.x * kMaThreads) {
    float v = 0.f;
    if (n < (size_t)r.len) {
      v = __ldg(x + n);
      if (rescale) v = __fmul_rn(__fdiv_rn(v, r.wav_peak), A.rescale_max_f);
    }
    y[n] = v;
  }
}

}  // namespace b200tts
