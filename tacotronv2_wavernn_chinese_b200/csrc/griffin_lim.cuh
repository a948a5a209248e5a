// Griffin-Lim mel inversion (tacotron/datasets/audio.py:122-137 inv_mel_spectrogram, :176-186 _griffin_lim, :203-210 _stft /
// _istft with librosa 0.7.2, :256-260 _mel_to_linear, :297-309 _denormalize, :52-55
// inv_preemphasis).  Three kernels:
//   gl_magnitude_kernel  mel -> S = max(1e-10, pinv(M) . db_to_amp(denormalize(mel) + ref)^(1/mag_power))^power, once per call
//   gl_frame_kernel      one CTA per (row, frame): gather the frame's window support from the previous iteration's windowed
//                        frames (overlap-add / window sum-square, zero outside the row's signal), window, rfft, unit phasor,
//                        times S, irfft, window -> the frame's windowed time signal.  kInit: the phasor comes from u instead.
//   gl_finish_kernel     one CTA per row: overlap-add, envelope, inverse pre-emphasis (chunked scan with carries), zero tail
// The 2048-point real FFT is fft2048.cuh's; the inverse mirrors it.  No atomics: every value a row produces depends only on
// that row's inputs.
#pragma once
#include "common.cuh"
#include "fft2048.cuh"

namespace b200tts {

constexpr int kGlMagFrames = 16;     // frames per CTA of the magnitude GEMV (the pinv basis is read once per 16 frames)
constexpr int kGlMaxMels = 128;
constexpr int kGlFinishThreads = 1024;

struct GlArgs {
  const float* S;           // [B][Tmax][kGlBins]
  const float* win;         // [win] periodic Hann
  const float* win2;        // [win] its square
  const float2* tw;         // [kGlHalf/2]  e^{-2 pi i m / 1024}
  const float2* tws;        // [kGlHalf/2 + 1] e^{-2 pi i k / 2048} (real split step)
  const int* frames;        // optional [B]
  int Tmax, hop, win_len;
  const float* prev;        // [B][Tmax][win] windowed frames of the previous iteration (not read by kInit)
  float* next;              // [B][Tmax][win]
  float* u_out;             // optional [B][Tmax][kGlBins]: phase (u form) this pass used
  // kInit only
  int ext;                  // 1: read u from u_in; 0: Philox
  const float* u_in;        // [B][Tmax][kGlBins]
  unsigned long long seed, utt0;
};

__device__ __forceinline__ int gl_row_frames(const int* frames, int b, int Tmax) {
  if (!frames) return Tmax;
  int T = frames[b];
  return T < 0 ? 0 : (T > Tmax ? Tmax : T);
}

// Uniform in [0,1) for (utterance, frame, bin); counter word 1 carries a tag bit so the stream is disjoint from the other
// streams keyed with the same seed (the map is in common.cuh).  Shared by the frame kernel and b200tts_gl_philox_uniform
// (bit-identical dumps).
__device__ __forceinline__ float gl_philox_uniform(uint64_t seed, uint64_t utt, uint32_t frame, uint32_t bin) {
  uint32_t c[4] = {frame, 0x80000000u | (bin >> 2), (uint32_t)utt, (uint32_t)(utt >> 32)};
  philox4x32_10(c, seed);
  const uint32_t q = bin & 3, x = q == 0 ? c[0] : q == 1 ? c[1] : q == 2 ? c[2] : c[3];     // no dynamic index: stays in registers
  return (float)(x >> 8) * (1.0f / 16777216.0f);
}

__device__ __forceinline__ float gl_phase_u(float x, float y) {     // np.angle / 2 pi mod 1 (angle(0) = 0)
  float u = atan2f(y, x) * 0.15915494309189535f;
  if (u < 0.f) u += 1.f;
  return u >= 1.f ? 0.f : u;
}

__device__ __forceinline__ float2 conjf2(float2 a) { return make_float2(a.x, -a.y); }

// Spectrum pair (k, 1024-k) -> inverse-split inputs Z'[k], Z'[1024-k] (irfft of Y = (Y[0..1024]) as a 1024-point complex IFFT).
// Y0/Y1 are Y[k], Y[1024-k]; for k = 0 they are Y[0], Y[1024] (imaginary parts already dropped, as irfft does).
__device__ __forceinline__ void gl_inverse_split(int k, float2 Y0, float2 Y1, float2 w, float2* out) {
  const float2 e = make_float2(0.5f * (Y0.x + Y1.x), 0.5f * (Y0.y - Y1.y));     // (Y[k] + conj Y[N-k]) / 2
  const float2 d = make_float2(0.5f * (Y0.x - Y1.x), 0.5f * (Y0.y + Y1.y));     // (Y[k] - conj Y[N-k]) / 2
  const float2 o = cmul(d, conjf2(w));                                          // * e^{+2 pi i k / 2048}
  out[k] = make_float2(e.x - o.y, e.y + o.x);                                    // e + i o
  if (k > 0 && k < kGlHalf / 2) out[kGlHalf - k] = make_float2(e.x + o.y, -e.y + o.x);   // conj(e) + i conj(o)
}

// Overlap-add of sample n (0 <= n < L) from the windowed frames of one row, divided by the window sum-square (fixed order,
// ascending frame).  off = lpad - n_fft/2 maps sample n to window index n - hop*t - off of frame t.
__device__ __forceinline__ float gl_ola(const float* __restrict__ fr, const float* __restrict__ win2, int n, int T, int hop,
                                        int win_len, int off) {
  const int hi_num = n - off;                       // >= 0
  const int lo_num = hi_num - win_len;
  int tlo = lo_num >= 0 ? lo_num / hop + 1 : 0;
  int thi = hi_num / hop;
  if (thi > T - 1) thi = T - 1;
  float acc = 0.f, env = 0.f;
  for (int t = tlo; t <= thi; ++t) {
    const int jj = hi_num - hop * t;
    acc += __ldg(fr + (size_t)t * win_len + jj);
    env += __ldg(win2 + jj);
  }
  return env > 1.17549435e-38f ? acc / env : acc;
}

template <bool kInit>
__global__ void __launch_bounds__(kGlThreads) gl_frame_kernel(GlArgs A) {
  __shared__ __align__(16) float2 buf[2][kGlHalf];
  const int t = blockIdx.x, b = blockIdx.y;
  const int T = gl_row_frames(A.frames, b, A.Tmax);
  if (t >= T || T < 2) return;
  const int lpad = (kGlN - A.win_len) / 2;
  const size_t fbase = ((size_t)b * A.Tmax + t);
  const float* __restrict__ S = A.S + fbase * kGlBins;
  float* __restrict__ u_out = A.u_out ? A.u_out + fbase * kGlBins : nullptr;

  if (kInit) {
    // Y = S e^{2 pi i u} straight into the inverse-split buffer
    const uint64_t utt = A.utt0 + (uint64_t)b;
    const float* __restrict__ u_in = A.ext ? A.u_in + fbase * kGlBins : nullptr;
    for (int k = threadIdx.x; k <= kGlHalf / 2; k += kGlThreads) {
      const int k2 = kGlHalf - k;
      float ua = u_in ? __ldg(u_in + k) : gl_philox_uniform(A.seed, utt, (uint32_t)t, (uint32_t)k);
      float ub = u_in ? __ldg(u_in + k2) : gl_philox_uniform(A.seed, utt, (uint32_t)t, (uint32_t)k2);
      if (u_out) { u_out[k] = ua; u_out[k2] = ub; }
      float sa, ca, sb, cb;
      sincospif(2.f * ua, &sa, &ca);
      sincospif(2.f * ub, &sb, &cb);
      float2 Y0 = make_float2(__ldg(S + k) * ca, __ldg(S + k) * sa);
      float2 Y1 = make_float2(__ldg(S + k2) * cb, __ldg(S + k2) * sb);
      if (k == 0) { Y0.y = 0.f; Y1.y = 0.f; }
      gl_inverse_split(k, Y0, Y1, __ldg(A.tws + k), buf[1]);
    }
    __syncthreads();
  } else {
    // gather the frame: x[lpad + j] = win[j] * y[hop*t - n_fft/2 + lpad + j], zero elsewhere
    float* xs = reinterpret_cast<float*>(buf[0]);
    for (int i = threadIdx.x; i < kGlN; i += kGlThreads) xs[i] = 0.f;
    __syncthreads();
    const int L = A.hop * (T - 1);
    const int off = lpad - kGlN / 2;
    const float* __restrict__ fr = A.prev + (size_t)b * A.Tmax * A.win_len;
    for (int j = threadIdx.x; j < A.win_len; j += kGlThreads) {
      const int n = A.hop * t + off + j;
      if (n >= 0 && n < L) xs[lpad + j] = __ldg(A.win + j) * gl_ola(fr, A.win2, n, T, A.hop, A.win_len, off);
    }
    __syncthreads();
    gl_fft1024<false>(buf[0], buf[1], A.tw);                     // 10 stages: result back in buf[0]
    // real split -> X[k], X[N-k]; unit phasor times S; inverse split into buf[1]
    for (int k = threadIdx.x; k <= kGlHalf / 2; k += kGlThreads) {
      const int k2 = kGlHalf - k;
      const float2 w = __ldg(A.tws + k);
      float2 X0, X1;
      gl_forward_split(buf[0][k], buf[0][k2 & (kGlHalf - 1)], w, &X0, &X1);
      float2 Y[2];
      const float2 X[2] = {X0, X1};
      const int kk[2] = {k, k2};
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const float r = hypotf(X[q].x, X[q].y);
        const float s = __ldg(S + kk[q]);
        Y[q] = r > 0.f ? make_float2(s * (X[q].x / r), s * (X[q].y / r)) : make_float2(s, 0.f);
        if (u_out) u_out[kk[q]] = gl_phase_u(X[q].x, X[q].y);
      }
      if (k == 0) { Y[0].y = 0.f; Y[1].y = 0.f; }
      gl_inverse_split(k, Y[0], Y[1], w, buf[1]);
    }
    __syncthreads();
  }
  gl_fft1024<true>(buf[1], buf[0], A.tw);                         // result back in buf[1]
  const float* ys = reinterpret_cast<const float*>(buf[1]);
  float* __restrict__ out = A.next + fbase * A.win_len;
  for (int j = threadIdx.x; j < A.win_len; j += kGlThreads) out[j] = __ldg(A.win + j) * (ys[lpad + j] * (1.f / kGlHalf));
}

// mel [B][Tmax][M] -> S [B][Tmax][kGlBins]; kGlMagFrames frames per CTA, one bin per thread and pass.
struct GlMagArgs {
  const float* mel;
  const float* pinv;        // [kGlBins][M]
  const int* frames;
  float* S;
  int Tmax, M;
  float max_abs, min_db, ref_db, inv_mag_power, power;
};

__global__ void __launch_bounds__(kGlThreads) gl_magnitude_kernel(GlMagArgs A) {
  __shared__ float a[kGlMagFrames][kGlMaxMels];
  const int b = blockIdx.y, t0 = blockIdx.x * kGlMagFrames;
  const int T = gl_row_frames(A.frames, b, A.Tmax);
  if (t0 >= T) return;
  const int nf = min(kGlMagFrames, T - t0);
  for (int i = threadIdx.x; i < kGlMagFrames * A.M; i += kGlThreads) {
    const int f = i / A.M, m = i % A.M;
    float v = 0.f;
    if (f < nf) {
      double x = fmin(fmax((double)A.mel[((size_t)b * A.Tmax + t0 + f) * A.M + m], -(double)A.max_abs), (double)A.max_abs);
      double D = (x + A.max_abs) * (-(double)A.min_db / (2.0 * A.max_abs)) + A.min_db;          // _denormalize :297-309
      v = (float)pow(pow(10.0, (D + A.ref_db) * 0.05), (double)A.inv_mag_power);               // _db_to_amp ** (1/mag_power)
    }
    a[f][m] = v;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < kGlBins; k += kGlThreads) {
    float acc[kGlMagFrames];
#pragma unroll
    for (int f = 0; f < kGlMagFrames; ++f) acc[f] = 0.f;
    const float* __restrict__ row = A.pinv + (size_t)k * A.M;
    for (int m = 0; m < A.M; ++m) {
      const float p = __ldg(row + m);
#pragma unroll
      for (int f = 0; f < kGlMagFrames; ++f) acc[f] = fmaf(p, a[f][m], acc[f]);
    }
#pragma unroll
    for (int f = 0; f < kGlMagFrames; ++f)
      if (f < nf) A.S[((size_t)b * A.Tmax + t0 + f) * kGlBins + k] = powf(fmaxf(1e-10f, acc[f]), A.power);   // :260, ** power :137
  }
}

// One CTA per row: y[n] = OLA / envelope for n < L_row, then lfilter([1], [1, -k], y) as a chunked scan: every thread runs
// the recurrence over its chunk from a zero state (fp64), the chunk carries are chained serially, and each sample then gets
// carry * k^(i+1).  The chunks depend on L_row only, so a row of a ragged batch is bit-identical to a stand-alone run.
// Samples L_row <= n < L_max are zero.
__global__ void __launch_bounds__(kGlFinishThreads) gl_finish_kernel(const float* __restrict__ fr_all, const float* __restrict__ win2,
                                                                     const int* frames, int Tmax, int hop, int win_len, float preemph,
                                                                     float* __restrict__ wave) {
  __shared__ double last[kGlFinishThreads], carry[kGlFinishThreads];
  const int b = blockIdx.x;
  const int T = gl_row_frames(frames, b, Tmax);
  const int Lmax = hop * (Tmax - 1);
  const int L = T >= 2 ? hop * (T - 1) : 0;
  float* w = wave + (size_t)b * Lmax;
  for (int n = L + threadIdx.x; n < Lmax; n += kGlFinishThreads) w[n] = 0.f;
  if (L == 0) return;
  const int chunk = (L + kGlFinishThreads - 1) / kGlFinishThreads;
  const int n0 = min(L, threadIdx.x * chunk), n1 = min(L, n0 + chunk);
  const int off = (kGlN - win_len) / 2 - kGlN / 2;
  const float* fr = fr_all + (size_t)b * Tmax * win_len;
  const double k = preemph;
  double s = 0.0;
  for (int n = n0; n < n1; ++n) {
    s = fma(k, s, (double)gl_ola(fr, win2, n, T, hop, win_len, off));
    w[n] = (float)s;
  }
  last[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double c = 0.0;
    for (int i = 0; i < kGlFinishThreads; ++i) {
      carry[i] = c;
      const int a0 = min(L, i * chunk), a1 = min(L, a0 + chunk);
      c = last[i] + pow(k, (double)(a1 - a0)) * c;
    }
  }
  __syncthreads();
  const double c = carry[threadIdx.x];
  if (c != 0.0) {
    // second pass recomputes the local scan so the sum is formed in fp64 before the single rounding to fp32
    double p = k, s2 = 0.0;
    for (int n = n0; n < n1; ++n) {
      s2 = fma(k, s2, (double)gl_ola(fr, win2, n, T, hop, win_len, off));
      w[n] = (float)(s2 + p * c);
      p *= k;
    }
  }
}

__global__ void gl_philox_dump_kernel(unsigned long long seed, unsigned long long utt0, int B, int T, int n_bins, float* __restrict__ u) {
  const size_t total = (size_t)B * T * n_bins;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(e % n_bins);
    const size_t bt = e / n_bins;
    const int t = (int)(bt % T), b = (int)(bt / T);
    u[e] = gl_philox_uniform(seed, utt0 + (unsigned long long)b, (uint32_t)t, (uint32_t)k);
  }
}

}  // namespace b200tts
