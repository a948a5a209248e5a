// The 2048-point real FFT shared by Griffin-Lim (griffin_lim.cuh) and mel analysis (mel_analysis.cuh): a 1024-point complex
// radix-2 Stockham FFT in shared memory (even samples in .x, odd in .y) plus the real split step.  Twiddles are computed in
// fp64 on the host (fft2048_twiddles) and stored as fp32.  A CTA that runs gl_fft1024 has kGlThreads threads.
#pragma once
#include <cmath>

#include "common.cuh"

namespace b200tts {

constexpr int kGlN = 2048;           // n_fft (the only size the FFT below implements)
constexpr int kGlHalf = kGlN / 2;    // complex FFT length
constexpr int kGlBins = kGlHalf + 1; // rfft bins
constexpr int kGlThreads = 256;

__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

// Radix-2 Stockham, 10 stages, src -> (ping-pong) -> src.  Forward uses tw, inverse its conjugate; unnormalised.
template <bool kInverse>
__device__ __forceinline__ void gl_fft1024(float2* a, float2* b, const float2* __restrict__ tw) {
  float2* src = a;
  float2* dst = b;
#pragma unroll 1
  for (int Ns = 1; Ns < kGlHalf; Ns <<= 1) {
    const int shift = kGlHalf / 2 / Ns;
#pragma unroll
    for (int r = 0; r < kGlHalf / 2 / kGlThreads; ++r) {
      const int j = threadIdx.x + r * kGlThreads;
      const int k = j & (Ns - 1);
      float2 w = __ldg(tw + k * shift);
      if (kInverse) w.y = -w.y;
      const float2 x0 = src[j], x1 = cmul(src[j + kGlHalf / 2], w);
      const int o = ((j - k) << 1) + k;
      dst[o] = make_float2(x0.x + x1.x, x0.y + x1.y);
      dst[o + Ns] = make_float2(x0.x - x1.x, x0.y - x1.y);
    }
    __syncthreads();
    float2* t = src; src = dst; dst = t;
  }
}

// Real split step of the forward 2048-point rfft: Z = FFT1024 of the even/odd-packed signal, za = Z[k], zb = Z[(1024-k) mod
// 1024], w = e^{-2 pi i k / 2048}  ->  rfft bins *X0 = X[k] and *X1 = X[1024-k], 0 <= k <= 512.
__device__ __forceinline__ void gl_forward_split(float2 za, float2 zb, float2 w, float2* X0, float2* X1) {
  const float2 fe = make_float2(0.5f * (za.x + zb.x), 0.5f * (za.y - zb.y));   // (Z[k] + conj Z[N-k]) / 2
  const float2 fo = make_float2(0.5f * (za.y + zb.y), -0.5f * (za.x - zb.x));  // (Z[k] - conj Z[N-k]) / 2i
  const float2 wf = cmul(w, fo);
  *X0 = make_float2(fe.x + wf.x, fe.y + wf.y);          // X[k]
  *X1 = make_float2(fe.x - wf.x, -(fe.y - wf.y));       // X[N-k] = conj(fe - w fo)
}

// The twiddle tables the FFT reads, as float pairs: tw[m] = e^{-2 pi i m / 1024} for m < 512 (gl_fft1024) and
// tws[k] = e^{-2 pi i k / 2048} for k <= 512 (the real split steps).
inline void fft2048_twiddles(float* tw, float* tws) {
  const double pi = 3.14159265358979323846;
  for (int m = 0; m < kGlHalf / 2; ++m) {
    tw[2 * m] = (float)std::cos(-2.0 * pi * m / kGlHalf);
    tw[2 * m + 1] = (float)std::sin(-2.0 * pi * m / kGlHalf);
  }
  for (int k = 0; k <= kGlHalf / 2; ++k) {
    tws[2 * k] = (float)std::cos(-2.0 * pi * k / kGlN);
    tws[2 * k + 1] = (float)std::sin(-2.0 * pi * k / kGlN);
  }
}

}  // namespace b200tts
