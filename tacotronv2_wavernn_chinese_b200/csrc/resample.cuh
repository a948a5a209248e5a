// Band-limited resampling: librosa 0.7.2 core.resample(y, sr_orig, sr_new, res_type='kaiser_best'), which is resampy 0.2.2's
// resample / resample_f (interpolation from a tabulated half window, linear inside the table) followed by librosa's
// util.fix_length zero padding to ceil(L * ratio).  One kernel:
//   rs_kernel  one thread per (row, output sample t); a CTA stages the input samples its 256 outputs read as fp64 in shared
//              memory, then each thread sums its left wing and its right wing in resampy's order
// resampy's arithmetic is restated operation for operation, with explicit roundings so that nvcc contracts nothing into DFMA
// (resampy, compiled by numba, never fuses):
//   n = int(tau), frac = scale * (tau - n), offset = int(frac * num_table), eta = frac * num_table - offset
//   weight = table[o] + eta * delta[o]                           (fp64 multiply, then fp64 add)
//   y = float(double(y) + weight * double(x))                    (fp64 product and sum, every partial sum rounded to fp32)
// tau_t, the time register, is resampy's sequential fp64 sum tau_{t+1} = tau_t + 1 / ratio.  It depends on the rate pair only,
// so the host computes it once per context and the kernel reads it (t * (1 / ratio) is not the same number).  The table is
// {table[o], delta[o] = table[o + 1] - table[o]} interleaved, one 16-byte load per term, read through the L1 (read-only)
// path.  No atomics and no cross-row arithmetic: every row is computed exactly as a stand-alone run of that row.
#pragma once

#include "common.cuh"

namespace b200tts {

constexpr int kRsThreads = 256;

struct RsArgs {
  const float* x;       // [B][Lmax]
  const int* len;       // [B]
  int Lmax, Ymax;       // input / output row strides; Ymax = ceil(Lmax * ratio)
  const double2* tab;   // [nwin] {table, delta}, the table already scaled by ratio when ratio < 1
  const double* reg;    // [>= int(Lmax * ratio)] time register
  int nwin, index_step, num_table, wing;   // wing = nwin / index_step + 1 bounds the taps of either wing
  int xs_cap;           // doubles of the shared input window
  double ratio, scale;
  float* y;             // [B][Ymax]
  int* out_len;         // [B] ceil(len * ratio)
};

// One wing: sum_{i < imax} (tab[off + i*step].x + eta * tab[...].y) * x[n -/+ ...], accumulated in resampy's order.
template <int kDir>
__device__ __forceinline__ float rs_wing(const RsArgs& A, const double* __restrict__ xs, int base, int i0, int imax,
                                         int offset, double eta, float acc) {
  const double2* __restrict__ tab = A.tab + offset;
  for (int i = i0; i < imax; ++i) {
    const double2 te = __ldg(tab + i * A.index_step);
    const double w = __dadd_rn(te.x, __dmul_rn(eta, te.y));
    acc = __double2float_rn(__dadd_rn((double)acc, __dmul_rn(w, xs[base + kDir * i])));
  }
  return acc;
}

__global__ void __launch_bounds__(kRsThreads) rs_kernel(RsArgs A) {
  extern __shared__ double rs_xs[];
  const int b = blockIdx.y;
  int L = A.len[b];
  L = L < 0 ? 0 : (L > A.Lmax ? A.Lmax : L);
  const double Lr = __dmul_rn((double)L, A.ratio);
  const int n_out = (int)Lr;                                     // resampy's output length int(L * ratio)
  const int t0 = blockIdx.x * kRsThreads, t = t0 + threadIdx.x;
  if (blockIdx.x == 0 && threadIdx.x == 0) A.out_len[b] = (int)ceil(Lr);   // librosa's fix_length target
  float* __restrict__ y = A.y + (size_t)b * A.Ymax;
  if (t0 >= n_out) {                                             // the whole CTA is padding
    if (t < A.Ymax) y[t] = 0.f;
    return;
  }
  // input samples [lo, hi) that the CTA's outputs read (tau is non-decreasing in t)
  const int t_last = min(t0 + kRsThreads, n_out) - 1;
  const int lo = max(0, (int)A.reg[t0] - A.wing + 1);
  const int hi = min(L, (int)A.reg[t_last] + A.wing + 1);
  const float* __restrict__ x = A.x + (size_t)b * A.Lmax;
  for (int j = threadIdx.x; j < hi - lo; j += kRsThreads) rs_xs[j] = (double)__ldg(x + lo + j);
  __syncthreads();
  if (t >= A.Ymax) return;
  float acc = 0.f;
  if (t < n_out) {
    const double tau = A.reg[t];
    const int n = (int)tau;
    const double num_table = (double)A.num_table;
    // left wing: x[n - i], i < min(n + 1, (nwin - offset) / index_step)
    double frac = __dmul_rn(A.scale, __dsub_rn(tau, (double)n));
    double index_frac = __dmul_rn(frac, num_table);
    int offset = (int)index_frac;
    double eta = __dsub_rn(index_frac, (double)offset);
    const int i_max = min(n + 1, (A.nwin - offset) / A.index_step);
    // resampy never reads past the signal (tau_t < L for t < int(L * ratio)); samples from L on are skipped, not read
    acc = rs_wing<-1>(A, rs_xs, n - lo, max(0, n - (L - 1)), i_max, offset, eta, acc);
    // right wing: x[n + 1 + k], k < min(L - n - 1, (nwin - offset') / index_step), frac' = scale - frac
    frac = __dsub_rn(A.scale, frac);
    index_frac = __dmul_rn(frac, num_table);
    offset = (int)index_frac;
    eta = __dsub_rn(index_frac, (double)offset);
    const int k_max = min(L - n - 1, (A.nwin - offset) / A.index_step);
    acc = rs_wing<1>(A, rs_xs, n + 1 - lo, 0, k_max, offset, eta, acc);
  }
  y[t] = acc;
}

}  // namespace b200tts
