// libb200tts.so -- resampling (resample.cuh): b200tts_resample_*.
#include <algorithm>
#include <cmath>

#include "api.h"
#include "resample.cuh"

using namespace b200tts;

struct b200tts_resampler {
  int device = 0;
  int sr_orig = 0, sr_new = 0, nwin = 0, num_table = 0, index_step = 0, wing = 0, xs_cap = 0;
  double ratio = 0.0, scale = 0.0, time_increment = 0.0;
  DeviceBuf tab;                // [nwin] double2 {table, delta}
  DeviceBuf reg;                // [n_reg] time register
  int64_t n_reg = 0;
  std::vector<double> h_reg;
  int64_t launches = 0;
};

extern "C" int b200tts_resample_create(b200tts_resampler** out, int device, int sr_orig, int sr_new,
                                       const double* h_half_window, int nwin, int num_table) {
  API_BEGIN
  REQUIRE(out && h_half_window, B200TTS_EINVAL, "null argument");
  *out = nullptr;
  REQUIRE(sr_orig > 0 && sr_new > 0, B200TTS_EINVAL, "sample rates must be positive");
  REQUIRE(sr_orig != sr_new, B200TTS_EINVAL, "sr_orig equals sr_new: there is nothing to resample (librosa returns the input)");
  REQUIRE(nwin >= 2 && num_table >= 1, B200TTS_EINVAL, "nwin must be >= 2 and num_table >= 1");
  const double ratio = (double)sr_new / sr_orig;                      // resampy: float(sr_new) / sr_orig
  const double scale = std::min(1.0, ratio);
  const int index_step = (int)(scale * num_table);
  REQUIRE(index_step >= 1, B200TTS_EINVAL, "sr_new / sr_orig too small: index_step = int(scale * num_table) is 0");
  const double inc = 1.0 / ratio;
  const int wing = nwin / index_step + 1;
  const double cap = std::ceil((kRsThreads - 1) * inc) + 2.0 * wing + 4.0;
  REQUIRE(cap * sizeof(double) <= 200.0 * 1024, B200TTS_EINVAL,
          "sr_new / sr_orig too small: a CTA's input window exceeds 200 KB of shared memory");
  check_device(device);
  DeviceGuard dg(device);
  std::unique_ptr<b200tts_resampler> ctx(new b200tts_resampler());
  ctx->device = device;
  ctx->sr_orig = sr_orig; ctx->sr_new = sr_new;
  ctx->nwin = nwin; ctx->num_table = num_table; ctx->index_step = index_step; ctx->wing = wing;
  ctx->xs_cap = (int)cap;
  ctx->ratio = ratio; ctx->scale = scale; ctx->time_increment = inc;
  std::vector<double> h(2 * (size_t)nwin);
  for (int o = 0; o < nwin; ++o) h[2 * o] = ratio < 1.0 ? h_half_window[o] * ratio : h_half_window[o];   // interp_win *= ratio
  for (int o = 0; o < nwin; ++o) h[2 * o + 1] = o + 1 < nwin ? h[2 * o + 2] - h[2 * o] : 0.0;             // delta[:-1] = diff
  ctx->tab.ensure(h.size() * sizeof(double));
  B200_CUDA(cudaMemcpy(ctx->tab.p, h.data(), h.size() * sizeof(double), cudaMemcpyHostToDevice));
  if (ctx->xs_cap * sizeof(double) > 48 * 1024)
    B200_CUDA(cudaFuncSetAttribute(rs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(ctx->xs_cap * sizeof(double))));
  *out = ctx.release();
  API_END
}

extern "C" void b200tts_resample_destroy(b200tts_resampler* ctx) {
  if (!ctx) return;
  DeviceGuard dg(ctx->device, true);
  delete ctx;
}

extern "C" int64_t b200tts_resample_launch_count(const b200tts_resampler* ctx) { return ctx ? ctx->launches : -1; }

extern "C" int b200tts_resample(b200tts_resampler* ctx, const float* d_x, const int32_t* d_len, int B, int L_max, float* d_y,
                                int32_t* d_out_len, void* stream) {
  API_BEGIN
  REQUIRE(ctx && d_x && d_len && d_y && d_out_len, B200TTS_EINVAL, "null argument");
  REQUIRE(B >= 1 && B <= 65535, B200TTS_EINVAL, "B must be 1..65535");
  REQUIRE(L_max >= 1 && L_max < (1 << 30), B200TTS_EINVAL, "L_max must be 1..2^30-1");
  const double Lr = (double)L_max * ctx->ratio;                                               // first read of *ctx
  const int64_t n_need = (int64_t)Lr, Y_max = (int64_t)std::ceil(Lr);
  REQUIRE(n_need >= 1, B200TTS_EINVAL, "L_max is too short to resample: int(L_max * sr_new / sr_orig) < 1");
  REQUIRE(Y_max < (1 << 30), B200TTS_EINVAL, "output rows would exceed 2^30-1 samples");
  DeviceGuard dg(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (n_need > ctx->n_reg) {     // extend the time register: resampy's sequential sum, continued from where it stopped
    const int64_t n0 = ctx->n_reg;
    ctx->h_reg.resize((size_t)n_need);
    double tr = n0 > 0 ? ctx->h_reg[n0 - 1] + ctx->time_increment : 0.0;
    for (int64_t t = n0; t < n_need; ++t) {
      ctx->h_reg[t] = tr;
      tr += ctx->time_increment;
    }
    ctx->reg.ensure((size_t)n_need * sizeof(double));     // cudaFree waits for earlier launches that read the old buffer
    B200_CUDA(cudaMemcpyAsync(ctx->reg.p, ctx->h_reg.data(), (size_t)n_need * sizeof(double), cudaMemcpyHostToDevice, st));
    B200_CUDA(cudaStreamSynchronize(st));                 // h_reg is only touched again after the copy has finished
    ctx->n_reg = n_need;
  }
  RsArgs a{};
  a.x = d_x; a.len = d_len; a.Lmax = L_max; a.Ymax = (int)Y_max;
  a.tab = ctx->tab.as<double2>(); a.reg = ctx->reg.as<double>();
  a.nwin = ctx->nwin; a.index_step = ctx->index_step; a.num_table = ctx->num_table; a.wing = ctx->wing;
  a.xs_cap = ctx->xs_cap; a.ratio = ctx->ratio; a.scale = ctx->scale;
  a.y = d_y; a.out_len = d_out_len;
  const unsigned gx = (unsigned)((Y_max + kRsThreads - 1) / kRsThreads);
  rs_kernel<<<dim3(gx, B), kRsThreads, (size_t)ctx->xs_cap * sizeof(double), st>>>(a);
  B200_CUDA(cudaGetLastError());
  ctx->launches++;
  API_END
}
