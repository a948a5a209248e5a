// libb200tts.so -- mel analysis (mel_analysis.cuh): b200tts_mel_*.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>

#include "api.h"
#include "mel_analysis.cuh"

using namespace b200tts;

struct b200tts_mel {
  int device = 0;
  b200tts_mel_cfg cfg{};
  double preemph = 0.0, rescale_max = 0.0, min_level = 0.0;
  DeviceBuf consts;             // basis [M][kGlBins] | tw [512] float2 | tws [513] float2 | band [M] int2 | win [W] double
  const float* basis = nullptr;
  const float2 *tw = nullptr, *tws = nullptr;
  const int2* band = nullptr;
  const double* win = nullptr;
  DeviceBuf ms, rows;
  int64_t launches = 0;
};

namespace {
// The shortest decimal that rounds to f, as a double: a float parameter means the Python value it was converted from.
double shortest_decimal(float f) {
  char buf[32];
  for (int digits = 1; digits <= 9; ++digits) {
    std::snprintf(buf, sizeof buf, "%.*g", digits, (double)f);
    const double d = std::strtod(buf, nullptr);
    if ((float)d == f) return d;
  }
  return (double)f;
}
}  // namespace

extern "C" int b200tts_mel_create(b200tts_mel** out, int device, const b200tts_mel_cfg* cfg, const float* h_mel_basis) {
  API_BEGIN
  REQUIRE(out && cfg && h_mel_basis, B200TTS_EINVAL, "null argument");
  *out = nullptr;
  const b200tts_mel_cfg c = *cfg;
  REQUIRE(c.n_fft == kGlN, B200TTS_EINVAL, "n_fft must be 2048 (the only FFT size implemented)");
  REQUIRE(c.win_size >= 1 && c.win_size <= c.n_fft, B200TTS_EINVAL, "win_size must be in [1, n_fft]");
  REQUIRE(c.hop_size >= 1, B200TTS_EINVAL, "hop_size must be positive");
  REQUIRE(c.num_mels >= 1 && c.num_mels <= kMaMaxMels, B200TTS_EINVAL, "num_mels must be 1..128");
  REQUIRE(c.max_abs_value > 0.f && c.magnitude_power > 0.f && c.rescaling_max > 0.f, B200TTS_EINVAL,
          "max_abs_value, magnitude_power and rescaling_max must be positive");
  REQUIRE(c.min_level_db < 0.f, B200TTS_EINVAL, "min_level_db must be negative");
  REQUIRE(c.trim_fft_size >= 2 && c.trim_hop_size >= 1 && c.trim_top_db > 0.f, B200TTS_EINVAL,
          "trim_fft_size must be >= 2, trim_hop_size and trim_top_db positive");
  check_device(device);
  DeviceGuard dg(device);
  std::unique_ptr<b200tts_mel> ctx(new b200tts_mel());
  ctx->device = device;
  ctx->cfg = c;
  ctx->preemph = shortest_decimal(c.preemphasis);
  ctx->rescale_max = shortest_decimal(c.rescaling_max);
  ctx->min_level = std::exp((double)c.min_level_db / 20 * std::log(10.0));     // _amp_to_db :274
  const int M = c.num_mels, W = c.win_size;
  Packer pk;
  const size_t o_basis = pk.add((size_t)M * kGlBins);
  const size_t o_tw = pk.add(2 * (kGlHalf / 2)), o_tws = pk.add(2 * (kGlHalf / 2 + 1));
  const size_t o_band = pk.add(2 * M), o_win = pk.add(2 * W);
  std::memcpy(pk.h.data() + o_basis, h_mel_basis, sizeof(float) * M * kGlBins);
  int* band = reinterpret_cast<int*>(pk.h.data() + o_band);
  for (int m = 0; m < M; ++m) {                     // non-zero bin range of each band
    int lo = 0, hi = 0;
    const float* row = h_mel_basis + (size_t)m * kGlBins;
    for (int k = 0; k < kGlBins; ++k)
      if (row[k] != 0.f) { if (hi == 0) lo = k; hi = k + 1; }
    band[2 * m] = lo;
    band[2 * m + 1] = hi;
  }
  const double pi = 3.14159265358979323846;
  double* win = reinterpret_cast<double*>(pk.h.data() + o_win);
  for (int j = 0; j < W; ++j) win[j] = 0.5 - 0.5 * std::cos(2.0 * pi * j / W);    // scipy get_window('hann', W): periodic
  fft2048_twiddles(pk.h.data() + o_tw, pk.h.data() + o_tws);
  ctx->consts.ensure(pk.h.size() * sizeof(float));
  B200_CUDA(cudaMemcpy(ctx->consts.p, pk.h.data(), pk.h.size() * sizeof(float), cudaMemcpyHostToDevice));
  const float* base = ctx->consts.as<float>();
  ctx->basis = base + o_basis;
  ctx->tw = reinterpret_cast<const float2*>(base + o_tw);
  ctx->tws = reinterpret_cast<const float2*>(base + o_tws);
  ctx->band = reinterpret_cast<const int2*>(base + o_band);
  ctx->win = reinterpret_cast<const double*>(base + o_win);
  *out = ctx.release();
  API_END
}

extern "C" void b200tts_mel_destroy(b200tts_mel* ctx) {
  if (!ctx) return;
  DeviceGuard dg(ctx->device, true);
  delete ctx;
}

extern "C" int64_t b200tts_mel_launch_count(const b200tts_mel* ctx) { return ctx ? ctx->launches : -1; }

extern "C" int b200tts_mel_analyze(b200tts_mel* ctx, const float* d_wav, const int32_t* d_len, int B, int L_max, int flags,
                                   float* d_mel, int32_t* d_frames, int32_t* d_bounds, float* d_audio, void* stream) {
  API_BEGIN
  REQUIRE(ctx && d_wav && d_len && d_mel && d_frames, B200TTS_EINVAL, "null argument");
  REQUIRE(B >= 1 && B <= 65535, B200TTS_EINVAL, "B must be 1..65535");
  REQUIRE(L_max >= 1 && L_max < (1 << 30), B200TTS_EINVAL, "L_max must be 1..2^30-1");
  REQUIRE((flags & ~(B200TTS_MEL_TRIM | B200TTS_MEL_PREEMPHASIS | B200TTS_MEL_RESCALE)) == 0, B200TTS_EINVAL, "unknown flags");
  const b200tts_mel_cfg& c = ctx->cfg;                                                        // first read of *ctx
  REQUIRE(!(flags & B200TTS_MEL_TRIM) || L_max >= c.trim_fft_size, B200TTS_EINVAL,
          "TRIM needs rows of at least trim_fft_size samples");
  DeviceGuard dg(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  const int T_max = 1 + L_max / c.hop_size;
  const int F_max = 1 + L_max / c.trim_hop_size;
  ctx->rows.ensure((size_t)B * sizeof(MaRow));
  if (flags & B200TTS_MEL_TRIM) ctx->ms.ensure((size_t)B * F_max * sizeof(double));

  MaArgs a{};
  a.wav = d_wav; a.len = d_len; a.Lmax = L_max; a.flags = flags;
  a.trim_n = c.trim_fft_size; a.trim_hop = c.trim_hop_size; a.trim_top_db = c.trim_top_db;
  a.ms = ctx->ms.as<double>(); a.rows = ctx->rows.as<MaRow>(); a.frames = d_frames; a.bounds = d_bounds;
  a.hop = c.hop_size; a.win_len = c.win_size; a.M = c.num_mels; a.Tmax = T_max;
  a.preemph = ctx->preemph; a.rescale_max_d = ctx->rescale_max; a.rescale_max_f = c.rescaling_max;
  a.win = ctx->win; a.tw = ctx->tw; a.tws = ctx->tws; a.basis = ctx->basis; a.band = ctx->band;
  a.mag_power = c.magnitude_power; a.min_level = ctx->min_level; a.min_db = c.min_level_db; a.ref_db = c.ref_level_db;
  a.max_abs = c.max_abs_value;
  a.mel = d_mel; a.audio = d_audio;

  if (flags & B200TTS_MEL_TRIM) {
    ma_trim_power_kernel<<<dim3((F_max + kMaTrimWarps - 1) / kMaTrimWarps, B), kMaThreads, 0, st>>>(a);
    B200_CUDA(cudaGetLastError());
    ctx->launches++;
  }
  ma_bounds_kernel<<<B, kMaBoundsThreads, 0, st>>>(a);
  B200_CUDA(cudaGetLastError());
  ctx->launches++;
  ma_frame_kernel<<<dim3(T_max, B), kMaThreads, 0, st>>>(a);
  B200_CUDA(cudaGetLastError());
  ctx->launches++;
  if (d_audio) {
    const size_t Lout = (size_t)T_max * c.hop_size;
    const unsigned gx = (unsigned)std::min<size_t>((Lout + 4 * kMaThreads - 1) / (4 * kMaThreads), 4096);
    ma_audio_kernel<<<dim3(gx, B), kMaThreads, 0, st>>>(a);
    B200_CUDA(cudaGetLastError());
    ctx->launches++;
  }
  API_END
}
