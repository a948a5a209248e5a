// libb200tts.so -- Griffin-Lim mel inversion (griffin_lim.cuh): b200tts_gl_* and b200tts_griffin_lim.
#include <algorithm>
#include <cmath>

#include "api.h"
#include "griffin_lim.cuh"

using namespace b200tts;

struct b200tts_gl {
  int device = 0;
  b200tts_gl_cfg cfg{};
  DeviceBuf consts;             // pinv [kGlBins][M] | win [W] | win2 [W] | tw [512] float2 | tws [513] float2
  const float *pinv = nullptr, *win = nullptr, *win2 = nullptr;
  const float2 *tw = nullptr, *tws = nullptr;
  DeviceBuf S, frames[2];
  int64_t launches = 0;
};

extern "C" int b200tts_gl_create(b200tts_gl** out, int device, const b200tts_gl_cfg* cfg, const float* h_inv_mel_basis) {
  API_BEGIN
  REQUIRE(out && cfg && h_inv_mel_basis, B200TTS_EINVAL, "null argument");
  *out = nullptr;
  const b200tts_gl_cfg c = *cfg;
  REQUIRE(c.n_fft == kGlN, B200TTS_EINVAL, "n_fft must be 2048 (the only FFT size implemented)");
  REQUIRE(c.win_size >= 1 && c.win_size <= c.n_fft, B200TTS_EINVAL, "win_size must be in [1, n_fft]");
  REQUIRE(c.hop_size >= 1, B200TTS_EINVAL, "hop_size must be positive");
  REQUIRE(c.num_mels >= 1 && c.num_mels <= kGlMaxMels, B200TTS_EINVAL, "num_mels must be 1..128");
  REQUIRE(c.max_abs_value > 0.f && c.magnitude_power > 0.f && c.power > 0.f, B200TTS_EINVAL,
          "max_abs_value, magnitude_power and power must be positive");
  check_device(device);
  DeviceGuard dg(device);
  std::unique_ptr<b200tts_gl> ctx(new b200tts_gl());
  ctx->device = device;
  ctx->cfg = c;
  const int M = c.num_mels, W = c.win_size;
  Packer pk;
  const size_t o_pinv = pk.add((size_t)kGlBins * M), o_win = pk.add(W), o_win2 = pk.add(W);
  const size_t o_tw = pk.add(2 * (kGlHalf / 2)), o_tws = pk.add(2 * (kGlHalf / 2 + 1));
  std::memcpy(pk.h.data() + o_pinv, h_inv_mel_basis, sizeof(float) * kGlBins * M);
  const double pi = 3.14159265358979323846;
  for (int j = 0; j < W; ++j) {                     // scipy get_window('hann', W, fftbins=True): periodic
    const double w = 0.5 - 0.5 * std::cos(2.0 * pi * j / W);
    pk.h[o_win + j] = (float)w;
    pk.h[o_win2 + j] = (float)(w * w);
  }
  fft2048_twiddles(pk.h.data() + o_tw, pk.h.data() + o_tws);
  ctx->consts.ensure(pk.h.size() * sizeof(float));
  B200_CUDA(cudaMemcpy(ctx->consts.p, pk.h.data(), pk.h.size() * sizeof(float), cudaMemcpyHostToDevice));
  const float* base = ctx->consts.as<float>();
  ctx->pinv = base + o_pinv;
  ctx->win = base + o_win;
  ctx->win2 = base + o_win2;
  ctx->tw = reinterpret_cast<const float2*>(base + o_tw);
  ctx->tws = reinterpret_cast<const float2*>(base + o_tws);
  *out = ctx.release();
  API_END
}

extern "C" void b200tts_gl_destroy(b200tts_gl* ctx) {
  if (!ctx) return;
  DeviceGuard dg(ctx->device, true);
  delete ctx;
}

extern "C" int64_t b200tts_gl_launch_count(const b200tts_gl* ctx) { return ctx ? ctx->launches : -1; }

extern "C" int b200tts_griffin_lim(b200tts_gl* ctx, const float* d_mel, const int32_t* d_frames, int B, int T_max,
                                   const b200tts_gl_phase* init, int n_iters, float* d_wave, float* d_u_out, void* stream) {
  API_BEGIN
  REQUIRE(ctx && d_mel && init && d_wave, B200TTS_EINVAL, "null argument");
  REQUIRE(init->mode == B200TTS_GL_PHASE_PHILOX || init->mode == B200TTS_GL_PHASE_EXT, B200TTS_EINVAL, "unknown phase mode");
  REQUIRE(init->mode != B200TTS_GL_PHASE_EXT || init->d_u, B200TTS_EINVAL, "null argument: the EXT phase mode needs d_u");
  REQUIRE(B >= 1 && B <= 65535, B200TTS_EINVAL, "B must be 1..65535");
  REQUIRE(T_max >= 2, B200TTS_EINVAL, "rows need at least 2 frames (T frames give hop * (T - 1) samples)");
  REQUIRE(n_iters >= 0, B200TTS_EINVAL, "n_iters must be >= 0");
  REQUIRE((int64_t)ctx->cfg.hop_size * (T_max - 1) < (1LL << 30), B200TTS_EINVAL, "T_max too large");   // first read of *ctx
  DeviceGuard dg(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  const b200tts_gl_cfg& c = ctx->cfg;
  const size_t nft = (size_t)B * T_max;
  ctx->S.ensure(nft * kGlBins * sizeof(float));
  ctx->frames[0].ensure(nft * c.win_size * sizeof(float));
  ctx->frames[1].ensure(nft * c.win_size * sizeof(float));

  GlMagArgs m{};
  m.mel = d_mel; m.pinv = ctx->pinv; m.frames = d_frames; m.S = ctx->S.as<float>();
  m.Tmax = T_max; m.M = c.num_mels;
  m.max_abs = c.max_abs_value; m.min_db = c.min_level_db; m.ref_db = c.ref_level_db;
  m.inv_mag_power = 1.f / c.magnitude_power; m.power = c.power;
  gl_magnitude_kernel<<<dim3((T_max + kGlMagFrames - 1) / kGlMagFrames, B), kGlThreads, 0, st>>>(m);
  B200_CUDA(cudaGetLastError());
  ctx->launches++;

  GlArgs a{};
  a.S = ctx->S.as<float>(); a.win = ctx->win; a.win2 = ctx->win2; a.tw = ctx->tw; a.tws = ctx->tws; a.frames = d_frames;
  a.Tmax = T_max; a.hop = c.hop_size; a.win_len = c.win_size;
  a.ext = init->mode == B200TTS_GL_PHASE_EXT; a.u_in = init->d_u; a.seed = init->seed; a.utt0 = init->utterance_offset;
  const dim3 grid(T_max, B);
  int cur = 0;
  a.next = ctx->frames[cur].as<float>();
  a.u_out = n_iters == 0 ? d_u_out : nullptr;
  gl_frame_kernel<true><<<grid, kGlThreads, 0, st>>>(a);
  B200_CUDA(cudaGetLastError());
  ctx->launches++;
  for (int i = 0; i < n_iters; ++i) {
    a.prev = ctx->frames[cur].as<float>();
    a.next = ctx->frames[cur ^ 1].as<float>();
    a.u_out = i == n_iters - 1 ? d_u_out : nullptr;
    gl_frame_kernel<false><<<grid, kGlThreads, 0, st>>>(a);
    B200_CUDA(cudaGetLastError());
    ctx->launches++;
    cur ^= 1;
  }
  gl_finish_kernel<<<B, kGlFinishThreads, 0, st>>>(ctx->frames[cur].as<float>(), ctx->win2, d_frames, T_max, c.hop_size, c.win_size,
                                                   c.preemphasis, d_wave);
  B200_CUDA(cudaGetLastError());
  ctx->launches++;
  API_END
}

extern "C" int b200tts_gl_philox_uniform(int device, uint64_t seed, uint64_t utterance_offset, int B, int T, int n_bins, float* d_u,
                                         void* stream) {
  API_BEGIN
  REQUIRE(d_u, B200TTS_EINVAL, "null argument");
  REQUIRE(B >= 1 && T >= 1 && n_bins >= 1, B200TTS_EINVAL, "B, T and n_bins must be positive");
  DeviceGuard dg(device);
  const size_t total = (size_t)B * T * n_bins;
  const unsigned grid = (unsigned)std::min<size_t>((total + 255) / 256, 132 * 16);
  gl_philox_dump_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(seed, utterance_offset, B, T, n_bins, d_u);
  B200_CUDA(cudaGetLastError());
  API_END
}
