// libb200tts.so -- WaveRNN vocoder (wavernn_*.cuh): b200tts_wavernn_*, b200tts_philox_exponential / _mol_uniform, weight
// packing and the choice of generation kernel.
#include <cooperative_groups.h>
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <set>

#include "api.h"
#include "wavernn_upsample.cuh"
#include "wavernn_utt.cuh"
#include "wavernn_grid.cuh"
#include "wavernn_push.cuh"
#include "wavernn_tc.cuh"
#include "wavernn_open.cuh"

using namespace b200tts;

// One RAW utterance generated in pieces on the push kernel or the tensor cores (b200tts_wavernn_session_*): its conditioning
// tables, computed once at open, and the state its last run saved (SessRow; its layout depends on the kernel, so a session stays
// on the kernel it was opened for).  Owned by its context, which frees the sessions still open.
struct b200tts_wavernn_session {
  b200tts_wavernn* ctx = nullptr;
  bool tc = false;                          // runs on wavernn_tc_session_kernel (else the push session kernel)
  int T = 0, mu_law = 1;
  int64_t pos = 0, S = 0, wave_len = 0;     // next step; steps of the utterance; samples of its wave
  uint64_t seed = 0, id = 0;
  std::shared_ptr<DeviceBuf> mem;           // one allocation for the sessions opened together, freed with the last of them
  float* tab = nullptr;                     // this session's tables and state, in `mem`
  float* state = nullptr;
};

struct b200tts_wavernn {
  int device = 0;
  b200tts_wavernn_cfg cfg{};
  bool mol = false;               // voc_mode = 'MOL' (b200tts_wavernn_create_mol): fc3 gives 30 mixture parameters
  int NC = 0, NT = 0, sm_count = 0;   // NC: fc3 rows as packed (MOL: the 30 parameters padded to 32)
  DeviceBuf weights;          // original layouts, one blob (pack_original)
  StepWeights sw{};
  ResnetParams rp{};
  const float* d_fir = nullptr;   // [hop][NT]
  GridModel gm{};                 // per-CTA weight blobs of the grid kernel
  DeviceBuf grid_blob, mels_T, aux_T, grid_sync, fold_mels, fold_aux, grid_mol_par;
  PushModel pm{};                 // small-batch push kernel (wavernn_push.cuh): per-CTA blobs + conditioning-projection weights
  PushCondW pcw{};
  DeviceBuf push_blob, push_condw, push_tab, push_vec, push_best;
  DeviceBuf tc_wimg, tc_prm, tc_vec, tc_x1f, tc_win, tc_cnt, tc_cond;     // tensor-core pipeline (wavernn_tc.cuh)
  bool tc_ok = false;
  // the last launch of a step kernel
  int last_kernel = 0;            // its StepKernel; 0 before the first
  DeviceBuf prof;                 // its phase counters [prof_ncta][12] (B200TTS_GRID_PROF)
  int prof_ncta = 0;              // 0: it recorded none
  DeviceBuf error;                // one int, zeroed per generate call; set by any of its kernels that gave up waiting for a peer CTA
  // scratch
  DeviceBuf mels_up, aux_frames, labels, mel_in, wave, grid_scratch;
  HostPinned h_stage;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  bool ev_valid = false;
  int64_t launches = 0;
  bool warned_fallback = false;
  std::set<b200tts_wavernn_session*> sessions;   // open sessions, freed with the context
  DeviceBuf sess_labels;                         // labels of a session run whose caller passed none
  ~b200tts_wavernn() {
    for (b200tts_wavernn_session* s : sessions) delete s;
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
  }
};

void b200tts::launch_push_init(uint32_t* vec, size_t nvec, unsigned long long* best, size_t nbest, int* error, int grid,
                                cudaStream_t st) {
  push_init_kernel<<<grid, 256, 0, st>>>(vec, nvec, best, nbest, error);
  B200_CUDA(cudaGetLastError());
}

// Composite polyphase FIR of the Stretch2d/Conv2d chain (see wavernn_upsample.cuh).  Returns [hop][NT] doubles.
static std::vector<double> composite_fir(const b200tts_wavernn_cfg& c, const std::vector<std::vector<double>>& taps,
                                         int* NT_out) {
  const int hop = c.hop_length;
  // reach of the composite response beyond the frame's own box, in output samples
  int reach = 0, rate = hop;
  for (int j = 0; j < c.n_upsample; ++j) {
    rate /= c.upsample_factors[j];
    reach += c.upsample_factors[j] * rate;
  }
  int side = (reach + hop - 1) / hop;            // frames on each side that can contribute
  int NT = 2 * side + 1;
  REQUIRE(NT <= kMaxTaps, B200TTS_EINVAL, "upsample factors give a composite FIR wider than kMaxTaps frames");
  const int nf = 2 * side + 5, f0 = nf / 2;      // impulse in the middle, far from both ends
  std::vector<double> x(nf, 0.0);
  x[f0] = 1.0;
  for (int j = 0; j < c.n_upsample; ++j) {
    const int s = c.upsample_factors[j];
    std::vector<double> r(x.size() * s);
    for (size_t i = 0; i < r.size(); ++i) r[i] = x[i / s];
    std::vector<double> y(r.size(), 0.0);
    for (long i = 0; i < (long)r.size(); ++i) {
      double a = 0.0;
      for (int k = 0; k < 2 * s + 1; ++k) {
        long idx = i + k - s;
        if (idx >= 0 && idx < (long)r.size()) a += taps[j][k] * r[idx];
      }
      y[i] = a;
    }
    x.swap(y);
  }
  // out[n] = sum_f melpad[f] * Rsp[n - hop*f];  with n = hop*fr + ph and f = fr + (j - side):  Rsp[ph - hop*(j-side)]
  std::vector<double> fir((size_t)hop * NT);
  for (int ph = 0; ph < hop; ++ph)
    for (int j = 0; j < NT; ++j) {
      long idx = (long)hop * f0 + ph - (long)hop * (j - side);
      fir[(size_t)ph * NT + j] = (idx >= 0 && idx < (long)x.size()) ? x[idx] : 0.0;
    }
  *NT_out = NT;
  return fir;
}

// The original layouts: step weights (rows of I padded to ldI), MelResNet transposed to [in][out] with its BatchNorms folded, and
// the composite FIR.  Uploads them as one blob and points ctx->sw, ctx->rp and ctx->d_fir into it; returns the step weights as
// pointers into the host copy `pk`, from which the grid kernel's blobs are cut.
static StepWeights pack_original(b200tts_wavernn* ctx, const TensorMap& tm, Packer& pk) {
  const b200tts_wavernn_cfg& c = ctx->cfg;
  const int R = c.rnn_dims, F = c.fc_dims, AUX = c.res_out_dims / 4, FEAT = c.feat_dims, NC = ctx->NC;
  const int C = c.compute_dims, O = c.res_out_dims, K = 2 * c.pad + 1;
  // ---- step weights ----
  const int nin = 1 + FEAT + AUX, ldI = round4(nin);
  const float* Iw = need(tm, "I.weight", {R, nin})->data;
  size_t oI = pk.add((size_t)R * ldI);
  for (int r = 0; r < R; ++r) std::memcpy(&pk.h[oI + (size_t)r * ldI], Iw + (size_t)r * nin, sizeof(float) * nin);
  size_t oIb = pk.copy(tm, "I.bias", {R});
  size_t o_ih1 = pk.copy(tm, "rnn1.weight_ih_l0", {3 * R, R}), o_hh1 = pk.copy(tm, "rnn1.weight_hh_l0", {3 * R, R});
  size_t o_bih1 = pk.copy(tm, "rnn1.bias_ih_l0", {3 * R}), o_bhh1 = pk.copy(tm, "rnn1.bias_hh_l0", {3 * R});
  size_t o_ih2 = pk.copy(tm, "rnn2.weight_ih_l0", {3 * R, R + AUX}), o_hh2 = pk.copy(tm, "rnn2.weight_hh_l0", {3 * R, R});
  size_t o_bih2 = pk.copy(tm, "rnn2.bias_ih_l0", {3 * R}), o_bhh2 = pk.copy(tm, "rnn2.bias_hh_l0", {3 * R});
  size_t o_fc1 = pk.copy(tm, "fc1.weight", {F, R + AUX}), o_fc1b = pk.copy(tm, "fc1.bias", {F});
  size_t o_fc2 = pk.copy(tm, "fc2.weight", {F, F + AUX}), o_fc2b = pk.copy(tm, "fc2.bias", {F});
  size_t o_fc3, o_fc3b;
  if (ctx->mol) {               // 30 rows padded with zero rows to NC = 32: the step kernels dot whole quads of rows
    const float* w = need(tm, "fc3.weight", {kMolParams, F})->data;
    const float* b = need(tm, "fc3.bias", {kMolParams})->data;
    o_fc3 = pk.add((size_t)NC * F);
    o_fc3b = pk.add((size_t)NC);
    std::memcpy(&pk.h[o_fc3], w, sizeof(float) * kMolParams * F);
    std::memcpy(&pk.h[o_fc3b], b, sizeof(float) * kMolParams);
  } else {
    o_fc3 = pk.copy(tm, "fc3.weight", {NC, F});
    o_fc3b = pk.copy(tm, "fc3.bias", {NC});
  }

  // ---- MelResNet, transposed to [in][out]; BatchNorm (eval, eps 1e-5) folded to scale/shift in double ----
  const float* cin = need(tm, "upsample.resnet.conv_in.weight", {C, FEAT, K})->data;
  size_t o_cin = pk.add((size_t)FEAT * K * C);
  for (int cc = 0; cc < C; ++cc)
    for (int i = 0; i < FEAT; ++i)
      for (int j = 0; j < K; ++j) pk.h[o_cin + ((size_t)i * K + j) * C + cc] = cin[((size_t)cc * FEAT + i) * K + j];
  const int nbn = 1 + 2 * c.res_blocks;
  size_t o_bns = pk.add((size_t)nbn * C), o_bnh = pk.add((size_t)nbn * C);
  auto fold_bn = [&](const std::string& prefix, int slot) {
    const float* g = need(tm, prefix + ".weight", {C})->data;
    const float* b = need(tm, prefix + ".bias", {C})->data;
    const float* m = need(tm, prefix + ".running_mean", {C})->data;
    const float* v = need(tm, prefix + ".running_var", {C})->data;
    for (int cc = 0; cc < C; ++cc) {
      double sc = (double)g[cc] / std::sqrt((double)v[cc] + 1e-5);
      pk.h[o_bns + (size_t)slot * C + cc] = (float)sc;
      pk.h[o_bnh + (size_t)slot * C + cc] = (float)((double)b[cc] - (double)m[cc] * sc);
    }
  };
  fold_bn("upsample.resnet.batch_norm", 0);
  size_t o_res = pk.add((size_t)c.res_blocks * 2 * C * C);
  for (int blk = 0; blk < c.res_blocks; ++blk) {
    std::string p = "upsample.resnet.layers." + std::to_string(blk);
    for (int h = 0; h < 2; ++h) {
      const float* w = need(tm, p + (h ? ".conv2.weight" : ".conv1.weight"), {C, C, 1})->data;
      size_t base = o_res + ((size_t)blk * 2 + h) * C * C;
      for (int co = 0; co < C; ++co)
        for (int ci = 0; ci < C; ++ci) pk.h[base + (size_t)ci * C + co] = w[(size_t)co * C + ci];
    }
    fold_bn(p + ".batch_norm1", 1 + 2 * blk);
    fold_bn(p + ".batch_norm2", 2 + 2 * blk);
  }
  const float* cow = need(tm, "upsample.resnet.conv_out.weight", {O, C, 1})->data;
  size_t o_cout = pk.add((size_t)C * O);
  for (int o = 0; o < O; ++o)
    for (int ci = 0; ci < C; ++ci) pk.h[o_cout + (size_t)ci * O + o] = cow[(size_t)o * C + ci];
  size_t o_coutb = pk.copy(tm, "upsample.resnet.conv_out.bias", {O});

  // ---- composite FIR ----
  std::vector<std::vector<double>> taps(c.n_upsample);
  for (int j = 0; j < c.n_upsample; ++j) {
    int s = c.upsample_factors[j];
    const float* w = need(tm, "upsample.up_layers." + std::to_string(2 * j + 1) + ".weight", {1, 1, 1, 2 * s + 1})->data;
    taps[j].assign(w, w + 2 * s + 1);
  }
  int NT = 0;
  std::vector<double> fir = composite_fir(c, taps, &NT);
  ctx->NT = NT;
  size_t o_fir = pk.add(fir.size());
  for (size_t i = 0; i < fir.size(); ++i) pk.h[o_fir + i] = (float)fir[i];

  ctx->weights.ensure(pk.h.size() * sizeof(float));
  B200_CUDA(cudaMemcpy(ctx->weights.p, pk.h.data(), pk.h.size() * sizeof(float), cudaMemcpyHostToDevice));
  auto step_weights = [&](const float* base) {
    StepWeights sw{};
    sw.I_w = base + oI; sw.I_b = base + oIb;
    sw.ih1_w = base + o_ih1; sw.hh1_w = base + o_hh1; sw.ih1_b = base + o_bih1; sw.hh1_b = base + o_bhh1;
    sw.ih2_w = base + o_ih2; sw.hh2_w = base + o_hh2; sw.ih2_b = base + o_bih2; sw.hh2_b = base + o_bhh2;
    sw.fc1_w = base + o_fc1; sw.fc1_b = base + o_fc1b; sw.fc2_w = base + o_fc2; sw.fc2_b = base + o_fc2b;
    sw.fc3_w = base + o_fc3; sw.fc3_b = base + o_fc3b;
    sw.R = R; sw.F = F; sw.aux = AUX; sw.feat = FEAT; sw.NC = NC; sw.ldI = ldI;
    return sw;
  };
  const float* base = ctx->weights.as<float>();
  ctx->sw = step_weights(base);
  ResnetParams& rp = ctx->rp;
  rp.conv_in_t = base + o_cin; rp.bn_scale = base + o_bns; rp.bn_shift = base + o_bnh; rp.res_w_t = base + o_res;
  rp.conv_out_t = base + o_cout; rp.conv_out_b = base + o_coutb;
  rp.feat = FEAT; rp.k = K; rp.C = C; rp.O = O; rp.blocks = c.res_blocks; rp.pad = c.pad;
  ctx->d_fir = base + o_fir;
  return step_weights(pk.h.data());
}

template <class V>
static void upload(DeviceBuf& d, const V& h) {
  if (h.empty()) return;
  d.ensure(h.size() * sizeof(h[0]));
  B200_CUDA(cudaMemcpy(d.p, h.data(), h.size() * sizeof(h[0]), cudaMemcpyHostToDevice));
}

static int create_context(b200tts_wavernn** out, int device, const b200tts_wavernn_cfg* cfg, const b200tts_tensor* weights,
                          int n_weights, bool mol) {
  API_BEGIN
  REQUIRE(out && cfg && weights && n_weights > 0, B200TTS_EINVAL, "null argument");
  *out = nullptr;
  const b200tts_wavernn_cfg& c = *cfg;
  REQUIRE(c.n_upsample >= 1 && c.n_upsample <= 4, B200TTS_EINVAL, "n_upsample must be 1..4");
  int prod = 1;
  for (int j = 0; j < c.n_upsample; ++j) {
    REQUIRE(c.upsample_factors[j] >= 1, B200TTS_EINVAL, "bad upsample factor");
    prod *= c.upsample_factors[j];
  }
  REQUIRE(prod == c.hop_length, B200TTS_EINVAL, "prod(upsample_factors) != hop_length (wavernn_train.py:67 asserts the same)");
  REQUIRE(c.res_out_dims % 4 == 0, B200TTS_EINVAL, "res_out_dims must be divisible by 4");
  REQUIRE(c.rnn_dims % 128 == 0 && c.fc_dims % 128 == 0, B200TTS_EINVAL, "rnn_dims / fc_dims must be multiples of 128");
  REQUIRE(mol || (c.bits >= 2 && c.bits <= 15), B200TTS_EINVAL, "bits must be 2..15 (labels are int16)");
  REQUIRE(c.compute_dims <= 1024 && c.res_out_dims <= 1024, B200TTS_EINVAL, "compute/res_out dims too large");
  REQUIRE(c.pad >= 1, B200TTS_EINVAL,
          "pad must be >= 1: the reference trims pad * hop_length samples from each end of the upsampled mels "
          "(fatchord_version.py:88), which leaves nothing at pad 0");
  REQUIRE(c.feat_dims >= 1, B200TTS_EINVAL, "feat_dims must be >= 1 (mel channels)");
  REQUIRE(c.compute_dims >= 1, B200TTS_EINVAL, "compute_dims must be >= 1 (MelResNet channels)");
  REQUIRE(c.res_blocks >= 0, B200TTS_EINVAL, "res_blocks must be >= 0");
  const int AUX = c.res_out_dims / 4, FEAT = c.feat_dims;
  REQUIRE(AUX % 4 == 0, B200TTS_EINVAL, "aux dims (res_out_dims/4) must be a multiple of 4");
  check_device(device);
  DeviceGuard dg(device);

  TensorMap tm;
  for (int i = 0; i < n_weights; ++i)
    if (weights[i].name) tm[weights[i].name] = &weights[i];

  std::unique_ptr<b200tts_wavernn> ctx(new b200tts_wavernn());
  ctx->device = device;
  ctx->cfg = c;
  ctx->mol = mol;
  ctx->NC = mol ? round4(kMolParams) : 1 << c.bits;
  int coop = 0;
  B200_CUDA(cudaDeviceGetAttribute(&ctx->sm_count, cudaDevAttrMultiProcessorCount, device));
  B200_CUDA(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, device));

  // Each kernel's weights are cut from the host blobs of the one before it (grid -> push -> tensor cores), so each capability
  // implies the previous one.
  Packer pk;
  StepWeights hw = pack_original(ctx.get(), tm, pk);
  std::vector<float> mol_w3, mol_b3;
  if (mol) {                    // the grid and push kernels take fc3 as 2R classes, 8 per CTA: parameter j becomes class 8j
    mol_w3.assign((size_t)2 * c.rnn_dims * c.fc_dims, 0.f);
    mol_b3.assign((size_t)2 * c.rnn_dims, 0.f);
    for (int j = 0; j < kMolParams; ++j) {
      std::memcpy(&mol_w3[(size_t)kCPC * j * c.fc_dims], hw.fc3_w + (size_t)j * c.fc_dims, sizeof(float) * c.fc_dims);
      mol_b3[(size_t)kCPC * j] = hw.fc3_b[j];
    }
    hw.fc3_w = mol_w3.data();
    hw.fc3_b = mol_b3.data();
    hw.NC = 2 * c.rnn_dims;
  }
  {
    const std::vector<float> gb = pack_grid_model(hw, ctx->sm_count, coop != 0, ctx->gm);
    upload(ctx->grid_blob, gb);
    std::vector<float> cw;
    const std::vector<float> pb = pack_push_model(ctx->gm, gb, c.hop_length, ctx->NT, ctx->pm, cw);
    upload(ctx->push_blob, pb);
    upload(ctx->push_condw, cw);
    if (ctx->pm.ok) {
      const int n = ctx->pm.ncta;
      const float* cwd = ctx->push_condw.as<float>();
      ctx->pcw = PushCondW{cwd, cwd + (size_t)n * 16 * FEAT, cwd + (size_t)n * (16 * FEAT + 36 * AUX), n, FEAT, AUX};
    }
    if (!mol) {                 // MOL models do not run on the tensor cores (choose_kernel)
      std::vector<uint16_t> img;
      std::vector<float> prm;
      ctx->tc_ok = pack_tc_images(ctx->pm, pb, ctx->sm_count, c.hop_length * ctx->NT, img, prm);
      upload(ctx->tc_wimg, img);
      upload(ctx->tc_prm, prm);
    }
  }

  ctx->error.ensure(sizeof(int));
  B200_CUDA(cudaMemset(ctx->error.p, 0, sizeof(int)));
  B200_CUDA(cudaEventCreate(&ctx->ev0));
  B200_CUDA(cudaEventCreate(&ctx->ev1));
  *out = ctx.release();
  API_END
}

extern "C" int b200tts_wavernn_create(b200tts_wavernn** out, int device, const b200tts_wavernn_cfg* cfg,
                                      const b200tts_tensor* weights, int n_weights) {
  return create_context(out, device, cfg, weights, n_weights, false);
}

extern "C" int b200tts_wavernn_create_mol(b200tts_wavernn** out, int device, const b200tts_wavernn_cfg* cfg,
                                          const b200tts_tensor* weights, int n_weights) {
  return create_context(out, device, cfg, weights, n_weights, true);
}

extern "C" void b200tts_wavernn_destroy(b200tts_wavernn* ctx) {
  if (!ctx) return;
  DeviceGuard dg(ctx->device, true);
  delete ctx;
}

extern "C" int64_t b200tts_wavernn_launch_count(const b200tts_wavernn* ctx) { return ctx ? ctx->launches : -1; }

extern "C" int b200tts_wavernn_last_kernel(const b200tts_wavernn* ctx) { return ctx ? ctx->last_kernel : 0; }

// After the stream has been synchronised: did a kernel of the last generate call or session run give up waiting for a peer CTA?
static void check_call_error(b200tts_wavernn* ctx) {
  int flag = 0;
  B200_CUDA(cudaMemcpy(&flag, ctx->error.p, sizeof(int), cudaMemcpyDeviceToHost));
  REQUIRE(flag == 0, B200TTS_ECUDA, "grid kernel: a grid-barrier wait timed out (co-resident CTA missing); results are invalid");
}

extern "C" double b200tts_wavernn_last_kernel_ms(b200tts_wavernn* ctx) {
  if (!ctx || !ctx->ev_valid) {
    g_err = "no generate call has been timed on this context";
    return -1.0;
  }
  float ms = 0.f;
  cudaError_t e = cudaEventSynchronize(ctx->ev1);
  if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1);
  if (e != cudaSuccess) {
    g_err = std::string("cudaEventElapsedTime: ") + cudaGetErrorString(e);
    return -1.0;
  }
  try {
    check_call_error(ctx);
  } catch (const Error& err) {
    g_err = err.what();
    return -1.0;
  }
  return (double)ms;
}

// ---- conditioning ---------------------------------------------------------------------------------
static void run_upsample(b200tts_wavernn* ctx, const float* d_mel, int B, int T, float* d_mels_up, float* d_aux_frames,
                         float* d_aux_full, cudaStream_t st) {
  const b200tts_wavernn_cfg& c = ctx->cfg;
  const int hop = c.hop_length, O = c.res_out_dims;
  float* auxf = d_aux_frames;
  if (!auxf && d_aux_full) {
    ctx->aux_frames.ensure((size_t)B * T * O * sizeof(float));
    auxf = ctx->aux_frames.as<float>();
  }
  if (auxf) {
    constexpr int FT = 8;
    int threads = ((std::max(c.compute_dims, 32) + 31) / 32) * 32;
    size_t smem = ((size_t)c.feat_dims * (2 * c.pad + 1) * FT + 2 * (size_t)c.compute_dims * FT) * sizeof(float);
    if (smem > 48 * 1024)
      B200_CUDA(cudaFuncSetAttribute(melresnet_kernel<FT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid((T + FT - 1) / FT, B);
    melresnet_kernel<FT><<<grid, threads, smem, st>>>(ctx->rp, d_mel, T, auxf);
    B200_CUDA(cudaGetLastError());
    ctx->launches++;
  }
  if (d_mels_up) {
    size_t n = (size_t)T * hop * c.feat_dims;
    dim3 grid((unsigned)std::min<size_t>((n + 255) / 256, 4096), B);
    mel_fir_kernel<<<grid, 256, 0, st>>>(d_mel, ctx->d_fir, T, c.feat_dims, hop, c.pad, ctx->NT, d_mels_up);
    B200_CUDA(cudaGetLastError());
    ctx->launches++;
  }
  if (d_aux_full) {
    size_t n = (size_t)T * hop * O;
    dim3 grid((unsigned)std::min<size_t>((n + 255) / 256, 4096), B);
    aux_repeat_kernel<<<grid, 256, 0, st>>>(auxf, T, hop, O, d_aux_full);
    B200_CUDA(cudaGetLastError());
    ctx->launches++;
  }
}

extern "C" int b200tts_wavernn_upsample(b200tts_wavernn* ctx, const float* d_mel, int B, int T, float* d_mels_up,
                                        float* d_aux_frames, float* d_aux_full, void* stream) {
  API_BEGIN
  REQUIRE(ctx && d_mel, B200TTS_EINVAL, "null argument");
  REQUIRE(B >= 1 && T >= 1, B200TTS_EINVAL, "B and T must be positive");
  REQUIRE(B <= 65535, B200TTS_EINVAL, "B must be <= 65535");
  DeviceGuard dg(ctx->device);
  run_upsample(ctx, d_mel, B, T, d_mels_up, d_aux_frames, d_aux_full, (cudaStream_t)stream);
  API_END
}

// ---- generation -----------------------------------------------------------------------------------
// The step kernel a launch runs; the values are those b200tts_wavernn_last_kernel reports.
enum StepKernel { SK_UTTERANCE = 1, SK_GRID = 2, SK_PUSH = 3, SK_TC = 5, SK_SESSION = 6, SK_TC_SESSION = 7 };

// The fields every step kernel's arguments take from GenArgs as they are: noise, debug buffers, labels.
template <class Args>
static void copy_gen_fields(Args& a, const GenArgs& g) {
  a.rng_mode = g.rng_mode; a.seed = g.seed; a.utt_offset = g.utt_offset; a.utt_ids = g.utt_ids; a.q = g.q;
  a.teacher = g.teacher; a.logits_out = g.logits_out; a.labels = g.labels;
}

// Zeroed phase counters [ncta][12] for the launch when `prof`, else null.
static long long* phase_counters(b200tts_wavernn* ctx, bool prof, int ncta, cudaStream_t st) {
  if (!prof) return nullptr;
  const size_t bytes = (size_t)ncta * 12 * sizeof(long long);
  ctx->prof.ensure(bytes);
  B200_CUDA(cudaMemsetAsync(ctx->prof.p, 0, bytes, st));
  return ctx->prof.as<long long>();
}

// Launches `kern`, step kernel `sk` of a generate call or session run, on `grid` CTAs, timed by ev0 / ev1 (`prof`: it fills
// the phase counters), and records what b200tts_wavernn_last_kernel, _last_kernel_ms and _debug_phase_cycles report.  The
// kernel is recorded before the checks here, so a call they refuse reports the kernel it chose; nothing between a call's
// choice of kernel and this launch refuses.  Every step kernel but the utterance kernel keeps all its CTAs resident at once
// and is launched cooperatively.  `args` may hold more arguments than the kernel takes.
static void launch_step(b200tts_wavernn* ctx, StepKernel sk, const void* kern, const char* what, int grid, int threads, size_t smem,
                        void** args, bool prof, cudaStream_t st) {
  ctx->last_kernel = sk;
  ctx->prof_ncta = prof ? grid : 0;
  const bool coop = sk != SK_UTTERANCE;
  REQUIRE(coop || smem <= 227 * 1024, B200TTS_EINVAL, "model too large for the utterance kernel's shared memory");
  B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  if (coop) B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem));
  REQUIRE(!coop || per_sm * ctx->sm_count >= grid, B200TTS_EINVAL, std::string(what) + " cannot be made co-resident on this device");
  B200_CUDA(cudaEventRecord(ctx->ev0, st));
  if (coop) B200_CUDA(cudaLaunchCooperativeKernel(kern, dim3(grid), dim3(threads), args, smem, st));
  else B200_CUDA(cudaLaunchKernel(kern, dim3(grid), dim3(threads), args, smem, st));
  ctx->launches++;
  B200_CUDA(cudaEventRecord(ctx->ev1, st));
  ctx->ev_valid = true;
}

template <int G>
static void launch_utt(b200tts_wavernn* ctx, GenArgs& a, const MolIO* mol, cudaStream_t st) {
  StepWeights w = ctx->sw;
  MolIO io = mol ? *mol : MolIO{};
  void* args[] = {(void*)&w, (void*)&a, (void*)&io};
  const void* kern = mol ? (const void*)wavernn_utt_mol_kernel<G> : (const void*)wavernn_utt_kernel<G>;
  launch_step(ctx, SK_UTTERANCE, kern, "utterance kernel", (a.B + G - 1) / G, kUttThreads, utt_smem_floats(w, G) * sizeof(float),
              args, false, st);
}

struct FoldGeom {           // fold_with_overlap geometry (fatchord_version.py:319-330)
  int nfold, L, stride;
};
// The geometry of an S-sample utterance, or a refusal.  The fold length target + 2 * overlap must fit an int: it is the step
// count of every fold.
static FoldGeom fold_geometry(long long S, int target, int overlap) {
  REQUIRE(target >= 1 && overlap >= 2, B200TTS_EINVAL, "fold target/overlap out of range (target >= 1, overlap >= 2)");
  REQUIRE(S > overlap, B200TTS_EINVAL, "utterance shorter than the fold overlap");
  REQUIRE(S <= INT_MAX && (long long)target + 2LL * overlap <= INT_MAX, B200TTS_EINVAL,
          "utterance or fold longer than 2^31 - 1 samples");
  FoldGeom g{};
  g.stride = target + overlap;
  g.L = target + 2 * overlap;
  const long long num_folds = (S - overlap) / g.stride;
  const long long extended = num_folds * g.stride + overlap;
  g.nfold = (int)(num_folds + (S - extended != 0 ? 1 : 0));
  return g;
}

// `fold` != null: `a` describes the folded problem (B = nfold, S = T = L, hop = 1); the conditioning of the single source utterance
// of S0 samples, in ctx->mels_up [S0][feat] / ctx->aux_frames [T0][O], is cut into the per-fold rows this kernel reads first.
// `mol` != null: a MOL context's generation, with its sample buffers.
static void launch_utterance(b200tts_wavernn* ctx, GenArgs a, const MolIO* mol, cudaStream_t st, const FoldGeom* fold, int S0) {
  const b200tts_wavernn_cfg& c = ctx->cfg;
  if (fold) {
    const int O = c.res_out_dims;
    ctx->fold_mels.ensure((size_t)a.B * a.S * c.feat_dims * sizeof(float));
    ctx->fold_aux.ensure((size_t)a.B * a.S * O * sizeof(float));
    size_t n = (size_t)a.B * a.S * (c.feat_dims + O);
    unsigned grid = (unsigned)std::min<size_t>((n + 255) / 256, (size_t)ctx->sm_count * 32);
    fold_cond_kernel<<<grid, 256, 0, st>>>(ctx->mels_up.as<float>(), ctx->aux_frames.as<float>(), S0, c.hop_length, c.feat_dims, O,
                                           fold->L, fold->stride, fold->nfold, ctx->fold_mels.as<float>(), ctx->fold_aux.as<float>());
    B200_CUDA(cudaGetLastError());
    ctx->launches++;
    a.mels_up = ctx->fold_mels.as<float>();
    a.aux_frames = ctx->fold_aux.as<float>();
  }
  // utterances per CTA: enough CTAs to cover the SMs first, then amortise the L2 weight stream over more rows, as many as fit in
  // shared memory (wide or many-class models: 8 rows of 12-bit classes need 285 KB); choose_kernel refuses a model whose
  // single row does not fit
  const int per = (a.B + ctx->sm_count - 1) / ctx->sm_count;
  int G = per <= 1 ? 1 : per <= 2 ? 2 : per <= 4 ? 4 : 8;
  while (G > 1 && !utt_fits(ctx->sw, G)) G /= 2;
  if (G == 1) launch_utt<1>(ctx, a, mol, st);
  else if (G == 2) launch_utt<2>(ctx, a, mol, st);
  else if (G == 4) launch_utt<4>(ctx, a, mol, st);
  else launch_utt<8>(ctx, a, mol, st);
}

template <int U, int UW, int GROUPS>
static void launch_grid_t(b200tts_wavernn* ctx, GridArgs& a, const MolIO* mol, cudaStream_t st) {
  using MT = MapTraits<U, UW, GROUPS>;
  GridModel gm = ctx->gm;
  size_t smem = ((size_t)gm.blob + (size_t)MT::kScratchFloats) * sizeof(float);
  MolIO io = mol ? *mol : MolIO{};
  void* args[] = {(void*)&gm, (void*)&a, (void*)&io};
  const void* kern = mol ? (const void*)wavernn_grid_mol_kernel<U, UW, GROUPS> : (const void*)wavernn_grid_kernel<U, UW, GROUPS>;
  launch_step(ctx, SK_GRID, kern, "grid kernel", gm.ncta, MT::NW * 32, smem, args, a.prof != nullptr, st);
}

// Mapping for B utterances: returns the padded batch; variant = index into the dispatch table below.
enum { GV_N4, GV_W1, GV_W2, GV_W4, GV_W4x2 };
static int grid_variant(int B, int* variant) {
  if (B <= 4) { *variant = GV_N4; return 4; }
  if (B <= 32) { *variant = GV_W1; return 32; }     // 5..8 utterances too: on the previous GPU the 8-row narrow mapping
                                                    // measured 30.7 us/step against 29.4 us for this one
  if (B <= 64) { *variant = GV_W2; return 64; }
  if (B <= 128) { *variant = GV_W4; return 128; }
  *variant = GV_W4x2;
  return (B + 255) / 256 * 256;
}

// `fold` != null: `ua` already describes the folded problem (B = nfold, S = T = L, hop = 1) and the conditioning of the
// single source utterance is in ctx->mels_up [S0][feat] / ctx->aux_frames [T0][O].
static void launch_grid(b200tts_wavernn* ctx, const float* d_mel, const GenArgs& ua, const MolIO* mol, bool prof, cudaStream_t st,
                        const FoldGeom* fold, int S0) {
  const b200tts_wavernn_cfg& c = ctx->cfg;
  const GridModel& g = ctx->gm;
  int variant = 0;
  const int B = ua.B, T = ua.T, S = ua.S, O = c.res_out_dims;
  const int Bp = grid_variant(B, &variant);
  // conditioning in K-major layout
  ctx->mels_T.ensure((size_t)S * c.feat_dims * Bp * sizeof(float));
  ctx->aux_T.ensure((size_t)T * O * Bp * sizeof(float));
  if (fold) {
    size_t n = (size_t)S * (c.feat_dims + O) * Bp;
    unsigned grid = (unsigned)std::min<size_t>((n + 255) / 256, (size_t)ctx->sm_count * 32);
    fold_cond_T_kernel<<<grid, 256, 0, st>>>(ctx->mels_up.as<float>(), ctx->aux_frames.as<float>(), S0, c.hop_length, c.feat_dims, O,
                                             fold->L, fold->stride, fold->nfold, Bp, ctx->mels_T.as<float>(), ctx->aux_T.as<float>());
    B200_CUDA(cudaGetLastError());
    ctx->launches += 1;
  } else {
    size_t n = (size_t)S * c.feat_dims * Bp;
    unsigned grid = (unsigned)std::min<size_t>((n + 255) / 256, (size_t)ctx->sm_count * 32);
    mel_fir_T_kernel<<<grid, 256, 0, st>>>(d_mel, ctx->d_fir, B, Bp, T, c.feat_dims, c.hop_length, c.pad, ctx->NT,
                                           ctx->mels_T.as<float>());
    B200_CUDA(cudaGetLastError());
    n = (size_t)T * O * Bp;
    grid = (unsigned)std::min<size_t>((n + 255) / 256, (size_t)ctx->sm_count * 32);
    aux_T_kernel<<<grid, 256, 0, st>>>(ua.aux_frames, B, Bp, T, O, ctx->aux_T.as<float>());
    B200_CUDA(cudaGetLastError());
    ctx->launches += 2;
  }
  // activations + sync words, zero-initialised (h1 = h2 = 0, fatchord_version.py:194-195)
  const size_t RB = (size_t)g.R * Bp;
  const size_t act_floats = 8 * RB;
  const size_t sync_bytes = 2 * (size_t)Bp * sizeof(unsigned long long) + 512;
  ctx->grid_scratch.ensure(act_floats * sizeof(float));
  ctx->grid_sync.ensure(sync_bytes);
  B200_CUDA(cudaMemsetAsync(ctx->grid_scratch.p, 0, act_floats * sizeof(float), st));
  B200_CUDA(cudaMemsetAsync(ctx->grid_sync.p, 0, sync_bytes, st));
  float* base = ctx->grid_scratch.as<float>();
  GridArgs a{};
  a.wblob = ctx->grid_blob.as<float>();
  a.h1 = base; a.h2 = base + 2 * RB; a.x1 = base + 4 * RB; a.x2 = base + 5 * RB;
  a.f1 = base + 6 * RB; a.f2 = base + 7 * RB;
  a.best = ctx->grid_sync.as<unsigned long long>();
  a.barrier = reinterpret_cast<unsigned int*>(ctx->grid_sync.as<char>() + 2 * (size_t)Bp * sizeof(unsigned long long));
  a.error = ctx->error.as<int>();
  a.mels_T = ctx->mels_T.as<float>();
  a.aux_T = ctx->aux_T.as<float>();
  a.B = B; a.Bp = Bp; a.S = S; a.T = T; a.hop = ua.hop; a.steps = ua.steps;
  copy_gen_fields(a, ua);
  a.prof = phase_counters(ctx, prof, g.ncta, st);
  MolIO io{};
  if (mol) {                    // the fc3 outputs of the last two steps, [2][Bp][32]
    io = *mol;
    ctx->grid_mol_par.ensure((size_t)2 * Bp * 32 * sizeof(float));
    io.par = ctx->grid_mol_par.as<float>();
  }
  const MolIO* iop = mol ? &io : nullptr;
  switch (variant) {
    case GV_N4: launch_grid_t<0, 4, 1>(ctx, a, iop, st); break;
    case GV_W1: launch_grid_t<1, 1, 1>(ctx, a, iop, st); break;
    case GV_W2: launch_grid_t<2, 1, 1>(ctx, a, iop, st); break;
    case GV_W4: launch_grid_t<4, 1, 1>(ctx, a, iop, st); break;
    case GV_W4x2: launch_grid_t<4, 1, 2>(ctx, a, iop, st); break;
    default: REQUIRE(false, B200TTS_EINVAL, "internal: unknown grid variant");
  }
}

// Conditioning tables [tab_rows][T+1][ncta][52] of the push and tensor-core kernels from the first `src_rows` utterances of the
// mels / frame-rate aux, into ctx->push_tab, which is sized to hold them; table rows past the utterances are zero.
static const float* launch_cond_table(b200tts_wavernn* ctx, const float* d_mel, const float* aux_frames, int src_rows, int tab_rows,
                                      int T, cudaStream_t st) {
  const b200tts_wavernn_cfg& c = ctx->cfg;
  constexpr int FT = 8;
  ctx->push_tab.ensure((size_t)tab_rows * (T + 1) * ctx->pm.ncta * kPushCondRows * sizeof(float));
  dim3 grid((T + 1 + FT - 1) / FT, tab_rows);
  size_t smem = (size_t)(c.feat_dims + c.res_out_dims) * FT * sizeof(float);
  push_cond_table_kernel<FT><<<grid, 256, smem, st>>>(ctx->pcw, d_mel, aux_frames, src_rows, T, ctx->push_tab.as<float>());
  B200_CUDA(cudaGetLastError());
  ctx->launches++;
  return ctx->push_tab.as<float>();
}

// ---- small-batch push kernel (wavernn_push.cuh) --------------------------------------------------------------------------
// rows of the push kernel variant: up to 8 rows run the 8-row variant (on the previous GPU a 4-row variant was slower, its
// 64 hot L2 lines being polled by 65 536 threads)
static inline int push_rows(int B) { return B <= 8 ? 8 : (B <= 16 ? 16 : kPushMaxRows); }

// What a push launch runs: a RAW or a MOL generate call, or a run of RAW generation sessions.
enum class PushFlavour { RAW, MOL, SESSION };

// The G-row push kernel of `f`, and the floats of shared memory it needs past the weight blob.
template <int G>
static const void* push_kernel(PushFlavour f, int hop, int NT, size_t* scratch_floats) {
  *scratch_floats = PushTraits<G>::scratch_floats(hop, NT);
  if (f == PushFlavour::MOL) return (const void*)wavernn_push_mol_kernel<G>;
  if (f == PushFlavour::SESSION) return (const void*)wavernn_push_session_kernel<G>;
  return (const void*)wavernn_push_kernel<G>;
}

// Launches the push kernel of `f` on `rows` rows, with `io` (MolIO or SessIO; the RAW kernel takes none) as its third argument.
// `a` comes with the fields of its flavour set; this arms the exchange buffers and sets the fields every push launch shares.
static void launch_push_kernel(b200tts_wavernn* ctx, PushFlavour f, int rows, PushArgs& a, void* io, bool prof, cudaStream_t st) {
  PushModel pm = ctx->pm;
  const int G = push_rows(rows);
  const size_t nvec = (size_t)kPushVecs * 2 * pm.ncta * G * 4, nbest = (size_t)pm.ncta * G;
  ctx->push_vec.ensure(nvec * sizeof(float));
  ctx->push_best.ensure(nbest * sizeof(unsigned long long));
  launch_push_init(ctx->push_vec.as<uint32_t>(), nvec, ctx->push_best.as<unsigned long long>(), nbest, nullptr, ctx->sm_count, st);
  ctx->launches++;
  a.wblob = ctx->push_blob.as<float>();
  a.vec = ctx->push_vec.as<float>();
  a.best = ctx->push_best.as<unsigned long long>();
  a.error = ctx->error.as<int>();
  a.fir = ctx->d_fir;
  a.NT = ctx->NT;
  a.hop = ctx->cfg.hop_length;
  a.prof = phase_counters(ctx, prof, pm.ncta, st);
  size_t scratch = 0;
  const void* kern = G == 8 ? push_kernel<8>(f, a.hop, a.NT, &scratch)
                   : G == 16 ? push_kernel<16>(f, a.hop, a.NT, &scratch) : push_kernel<32>(f, a.hop, a.NT, &scratch);
  void* args[] = {(void*)&pm, (void*)&a, io};
  const bool sess = f == PushFlavour::SESSION;
  launch_step(ctx, sess ? SK_SESSION : SK_PUSH, kern, sess ? "push session kernel" : "push kernel", pm.ncta, kPushThreads,
              ((size_t)pm.blob + scratch) * sizeof(float), args, prof, st);
}

// `fold` != null: rows are the folds of ONE source utterance of T0 frames (conditioning tables of utterance 0, row u
// starts at sample u * stride); otherwise row u is utterance u.
struct PackInfo {            // gen_opts.d_pack_*: kernel rows run queues of utterances
  const int* utt;
  const int* start;
  int rows, segs, steps, n_utt;
};
static void launch_push(b200tts_wavernn* ctx, const float* d_mel, const GenArgs& ua, const MolIO* mol, bool prof, cudaStream_t st,
                        const FoldGeom* fold, int T0, const PackInfo* pack) {
  const int rows = pack ? pack->rows : ua.B;
  const int T = fold ? T0 : ua.T;
  const int tab_rows = fold ? 1 : (pack ? pack->n_utt : push_rows(rows)), src_rows = fold ? 1 : (pack ? pack->n_utt : rows);
  PushArgs a{};
  a.tab = launch_cond_table(ctx, d_mel, ua.aux_frames, src_rows, tab_rows, T, st);
  a.B = pack ? pack->n_utt : rows; a.S = ua.S; a.T = T; a.steps = pack ? pack->steps : ua.steps;
  if (pack) { a.pack_utt = pack->utt; a.pack_start = pack->start; a.pack_segs = pack->segs; a.pack_rows = pack->rows; }
  a.row_stride = fold ? fold->stride : 0;
  a.S_src = T * ctx->cfg.hop_length;
  copy_gen_fields(a, ua);
  MolIO io = mol ? *mol : MolIO{};
  launch_push_kernel(ctx, mol ? PushFlavour::MOL : PushFlavour::RAW, rows, a, &io, prof, st);
}

// ---- tensor-core pipeline (wavernn_tc.cuh): plain batches of up to 256 rows ----------------------------------------------
// `sess` != null: a run of generation sessions (wavernn_tc_session_kernel), row u = session u of *sess, whose tables the
// sessions own; `ua` gives B = sessions and the lock-steps, `d_mel` is unused.
static void launch_tc(b200tts_wavernn* ctx, const float* d_mel, const GenArgs& ua, const TcSessIO* sess, bool prof, cudaStream_t st) {
  const int rows = ua.B, T = ua.T;
  const int ng = (rows + kTcRows - 1) / kTcRows;
  TcArgs a{};
  if (!sess) a.tab = launch_cond_table(ctx, d_mel, ua.aux_frames, rows, rows, T, st);
  ctx->tc_vec.ensure((size_t)TV_COUNT * ng * 2 * kTcVecBytes);
  ctx->tc_x1f.ensure((size_t)ng * 2 * kTcRows * 512 * sizeof(float));
  ctx->tc_win.ensure((size_t)ng * 2 * kTcWinCopies * kTcRows * 16 * sizeof(unsigned long long));
  ctx->tc_cond.ensure((size_t)32 * 2 * ng * kTcCondBlk * kTcCondSlot * sizeof(float));
  const size_t cnt_bytes = (size_t)ng * TCN_COUNT * 32 * sizeof(unsigned);
  ctx->tc_cnt.ensure(cnt_bytes);
  B200_CUDA(cudaMemsetAsync(ctx->tc_cnt.p, 0, cnt_bytes, st));
  a.wimg = ctx->tc_wimg.as<uint8_t>();
  a.prm = ctx->tc_prm.as<float>();
  a.vec = ctx->tc_vec.as<uint8_t>();
  a.x1f = ctx->tc_x1f.as<float>();
  a.winners = ctx->tc_win.as<unsigned long long>();
  a.cnt = ctx->tc_cnt.as<unsigned>();
  a.condg = ctx->tc_cond.as<float>();
  a.error = ctx->error.as<int>();
  a.fir = ctx->d_fir;
  a.NT = ctx->NT; a.B = rows; a.S = ua.S; a.T = T; a.hop = ctx->cfg.hop_length; a.steps = ua.steps; a.ng = ng; a.NC = ctx->NC;
  copy_gen_fields(a, ua);
  a.prof = phase_counters(ctx, prof, kTcCtas, st);
  void* args[] = {(void*)&a, (void*)sess};
  if (sess)
    launch_step(ctx, SK_TC_SESSION, (const void*)wavernn_tc_session_kernel, "tensor-core session kernel", kTcCtas, kTcThreads,
                kTcSmemBytes, args, prof, st);
  else
    launch_step(ctx, SK_TC, (const void*)wavernn_tc_kernel, "tensor-core kernel", kTcCtas, kTcThreads, kTcSmemBytes, args, prof, st);
}

// Smallest batch kernel=auto gives the tensor cores.  On an H100 80GB HBM3 at a 400 W power limit the tensor-core pipeline costs
// 38-41 us per lock-step whatever the row count (1 or 2 groups of 128 rows in flight; 64-69 us while its wgmma were serialized);
// the wide CUDA-core mapping took 37.5 us at 64 rows, 60.9 at 96-128 and 90-91 from 129 rows on (a second tile of 128; 700 W).
constexpr int kTcMinRows = 129;

// The step kernel for `rows` kernel rows (folds when folding) under `o`, or a refusal.  Every capability it reads is fixed at
// create time, so a refused call has launched nothing.
static StepKernel choose_kernel(b200tts_wavernn* ctx, int rows, const b200tts_gen_opts& o) {
  const bool packing = o.d_pack_utt != nullptr;
  if (ctx->mol)                 // never on the tensor cores: MOL takes the push kernel up to 32 rows and the wide grid above
    REQUIRE(o.kernel != B200TTS_KERNEL_TC, B200TTS_EINVAL,
            "kernel=tc is RAW only: a MOL model runs on kernel=auto (push / wide grid), grid or utterance");
  // tc_ok implies pm.ok implies gm.ok (pack_tc_images, pack_push_model)
  const bool tc = ctx->tc_ok && o.fold_target == 0 && !packing && rows <= kTcRows * kTcMaxGroups;
  const bool push = ctx->pm.ok && (packing ? o.pack_rows : rows) <= kPushMaxRows;
  int kernel = o.kernel;
  if (kernel == B200TTS_KERNEL_AUTO) {
    if (tc && rows >= kTcMinRows) return SK_TC;       // fold mode and packed rows stay on the other kernels
    if (!ctx->gm.ok && !ctx->warned_fallback) {      // never silently: this path is ~4x slower
      ctx->warned_fallback = true;
      fprintf(stderr, "libb200tts: these hparams / this device cannot run the weight-stationary grid kernel; kernel=auto falls "
                      "back to the L2-streaming utterance kernel (about 4x slower at large batch)\n");
    }
    kernel = ctx->gm.ok ? B200TTS_KERNEL_GRID : B200TTS_KERNEL_UTTERANCE;
  }
  switch (kernel) {
    case B200TTS_KERNEL_TC:
      REQUIRE(tc, B200TTS_EINVAL, "kernel=tc needs rnn_dims = fc_dims = 512, 10-bit classes, hop_length x FIR taps <= 8192, "
                                  ">= 128 SMs, 1..256 rows, no folding / packing");
      return SK_TC;
    case B200TTS_KERNEL_GRID:
      if (push) return SK_PUSH;
      break;
    case B200TTS_KERNEL_UTTERANCE: break;
    default: throw Error(B200TTS_EINVAL, "unknown kernel selector");
  }
  REQUIRE(!packing, B200TTS_EINVAL, "packed generation needs the push kernel (kernel=auto/grid, rnn_dims = fc_dims = 512)");
  if (kernel == B200TTS_KERNEL_UTTERANCE) {
    REQUIRE(utt_fits(ctx->sw, 1), B200TTS_EINVAL,
            "model too large for the utterance kernel's shared memory (one row of its activations and logits exceeds 227 KB)");
    return SK_UTTERANCE;
  }
  REQUIRE(ctx->gm.ok, B200TTS_EINVAL, "kernel=grid was requested but this model/device cannot run the weight-stationary grid kernel "
                                      "(needs rnn_dims == fc_dims, n_classes == 2*rnn_dims, cooperative launch, R/4 <= SM count)");
  return SK_GRID;
}

// RAW contexts write labels to d_labels; MOL contexts write float samples to d_samples and take d_teacher_x.
static void run_generate_rows(b200tts_wavernn* ctx, const float* d_mel, int B, int T, const b200tts_rng& r,
                              const b200tts_gen_opts& o, bool prof, int16_t* d_labels, double* d_wave, float* d_samples,
                              const float* d_teacher_x, cudaStream_t st) {
  const b200tts_wavernn_cfg& c = ctx->cfg;
  const int hop = c.hop_length, S = T * hop, O = c.res_out_dims;
  if (ctx->mol) {
    REQUIRE(r.mode == B200TTS_RNG_PHILOX || r.mode == B200TTS_RNG_EXT_UNIFORM, B200TTS_EINVAL,
            "MOL generation takes PHILOX or EXT_UNIFORM noise");
    REQUIRE(r.mode != B200TTS_RNG_EXT_UNIFORM || r.d_q, B200TTS_EINVAL, "EXT_UNIFORM needs d_q");
    REQUIRE(!o.d_teacher, B200TTS_EINVAL, "MOL generation is teacher-forced through d_teacher_x (float samples), not d_teacher");
    REQUIRE(!o.d_pack_utt, B200TTS_EINVAL, "packed rows are not built for MOL models: generate the utterances in plain batches");
  } else {
    REQUIRE(r.mode == B200TTS_RNG_PHILOX || r.mode == B200TTS_RNG_EXT_EXPONENTIAL, B200TTS_EINVAL, "unknown rng mode");
    REQUIRE(r.mode != B200TTS_RNG_EXT_EXPONENTIAL || r.d_q, B200TTS_EINVAL, "EXT_EXPONENTIAL needs d_q");
  }
  REQUIRE(o.max_steps >= 0 && o.max_steps <= S, B200TTS_EINVAL, "max_steps out of range");
  const int steps = o.max_steps ? o.max_steps : S;
  const int fade_len = 20 * hop;                      // fatchord_version.py:256
  const int wave_len = (T - 1) * hop;                 // :184
  if (d_wave) {
    REQUIRE(steps == S, B200TTS_EINVAL, "a wave needs all steps (max_steps must be 0)");
    REQUIRE(wave_len >= fade_len, B200TTS_EINVAL,
            "T must be >= 21 frames: the reference's 20-hop fade-out (fatchord_version.py:256-258) fails below that");
  }
  REQUIRE(o.fold_target >= 0, B200TTS_EINVAL, "fold target/overlap out of range (fold_target 0 turns folding off)");
  const bool folding = o.fold_target > 0;
  FoldGeom fg{};
  if (folding) {
    REQUIRE(B == 1, B200TTS_EINVAL, "fold-with-overlap generation takes exactly one utterance (the reference folds x[0] only)");
    REQUIRE(steps == S, B200TTS_EINVAL, "max_steps is not supported together with folding");
    REQUIRE(!r.d_utterance_ids, B200TTS_EINVAL, "d_utterance_ids cannot be combined with fold-with-overlap generation");
    fg = fold_geometry(S, o.fold_target, o.fold_overlap);
    REQUIRE(fg.nfold >= 1 && fg.nfold <= 65535, B200TTS_EINVAL, "fold count out of range");
  }
  const bool packing = o.d_pack_utt != nullptr;
  if (packing) {
    REQUIRE(!folding && o.d_pack_start && o.pack_rows >= 1 && o.pack_rows <= kPushMaxRows && o.pack_segs >= 1 && o.pack_steps >= 1, B200TTS_EINVAL,
            "bad packed-row schedule (pack_rows 1..32, pack_segs >= 1, pack_steps >= 1, not together with folding)");
    REQUIRE(o.max_steps == 0 && !o.d_logits && !o.d_teacher && r.mode == B200TTS_RNG_PHILOX && d_labels, B200TTS_EINVAL,
            "packed generation takes PHILOX noise, all steps, caller-owned labels and no debug buffers");
  }
  const int GB = folding ? fg.nfold : B;            // rows the generation kernels see
  const int GS = folding ? fg.L : S;                // steps per row
  const StepKernel kernel = choose_kernel(ctx, GB, o);
  ctx->aux_frames.ensure((size_t)B * T * O * sizeof(float));
  // the rows' output, RAW labels or MOL samples: the context's scratch when the caller passed no buffer
  int16_t* labels = d_labels;
  float* samples = d_samples;
  if (ctx->mol ? !samples : !labels) {
    ctx->labels.ensure((size_t)GB * GS * (ctx->mol ? sizeof(float) : sizeof(int16_t)));
    if (ctx->mol) samples = ctx->labels.as<float>();
    else labels = ctx->labels.as<int16_t>();
  }
  float* mels_up = nullptr;
  if (kernel == SK_UTTERANCE || (folding && kernel == SK_GRID)) {
    ctx->mels_up.ensure((size_t)B * S * c.feat_dims * sizeof(float));
    mels_up = ctx->mels_up.as<float>();
  }
  run_upsample(ctx, d_mel, B, T, mels_up, ctx->aux_frames.as<float>(), nullptr, st);

  GenArgs a{};
  a.mels_up = ctx->mels_up.as<float>();
  a.aux_frames = ctx->aux_frames.as<float>();
  a.B = GB; a.S = GS; a.T = folding ? GS : T; a.hop = folding ? 1 : hop; a.steps = folding ? GS : steps;
  a.rng_mode = r.mode; a.seed = r.seed; a.utt_offset = r.utterance_offset; a.q = r.d_q;
  a.utt_ids = reinterpret_cast<const unsigned long long*>(r.d_utterance_ids);
  a.teacher = o.d_teacher; a.logits_out = o.d_logits; a.labels = labels;

  const FoldGeom* fold = folding ? &fg : nullptr;
  const PackInfo pi{o.d_pack_utt, o.d_pack_start, o.pack_rows, o.pack_segs, o.pack_steps, B};
  const MolIO mol{d_teacher_x, samples};
  switch (kernel) {
    case SK_UTTERANCE: launch_utterance(ctx, a, ctx->mol ? &mol : nullptr, st, fold, S); break;
    case SK_GRID: launch_grid(ctx, d_mel, a, ctx->mol ? &mol : nullptr, prof, st, fold, S); break;
    case SK_PUSH: launch_push(ctx, d_mel, a, ctx->mol ? &mol : nullptr, prof, st, fold, T, packing ? &pi : nullptr); break;
    case SK_TC: launch_tc(ctx, d_mel, a, nullptr, prof, st); break;
  }
  if (d_wave) {
    const int* err = ctx->error.as<int>();
    if (folding) {
      const int blocks = (wave_len + 255) / 256;
      if (ctx->mol)
        xfade_unfold_mol_kernel<<<blocks, 256, 0, st>>>(samples, fg.nfold, fg.L, o.fold_target, o.fold_overlap, wave_len, fade_len,
                                                        err, d_wave);
      else
        xfade_unfold_kernel<<<blocks, 256, 0, st>>>(labels, fg.nfold, fg.L, o.fold_target, o.fold_overlap, wave_len, fade_len,
                                                    ctx->NC, o.mu_law, err, d_wave);
    } else {
      dim3 grid((wave_len + 255) / 256, B);
      if (ctx->mol)
        finish_wave_mol_kernel<<<grid, 256, 0, st>>>(samples, S, wave_len, fade_len, o.d_utt_frames, hop, err, d_wave);
      else
        finish_wave_kernel<<<grid, 256, 0, st>>>(labels, S, wave_len, fade_len, ctx->NC, o.mu_law, o.d_utt_frames, hop, err, d_wave);
    }
    B200_CUDA(cudaGetLastError());
    ctx->launches++;
  }
}

// The wide mapping streams a sample-rate mel buffer [S][feat][Bp] (1.8 GB at 256 rows x 80 frames, 22.5 GB at 256 x 1000): long
// utterances x large batches would run out of memory before anything else.  Such a call is cut into row ranges whose buffers stay
// under a budget (default 8 GB, env B200TTS_MAX_COND_BYTES); the noise is keyed by the global row, so the result is unchanged.
// (Not for the debug modes whose buffers are indexed [step][row]: external noise, logits.)
static void run_generate(b200tts_wavernn* ctx, const float* d_mel, int B, int T, const b200tts_rng* rng,
                         const b200tts_gen_opts* opts, int16_t* d_labels, double* d_wave, float* d_samples,
                         const float* d_teacher_x, cudaStream_t st) {
  b200tts_rng r{};
  if (rng) r = *rng;
  b200tts_gen_opts o{};
  if (opts) o = *opts;
  else o.mu_law = 1;
  const bool prof = getenv("B200TTS_GRID_PROF") != nullptr;
  B200_CUDA(cudaMemsetAsync(ctx->error.p, 0, sizeof(int), st));    // one error word for every slice of the call
  const double budget = getenv("B200TTS_MAX_COND_BYTES") ? atof(getenv("B200TTS_MAX_COND_BYTES")) : 8e9;   // read per call
  const b200tts_wavernn_cfg& c = ctx->cfg;
  const double per_row = (double)T * c.hop_length * c.feat_dims * sizeof(float);
  const bool whole = r.mode == B200TTS_RNG_EXT_EXPONENTIAL || r.mode == B200TTS_RNG_EXT_UNIFORM || o.d_logits || o.fold_target > 0 ||
                     o.d_pack_utt || !(d_labels || d_samples);
  // kernel=auto and more than 256 rows: launches of 256 rows through the tensor-core pipeline (66 us per lock-step each on an H100)
  // beat the wide mapping on the whole batch (91 us per 256 rows); the noise is keyed by the global row, so the result does not change
  constexpr int kTcSlice = kTcRows * kTcMaxGroups;
  const bool tc_slices = !whole && B > kTcSlice && o.kernel == B200TTS_KERNEL_AUTO && choose_kernel(ctx, kTcSlice, o) == SK_TC;
  if (whole || (!tc_slices && per_row * ((B + 255) / 256 * 256) <= budget)) {
    run_generate_rows(ctx, d_mel, B, T, r, o, prof, d_labels, d_wave, d_samples, d_teacher_x, st);
    return;
  }
  int rows = tc_slices ? kTcSlice : (int)(budget / per_row);
  if (!tc_slices) rows = rows >= 256 ? rows / 256 * 256 : (rows >= 32 ? 32 : std::max(rows, 1));
  const size_t S = (size_t)T * c.hop_length, wave_len = (size_t)(T - 1) * c.hop_length;
  for (int r0 = 0; r0 < B; r0 += rows) {
    const int nb = std::min(rows, B - r0);
    b200tts_rng rs = r;
    if (rs.d_utterance_ids) rs.d_utterance_ids += r0;
    else rs.utterance_offset += (uint64_t)r0;
    b200tts_gen_opts os = o;
    if (os.d_teacher) os.d_teacher += (size_t)r0 * S;
    if (os.d_utt_frames) os.d_utt_frames += r0;
    run_generate_rows(ctx, d_mel + (size_t)r0 * c.feat_dims * T, nb, T, rs, os, prof, d_labels ? d_labels + (size_t)r0 * S : nullptr,
                      d_wave ? d_wave + (size_t)r0 * wave_len : nullptr, d_samples ? d_samples + (size_t)r0 * S : nullptr,
                      d_teacher_x ? d_teacher_x + (size_t)r0 * S : nullptr, st);
  }
}

extern "C" int b200tts_wavernn_fold_geometry(int T, int hop, int target, int overlap, int* n_folds, int* fold_len) {
  API_BEGIN
  REQUIRE(T >= 1 && hop >= 1 && n_folds && fold_len, B200TTS_EINVAL, "bad argument");
  FoldGeom g = fold_geometry((long long)T * hop, target, overlap);
  *n_folds = g.nfold;
  *fold_len = g.L;
  API_END
}

extern "C" int b200tts_wavernn_generate(b200tts_wavernn* ctx, const float* d_mel, int B, int T, const b200tts_rng* rng,
                                        const b200tts_gen_opts* opts, int16_t* d_labels, double* d_wave, void* stream) {
  API_BEGIN
  REQUIRE(ctx && d_mel, B200TTS_EINVAL, "null argument");
  REQUIRE(B >= 1 && T >= 1 && B <= 65535, B200TTS_EINVAL, "B must be 1..65535 and T positive");
  REQUIRE(!ctx->mol, B200TTS_EINVAL, "this context holds a MOL model: generate with b200tts_wavernn_generate_mol");
  DeviceGuard dg(ctx->device);
  run_generate(ctx, d_mel, B, T, rng, opts, d_labels, d_wave, nullptr, nullptr, (cudaStream_t)stream);
  API_END
}

extern "C" int b200tts_wavernn_generate_mol(b200tts_wavernn* ctx, const float* d_mel, int B, int T, const b200tts_rng* rng,
                                            const b200tts_gen_opts* opts, const float* d_teacher_x, float* d_samples,
                                            double* d_wave, void* stream) {
  API_BEGIN
  REQUIRE(ctx && d_mel, B200TTS_EINVAL, "null argument");
  REQUIRE(B >= 1 && T >= 1 && B <= 65535, B200TTS_EINVAL, "B must be 1..65535 and T positive");
  REQUIRE(ctx->mol, B200TTS_EINVAL, "this context holds a RAW model: generate with b200tts_wavernn_generate");
  DeviceGuard dg(ctx->device);
  run_generate(ctx, d_mel, B, T, rng, opts, nullptr, d_wave, d_samples, d_teacher_x, (cudaStream_t)stream);
  API_END
}

extern "C" int b200tts_wavernn_generate_host(b200tts_wavernn* ctx, const float* h_mel, int B, int T, const b200tts_rng* rng,
                                             const b200tts_gen_opts* opts, int16_t* h_labels, double* h_wave) {
  API_BEGIN
  REQUIRE(ctx && h_mel, B200TTS_EINVAL, "null argument");
  REQUIRE(B >= 1 && T >= 1 && B <= 65535, B200TTS_EINVAL, "B must be 1..65535 and T positive");
  REQUIRE(!ctx->mol, B200TTS_EINVAL, "the host entry point is RAW only: generate a MOL model with b200tts_wavernn_generate_mol");
  REQUIRE(!opts || (!opts->d_teacher && !opts->d_logits), B200TTS_EINVAL, "device-side debug buffers need the device entry point");
  REQUIRE(!rng || rng->mode == B200TTS_RNG_PHILOX, B200TTS_EINVAL, "the host entry point only takes the PHILOX mode");
  REQUIRE(!opts || opts->fold_target == 0 || !h_labels, B200TTS_EINVAL, "folded generation returns only the wave through the host entry point");
  DeviceGuard dg(ctx->device);
  const b200tts_wavernn_cfg& c = ctx->cfg;
  const size_t S = (size_t)T * c.hop_length, wave_len = (size_t)(T - 1) * c.hop_length;
  const size_t mel_bytes = (size_t)B * c.feat_dims * T * sizeof(float);
  const size_t lab_bytes = (size_t)B * S * sizeof(int16_t), wav_bytes = (size_t)B * wave_len * sizeof(double);
  cudaStream_t st = nullptr;   // legacy default stream: ordered with everything else the caller enqueued
  ctx->mel_in.ensure(mel_bytes);
  ctx->h_stage.ensure(std::max(mel_bytes, std::max(lab_bytes, wav_bytes)));
  std::memcpy(ctx->h_stage.p, h_mel, mel_bytes);
  B200_CUDA(cudaMemcpyAsync(ctx->mel_in.p, ctx->h_stage.p, mel_bytes, cudaMemcpyHostToDevice, st));
  ctx->labels.ensure(lab_bytes);
  double* d_wave = nullptr;
  if (h_wave) {
    ctx->wave.ensure(wav_bytes);
    d_wave = ctx->wave.as<double>();
  }
  run_generate(ctx, ctx->mel_in.as<float>(), B, T, rng, opts, ctx->labels.as<int16_t>(), d_wave, nullptr, nullptr, st);
  if (h_labels) {
    B200_CUDA(cudaMemcpyAsync(ctx->h_stage.p, ctx->labels.p, lab_bytes, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    std::memcpy(h_labels, ctx->h_stage.p, lab_bytes);
  }
  if (h_wave) {
    B200_CUDA(cudaMemcpyAsync(ctx->h_stage.p, ctx->wave.p, wav_bytes, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    std::memcpy(h_wave, ctx->h_stage.p, wav_bytes);
  }
  B200_CUDA(cudaStreamSynchronize(st));
  check_call_error(ctx);
  API_END
}

extern "C" int b200tts_wavernn_check(b200tts_wavernn* ctx) {
  API_BEGIN
  REQUIRE(ctx, B200TTS_EINVAL, "null argument");
  DeviceGuard dg(ctx->device);
  B200_CUDA(cudaDeviceSynchronize());
  check_call_error(ctx);
  API_END
}

// Debug: per-phase cycle counters of the last step-kernel launch (needs env B200TTS_GRID_PROF=1 at generate time).
// Grid and push kernels: out[12] = mean over CTAs of {P0 compute, P0 barrier, P1 compute, P1 barrier, ...} in SM cycles.
// Tensor-core pipeline: out[3 j + p] = cycles summed over the run of job j (GRU-2's W_ih2 . x1, fc1, fc2, fc3), phase p (exchange
// wait, GEMM, epilogue), averaged over the CTAs of that role.
extern "C" int b200tts_wavernn_debug_phase_cycles(b200tts_wavernn* ctx, double* out12) {
  API_BEGIN
  REQUIRE(ctx && out12, B200TTS_EINVAL, "null argument");
  REQUIRE(ctx->prof_ncta > 0, B200TTS_EINVAL, "no phase profile recorded");
  DeviceGuard dg(ctx->device);
  const int n = ctx->prof_ncta;
  std::vector<long long> h((size_t)n * 12);
  B200_CUDA(cudaDeviceSynchronize());
  B200_CUDA(cudaMemcpy(h.data(), ctx->prof.p, h.size() * sizeof(long long), cudaMemcpyDeviceToHost));
  if (ctx->last_kernel == SK_TC) {
    int cnt[4] = {0, 0, 0, 0};
    for (int i = 0; i < 12; ++i) out12[i] = 0;
    for (int cta = 0; cta < n; ++cta) {
      const int j = tc_role(cta).role - 1;
      if (j < 0) continue;
      ++cnt[j];
      for (int p = 0; p < 3; ++p) out12[3 * j + p] += (double)h[(size_t)cta * 12 + 3 * j + p];
    }
    for (int i = 0; i < 12; ++i) out12[i] /= cnt[i / 3];
    return B200TTS_OK;
  }
  for (int i = 0; i < 12; ++i) {
    double s = 0;
    for (int c = 0; c < n; ++c) s += (double)h[(size_t)c * 12 + i];
    out12[i] = s / n;
  }
  API_END
}

// ---- generation sessions: one RAW utterance in pieces on the push kernel (wavernn_push_session_kernel) or the tensor cores
//      (wavernn_tc_session_kernel) ---------------------------------------------------------------------------------------------
// Every refusal below comes before the first CUDA call, so a refused call has launched and allocated nothing.
static void require_session_model(const b200tts_wavernn* ctx) {
  REQUIRE(!ctx->mol, B200TTS_EINVAL, "generation sessions are RAW only: this context holds a MOL model");
  REQUIRE(ctx->pm.ok, B200TTS_EINVAL, "generation sessions need the push kernel (rnn_dims = fc_dims = 512 on >= 128 SMs)");
}

// The kernel and noise of a session open: kernel = AUTO (the push kernel) or TC where kernel=tc runs, and PHILOX noise (refused
// with the message `noise`).  Returns whether the sessions run on the tensor cores.
static bool require_session_kernel(const b200tts_wavernn* ctx, int kernel, const b200tts_rng& rng, const char* noise) {
  REQUIRE(kernel == B200TTS_KERNEL_AUTO || kernel == B200TTS_KERNEL_TC, B200TTS_EINVAL,
          "a session runs on kernel = AUTO (the push kernel) or TC (the tensor cores)");
  const bool tc = kernel == B200TTS_KERNEL_TC;
  REQUIRE(!tc || ctx->tc_ok, B200TTS_EINVAL, "tensor-core sessions need a model and device that run kernel=tc (rnn_dims = fc_dims = "
                                             "512, 10-bit classes, hop_length x FIR taps <= 8192, >= 128 SMs)");
  REQUIRE(rng.mode == B200TTS_RNG_PHILOX, B200TTS_EINVAL, noise);
  return tc;
}

// The most sessions one run takes on ctx: a tensor-core run where that kernel runs, else a push run.
extern "C" int b200tts_wavernn_session_max_rows(const b200tts_wavernn* ctx) {
  return ctx && ctx->tc_ok ? kTcSessRows : kPushMaxRows;
}

extern "C" int b200tts_wavernn_session_open(b200tts_wavernn* ctx, const float* d_mel, int T, const b200tts_rng* rng, int mu_law,
                                            b200tts_wavernn_session** out, void* stream) {
  return b200tts_wavernn_session_open_kernel(ctx, d_mel, T, rng, mu_law, B200TTS_KERNEL_AUTO, out, stream);
}

// The rows of a session open from its mels' frame counts h_frames[n] (host): session i takes T = max(frames, 21) frames, zero-padded
// to the 21 frames the 20-hop fade-out needs, as StreamingVocoder pads.  Their tables are placed by open_sessions.
static OpenRows open_rows(const b200tts_wavernn* ctx, const int32_t* h_frames, int n, int T_max) {
  const int hop = ctx->cfg.hop_length, FEAT = ctx->cfg.feat_dims, O = ctx->cfg.res_out_dims;
  OpenRows R{};
  R.n = n;
  for (int i = 0; i < n; ++i) {
    REQUIRE(h_frames[i] >= 1 && h_frames[i] <= T_max, B200TTS_EINVAL, "every row needs 1..T_max frames");
    const int T = std::max(h_frames[i], 21);
    REQUIRE((long long)T * hop <= INT_MAX, B200TTS_EINVAL, "utterance longer than 2^31 - 1 samples");
    R.frames[i] = h_frames[i];
    R.T[i] = T;
    REQUIRE((long long)R.f0[i] + T <= INT_MAX / std::max(FEAT, O), B200TTS_EINVAL, "mels too long for one batch");
    R.f0[i + 1] = R.f0[i] + T;
    R.res0[i + 1] = R.res0[i] + (T + kOpenFT - 1) / kOpenFT;
    R.tab0[i + 1] = R.tab0[i] + (T + 1 + kOpenFT - 1) / kOpenFT;
  }
  return R;
}

// Opens the sessions of rows R (open_rows) from d_mel (`layout`, rows of T_max frames) in three launches (wavernn_open.cuh); session
// i takes the utterance id ids[i].  Their tables and states share one allocation, freed with the last of them: a cudaMalloc is
// most of a one-row open's time (DESIGN 3.11.1).  Checks nothing: its callers have.
static void open_sessions(b200tts_wavernn* ctx, const float* d_mel, int layout, float max_abs_value, OpenRows R, int T_max,
                          uint64_t seed, const uint64_t* ids, int mu_law, bool tc, b200tts_wavernn_session** out, cudaStream_t st) {
  const int n = R.n, hop = ctx->cfg.hop_length, FEAT = ctx->cfg.feat_dims, O = ctx->cfg.res_out_dims, ncta = ctx->pm.ncta;
  // the prepared mels and MelResNet's output go to the context's scratch, consumed in stream order by the table launch
  const int frames = R.f0[n];
  ctx->mel_in.ensure((size_t)frames * FEAT * sizeof(float));
  ctx->aux_frames.ensure((size_t)frames * O * sizeof(float));
  float* mel = ctx->mel_in.as<float>();
  float* aux = ctx->aux_frames.as<float>();
  session_mel_prep_kernel<<<dim3((unsigned)std::min((FEAT * 2048 + 255) / 256, 64), n), 256, 0, st>>>(
      d_mel, layout, T_max, FEAT, max_abs_value, R, mel);
  B200_CUDA(cudaGetLastError());
  const b200tts_wavernn_cfg& c = ctx->cfg;
  const int threads = ((std::max(c.compute_dims, 32) + 31) / 32) * 32;
  const size_t res_smem = ((size_t)c.feat_dims * (2 * c.pad + 1) * kOpenFT + 2 * (size_t)c.compute_dims * kOpenFT) * sizeof(float);
  if (res_smem > 48 * 1024)
    B200_CUDA(cudaFuncSetAttribute(melresnet_ragged_kernel<kOpenFT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)res_smem));
  melresnet_ragged_kernel<kOpenFT><<<R.res0[n], threads, res_smem, st>>>(ctx->rp, mel, R, aux);
  B200_CUDA(cudaGetLastError());
  ctx->launches += 2;
  // one allocation, made while those kernels run: the n tables, table i of T_i + 1 frames from frame f0[i] + i, then the n
  // states (each 256-byte aligned)
  const size_t tab_frame = (size_t)ncta * kPushCondRows, tab_floats = (size_t)(R.f0[n] + n) * tab_frame;
  const size_t state_floats = ((size_t)kSessStateFloats + 63) / 64 * 64;
  auto mem = std::make_shared<DeviceBuf>();
  mem->ensure((tab_floats + (size_t)n * state_floats) * sizeof(float));
  float* base = mem->as<float>();
  std::vector<std::unique_ptr<b200tts_wavernn_session>> ss(n);
  for (int i = 0; i < n; ++i) {
    ss[i].reset(new b200tts_wavernn_session());
    b200tts_wavernn_session& s = *ss[i];
    s.ctx = ctx;
    s.tc = tc;
    s.T = R.T[i];
    s.mu_law = mu_law ? 1 : 0;
    s.S = (int64_t)R.T[i] * hop;
    s.wave_len = (int64_t)(R.T[i] - 1) * hop;
    s.seed = seed;
    s.id = ids[i];
    s.mem = mem;
    s.tab = R.tab[i] = base + (size_t)(R.f0[i] + i) * tab_frame;
    s.state = base + tab_floats + (size_t)i * state_floats;
  }
  const size_t tab_smem = (size_t)(FEAT + O) * kOpenFT * sizeof(float);
  push_cond_table_ragged_kernel<kOpenFT><<<R.tab0[n], 256, tab_smem, st>>>(ctx->pcw, mel, aux, R);
  B200_CUDA(cudaGetLastError());
  ctx->launches++;
  for (int i = 0; i < n; ++i) {
    ctx->sessions.insert(ss[i].get());
    out[i] = ss[i].release();
  }
}

// A one-row batched open of the mel as it is (T >= 21 frames need no padding), with open_rows refusing one too long.
extern "C" int b200tts_wavernn_session_open_kernel(b200tts_wavernn* ctx, const float* d_mel, int T, const b200tts_rng* rng,
                                                   int mu_law, int kernel, b200tts_wavernn_session** out, void* stream) {
  API_BEGIN
  REQUIRE(ctx && d_mel && rng && out, B200TTS_EINVAL, "null argument");
  *out = nullptr;
  require_session_model(ctx);
  const char* noise = "a session takes PHILOX noise keyed by (seed, rng->utterance_offset as the utterance id); d_utterance_ids "
                      "must be NULL";
  const bool tc = require_session_kernel(ctx, kernel, *rng, noise);
  REQUIRE(!rng->d_utterance_ids, B200TTS_EINVAL, noise);
  REQUIRE(T >= 21, B200TTS_EINVAL, "T must be >= 21 frames: the reference's 20-hop fade-out (fatchord_version.py:256-258) fails below that");
  const OpenRows R = open_rows(ctx, &T, 1, T);
  DeviceGuard dg(ctx->device);
  open_sessions(ctx, d_mel, B200TTS_MEL_FEAT_T, 0.f, R, T, rng->seed, &rng->utterance_offset, mu_law, tc, out, (cudaStream_t)stream);
  API_END
}

extern "C" int b200tts_wavernn_session_open_batch(b200tts_wavernn* ctx, const float* d_mel, int layout, float max_abs_value,
                                                  const int32_t* h_frames, int n, int T_max, const b200tts_rng* rng, int mu_law,
                                                  int kernel, b200tts_wavernn_session** out, void* stream) {
  API_BEGIN
  REQUIRE(ctx && d_mel && h_frames && rng && out, B200TTS_EINVAL, "null argument");
  require_session_model(ctx);
  const bool tc = require_session_kernel(
      ctx, kernel, *rng, "sessions take PHILOX noise keyed by (seed, utterance id: d_utterance_ids[i], or utterance_offset + i)");
  REQUIRE(layout == B200TTS_MEL_FEAT_T || layout == B200TTS_MEL_TACO, B200TTS_EINVAL,
          "unknown mel layout (B200TTS_MEL_FEAT_T or B200TTS_MEL_TACO)");
  REQUIRE(layout != B200TTS_MEL_TACO || (std::isfinite(max_abs_value) && max_abs_value > 0.f), B200TTS_EINVAL,
          "max_abs_value must be positive and finite");
  REQUIRE(n >= 1 && n <= b200tts_wavernn_session_max_rows(ctx), B200TTS_EINVAL, "n must be 1..session_max_rows");
  REQUIRE(T_max >= 1, B200TTS_EINVAL, "T_max must be >= 1");
  const OpenRows R = open_rows(ctx, h_frames, n, T_max);
  DeviceGuard dg(ctx->device);
  const cudaStream_t st = (cudaStream_t)stream;
  std::vector<uint64_t> ids(n);
  if (rng->d_utterance_ids) {       // the run kernels take each session's id as a parameter: read them back, in stream order
    B200_CUDA(cudaMemcpyAsync(ids.data(), rng->d_utterance_ids, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
  } else {
    for (int i = 0; i < n; ++i) ids[i] = rng->utterance_offset + (uint64_t)i;
  }
  open_sessions(ctx, d_mel, layout, max_abs_value, R, T_max, rng->seed, ids.data(), mu_law, tc, out, st);
  API_END
}

// cudaFree waits for the work queued on the device, so no run still in flight reads the memory freed here (a batch's memory is
// freed with the last of its sessions).
extern "C" void b200tts_wavernn_session_destroy(b200tts_wavernn_session* s) {
  if (!s) return;
  DeviceGuard dg(s->ctx->device, true);
  s->ctx->sessions.erase(s);
  delete s;
}

extern "C" int b200tts_wavernn_session_info(const b200tts_wavernn_session* s, int64_t* pos, int64_t* steps, int64_t* wave_len) {
  API_BEGIN
  REQUIRE(s, B200TTS_EINVAL, "null argument");
  if (pos) *pos = s->pos;
  if (steps) *steps = s->S;
  if (wave_len) *wave_len = s->wave_len;
  API_END
}

extern "C" int b200tts_wavernn_session_run(b200tts_wavernn* ctx, b200tts_wavernn_session* const* s, int n, int max_steps,
                                           int16_t* d_labels, double* d_wave, void* stream) {
  API_BEGIN
  REQUIRE(ctx && s, B200TTS_EINVAL, "null argument");
  require_session_model(ctx);
  // the first session says which kernel the run takes; every other must be on the same one
  const bool tc = n >= 1 && s[0] && s[0]->tc;
  if (tc) REQUIRE(n <= kTcSessRows, B200TTS_EINVAL, "a tensor-core session run takes 1..256 sessions");
  else REQUIRE(n >= 1 && n <= kPushMaxRows, B200TTS_EINVAL, "a session run takes 1..32 sessions");
  REQUIRE(max_steps >= 1, B200TTS_EINVAL, "max_steps must be >= 1");
  const int hop = ctx->cfg.hop_length;
  REQUIRE(!tc || max_steps % hop == 0, B200TTS_EINVAL,
          "a tensor-core session run takes max_steps a multiple of hop_length (every position stays on a frame boundary)");
  for (int i = 0; i < n; ++i) {
    REQUIRE(s[i], B200TTS_EINVAL, "null session");
    REQUIRE(s[i]->ctx == ctx, B200TTS_EINVAL, "the session belongs to another context");
    REQUIRE(s[i]->tc == tc, B200TTS_EINVAL, "a session run cannot mix push and tensor-core sessions");
    for (int j = 0; j < i; ++j) REQUIRE(s[j] != s[i], B200TTS_EINVAL, "the same session appears twice in one run");
  }
  DeviceGuard dg(ctx->device);
  const cudaStream_t st = (cudaStream_t)stream;
  // the rows of either kernel: TcSessIO holds 256 SessRow, of which a push run passes the first 32 as its SessIO
  TcSessIO io{};
  int steps = 0;
  for (int i = 0; i < n; ++i) {
    SessRow& r = io.row[i];
    r.tab = s[i]->tab;
    r.state = s[i]->state;
    r.seed = s[i]->seed;
    r.id = s[i]->id;
    r.T = s[i]->T;
    r.pos = (int)s[i]->pos;
    r.n = (int)std::min<int64_t>(max_steps, s[i]->S - s[i]->pos);
    r.mu_law = s[i]->mu_law;
    steps = std::max(steps, r.n);
  }
  io.ld = max_steps;
  io.labels = d_labels;
  if (!io.labels) {
    ctx->sess_labels.ensure((size_t)n * max_steps * sizeof(int16_t));
    io.labels = ctx->sess_labels.as<int16_t>();
  }
  B200_CUDA(cudaMemsetAsync(ctx->error.p, 0, sizeof(int), st));     // b200tts_wavernn_check reports this run
  if (steps > 0 && tc) {
    GenArgs a{};
    a.B = n; a.steps = steps; a.hop = hop;
    a.rng_mode = B200TTS_RNG_PHILOX;
    launch_tc(ctx, nullptr, a, &io, false, st);
  } else if (steps > 0) {
    PushArgs a{};
    a.B = n; a.steps = steps;
    a.rng_mode = B200TTS_RNG_PHILOX;
    SessIO pio{};
    std::copy(io.row, io.row + n, pio.row);
    pio.labels = io.labels;
    pio.ld = io.ld;
    launch_push_kernel(ctx, PushFlavour::SESSION, n, a, &pio, false, st);
  }
  // the wave: session_wave_kernel takes 32 sessions per launch
  for (int i0 = 0; d_wave && i0 < n; i0 += kPushMaxRows) {
    const int m = std::min(n - i0, kPushMaxRows);
    SessIO wio{};
    std::copy(io.row + i0, io.row + i0 + m, wio.row);
    wio.labels = io.labels + (size_t)i0 * max_steps;
    wio.ld = max_steps;
    dim3 grid((max_steps + 255) / 256, m);
    session_wave_kernel<<<grid, 256, 0, st>>>(wio, hop, 20 * hop, ctx->NC, ctx->error.as<int>(), d_wave + (size_t)i0 * max_steps);
    B200_CUDA(cudaGetLastError());
    ctx->launches++;
  }
  for (int i = 0; i < n; ++i) s[i]->pos += io.row[i].n;     // at enqueue: the counts are known without a synchronisation
  API_END
}

// ---- PHILOX noise dump ------------------------------------------------------------------------------
__global__ void philox_dump_kernel(unsigned long long seed, unsigned long long utt0, int B, int step0, int n_steps, int NC,
                                   float* __restrict__ q) {
  size_t total = (size_t)n_steps * B * (NC / 4);
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    int c4 = (int)(e % (NC / 4));
    size_t sb = e / (NC / 4);
    int b = (int)(sb % B), s = (int)(sb / B);
    float v[4];
    philox_exp4(seed, utt0 + (unsigned long long)b, (uint32_t)(step0 + s), (uint32_t)c4, v);
    *reinterpret_cast<float4*>(q + sb * NC + (size_t)c4 * 4) = make_float4(v[0], v[1], v[2], v[3]);
  }
}

extern "C" int b200tts_philox_exponential(int device, uint64_t seed, uint64_t utterance_offset, int B, int step0, int n_steps,
                                          int n_classes, float* d_q, void* stream) {
  API_BEGIN
  REQUIRE(d_q && B >= 1 && n_steps >= 1 && n_classes >= 4 && n_classes % 4 == 0 && step0 >= 0, B200TTS_EINVAL, "bad argument");
  REQUIRE(n_steps <= INT_MAX - step0, B200TTS_EINVAL, "step0 + n_steps must not exceed 2^31 - 1");
  DeviceGuard dg(device);
  size_t total = (size_t)n_steps * B * (n_classes / 4);
  unsigned grid = (unsigned)std::min<size_t>((total + 255) / 256, 132 * 16);
  philox_dump_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(seed, utterance_offset, B, step0, n_steps, n_classes, d_q);
  B200_CUDA(cudaGetLastError());
  API_END
}

__global__ void philox_mol_dump_kernel(unsigned long long seed, unsigned long long utt0, int B, int step0, int n_steps,
                                       float* __restrict__ u) {
  const size_t total = (size_t)n_steps * B;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const int b = (int)(e % B), s = (int)(e / B);
    float v[kMolU];
    philox_mol_u(seed, utt0 + (unsigned long long)b, (uint32_t)(step0 + s), v);
#pragma unroll
    for (int j = 0; j < kMolU; ++j) u[e * kMolU + j] = v[j];
  }
}

extern "C" int b200tts_philox_mol_uniform(int device, uint64_t seed, uint64_t utterance_offset, int B, int step0, int n_steps,
                                          float* d_u, void* stream) {
  API_BEGIN
  REQUIRE(d_u && B >= 1 && n_steps >= 1 && step0 >= 0, B200TTS_EINVAL, "bad argument");
  REQUIRE(n_steps <= INT_MAX - step0, B200TTS_EINVAL, "step0 + n_steps must not exceed 2^31 - 1");
  DeviceGuard dg(device);
  const size_t total = (size_t)n_steps * B;
  unsigned grid = (unsigned)std::min<size_t>((total + 255) / 256, 132 * 16);
  philox_mol_dump_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(seed, utterance_offset, B, step0, n_steps, d_u);
  B200_CUDA(cudaGetLastError());
  API_END
}
