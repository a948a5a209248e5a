// libb200tts.so -- Tacotron-2 encoder, decoder and postnet (taco_decoder.cuh, taco_encpost.cuh, taco_grid.cuh): b200tts_taco_*.
// The kernels of the decoder sessions are in taco_session.cu.
//
// In one module, the dynamic shared memory of every kernel starts at the largest alignment any extern __shared__ array of the
// module asks for.  The Tacotron kernels' code and shared-memory budgets were settled while they shared a module with
// wavernn_tc_kernel (1024 bytes), so their own `sm` arrays ask for 1024: compiled here, ptxas gives them the same code.
#include <algorithm>
#include <cmath>
#include <set>

#include "api.h"
#include "taco_decoder.cuh"
#include "taco_encpost.cuh"
#include "taco_grid.cuh"

using namespace b200tts;

struct TacoConvW {          // one conv1d + folded BatchNorm
  const float *K, *bias, *scale, *shift;
  int k, Cin, Cout;
};
// One free-running decode cut into slices (b200tts_taco_session_*): its memory and keys, the state record its last slice saved,
// and its frames and stop values so far.  Owned by its context, which frees the sessions still open.
struct b200tts_taco_session {
  b200tts_taco* ctx = nullptr;
  std::shared_ptr<DeviceBuf> batch;         // the open's one allocation, freed with the last of its sessions
  const float *memory = nullptr, *keys = nullptr;
  float *state = nullptr, *frames = nullptr, *stop = nullptr;
  uint64_t seed = 0, id = 0;
  float mu_bias = 0.f;
  int Tx = 0, max_steps = 0, window = 0;
  int pos = 0;                              // steps decoded
  bool done = false;                        // the stop token fired, or pos reached max_steps
};
struct b200tts_taco {
  int device = 0;
  b200tts_taco_cfg cfg{};
  DeviceBuf weights, keys, act_a, act_b;
  TacoWeights tw{};
  // run-once neighbours (present when the weight list carried them)
  bool has_encoder = false, has_postnet = false;
  const float* embedding = nullptr;
  int vocab = 0, emb_dim = 0, enc_units = 0;
  TacoConvW enc_conv[3]{}, post_conv[5]{};
  const float *enc_kfw = nullptr, *enc_bfw = nullptr, *enc_kbw = nullptr, *enc_bbw = nullptr;
  const float *post_pk = nullptr, *post_pb = nullptr;
  int post_channels = 0;
  // weight-stationary single-sentence decoder (taco_grid.cuh)
  TacoGridModel tgm{};
  DeviceBuf tg_blob, tg_vec;
  bool tg_ok = false;
  int sm_count = 0;
  DeviceBuf mu_bias;          // [B] speaking-rate biases of the last b200tts_taco_decode_biased call
  std::set<b200tts_taco_session*> sessions;   // open decoder sessions, freed with the context
  DeviceBuf sess_status;                      // [kTacoSessRows][2] status words of the last session run ...
  HostPinned h_sess_status;                   // ... and their host copy
  ~b200tts_taco() {
    for (b200tts_taco_session* s : sessions) delete s;
  }
};

// Split-K partials of taco_decoder_kernel, in floats.  The matvecs and the context sum need at most 4096 of them; the attention
// step keeps the location features f[Tx][NF] there, so b200tts_taco_create accepts only configs with kTacoMaxTx * NF <= this.
constexpr int kTacoPartFloats = 16384;

// dynamic shared memory of taco_decoder_kernel (its carve-up, plus the split-K partials)
static size_t taco_decoder_smem_bytes(const TacoWeights& w) {
  const size_t fl = 128 + w.P + (w.P + w.E + w.U) + 2 * w.U + 4 * w.U + 2 * w.U + (w.U + w.E) + w.A + 3 * kTacoMaxTx + 96 + 64 +
                    (size_t)w.KW * w.NF + (size_t)w.NF * w.A + kTacoPartFloats;
  return fl * sizeof(float);
}

// Where each decoder weight sits in the packed blob, in floats; bind(base) points the decoder at a copy of the blob at `base`.
struct TacoWeightOffsets {
  size_t pre1_k, pre1_b, pre2_k, pre2_b, l1_k, l1_b, l2_k, l2_b, q_k, loc_k, loc_b, locl_k, v_a, b_a, mu_k, mu_b, fr_k, fr_b, st_k,
      st_b, mem_k;
  TacoWeights bind(const float* b, const b200tts_taco_cfg& c) const {
    TacoWeights w{};
    w.pre1_k = b + pre1_k; w.pre1_b = b + pre1_b; w.pre2_k = b + pre2_k; w.pre2_b = b + pre2_b;
    w.l1_k = b + l1_k; w.l1_b = b + l1_b; w.l2_k = b + l2_k; w.l2_b = b + l2_b;
    w.q_k = b + q_k; w.loc_k = b + loc_k; w.loc_b = b + loc_b; w.locl_k = b + locl_k; w.v_a = b + v_a; w.b_a = b + b_a;
    w.mu_k = b + mu_k; w.mu_b = b + mu_b; w.fr_k = b + fr_k; w.fr_b = b + fr_b; w.st_k = b + st_k; w.st_b = b + st_b;
    w.mem_k = b + mem_k;
    w.mels = c.num_mels; w.P = c.prenet_units; w.U = c.lstm_units; w.E = c.enc_dim; w.A = c.attn_dim; w.NF = c.attn_filters;
    w.KW = c.attn_kernel; w.zoneout = c.zoneout;
    return w;
  }
};

extern "C" int b200tts_taco_create(b200tts_taco** out, int device, const b200tts_taco_cfg* cfg, const b200tts_tensor* weights,
                                   int n_weights) {
  API_BEGIN
  REQUIRE(out && cfg && weights && n_weights > 0, B200TTS_EINVAL, "null argument");
  *out = nullptr;
  const b200tts_taco_cfg& c = *cfg;
  const int M = c.num_mels, P = c.prenet_units, U = c.lstm_units, E = c.enc_dim, AD = c.attn_dim, NF = c.attn_filters, KW = c.attn_kernel;
  REQUIRE(M % 4 == 0 && P % 4 == 0 && U % 4 == 0 && E % 4 == 0 && AD % 4 == 0, B200TTS_EINVAL, "dims must be multiples of 4");
  REQUIRE(M <= 96 && P == 256 && 4 * U == 1024 && E <= 1024 && AD <= 256 && KW % 2 == 1 && KW * NF <= 992 && NF * AD <= 4096,
          B200TTS_EINVAL, "decoder dims outside what taco_decoder_kernel is laid out for");
  REQUIRE(kTacoMaxTx * NF <= kTacoPartFloats, B200TTS_EINVAL,
          "attn_filters: the location features of a 512-token sentence must fit taco_decoder_kernel's partial buffer (NF <= 32)");
  check_device(device);
  DeviceGuard dg(device);
  TensorMap tm;
  for (int i = 0; i < n_weights; ++i)
    if (weights[i].name) tm[weights[i].name] = &weights[i];
  std::unique_ptr<b200tts_taco> ctx(new b200tts_taco());
  ctx->device = device;
  ctx->cfg = c;
  Packer pk;
  const std::string D = "decoder/", L = D + "Location_Sensitive_Attention/";
  TacoWeightOffsets o{};
  o.pre1_k = pk.copy(tm, D + "decoder_prenet/dense_1/kernel", {M, P}); o.pre1_b = pk.copy(tm, D + "decoder_prenet/dense_1/bias", {P});
  o.pre2_k = pk.copy(tm, D + "decoder_prenet/dense_2/kernel", {P, P}); o.pre2_b = pk.copy(tm, D + "decoder_prenet/dense_2/bias", {P});
  o.l1_k = pk.copy(tm, D + "decoder_LSTM/multi_rnn_cell/cell_0/decoder_LSTM_1/kernel", {P + E + U, 4 * U});
  o.l1_b = pk.copy(tm, D + "decoder_LSTM/multi_rnn_cell/cell_0/decoder_LSTM_1/bias", {4 * U});
  o.l2_k = pk.copy(tm, D + "decoder_LSTM/multi_rnn_cell/cell_1/decoder_LSTM_2/kernel", {2 * U, 4 * U});
  o.l2_b = pk.copy(tm, D + "decoder_LSTM/multi_rnn_cell/cell_1/decoder_LSTM_2/bias", {4 * U});
  o.q_k = pk.copy(tm, L + "query_layer/kernel", {U, AD});
  o.loc_k = pk.copy(tm, L + "location_features_convolution/kernel", {KW, 1, NF});
  o.loc_b = pk.copy(tm, L + "location_features_convolution/bias", {NF});
  o.locl_k = pk.copy(tm, L + "location_features_layer/kernel", {NF, AD});
  o.v_a = pk.copy(tm, L + "attention_variable_projection", {AD}); o.b_a = pk.copy(tm, L + "attention_bias", {AD});
  o.mu_k = pk.copy(tm, D + "dense/kernel", {E + U, 1}); o.mu_b = pk.copy(tm, D + "dense/bias", {1});
  o.fr_k = pk.copy(tm, D + "linear_transform_projection/projection_linear_transform_projection/kernel", {U + E, M});
  o.fr_b = pk.copy(tm, D + "linear_transform_projection/projection_linear_transform_projection/bias", {M});
  o.st_k = pk.copy(tm, D + "stop_token_projection/projection_stop_token_projection/kernel", {U + E, 1});
  o.st_b = pk.copy(tm, D + "stop_token_projection/projection_stop_token_projection/bias", {1});
  o.mem_k = pk.copy(tm, "memory_layer/kernel", {E, AD});
  // ---- optional run-once neighbours: encoder and postnet ----
  struct ConvOff { size_t K, bias, scale, shift; int k, Cin, Cout; };
  auto pack_conv = [&](const std::string& scope) {
    auto it = tm.find(scope + "/conv1d/kernel");
    REQUIRE(it != tm.end() && it->second->ndim == 3, B200TTS_EMISSING, "missing weight tensor '" + scope + "/conv1d/kernel'");
    const b200tts_tensor* kt = it->second;
    ConvOff c{};
    c.k = (int)kt->shape[0]; c.Cin = (int)kt->shape[1]; c.Cout = (int)kt->shape[2];
    c.K = pk.copy(tm, scope + "/conv1d/kernel", {c.k, c.Cin, c.Cout});
    c.bias = pk.copy(tm, scope + "/conv1d/bias", {c.Cout});
    const float* g = need(tm, scope + "/batch_normalization/gamma", {c.Cout})->data;
    const float* be = need(tm, scope + "/batch_normalization/beta", {c.Cout})->data;
    const float* mu = need(tm, scope + "/batch_normalization/moving_mean", {c.Cout})->data;
    const float* var = need(tm, scope + "/batch_normalization/moving_variance", {c.Cout})->data;
    c.scale = pk.add(c.Cout); c.shift = pk.add(c.Cout);
    for (int i = 0; i < c.Cout; ++i) {                 // tf.layers.batch_normalization, moving stats, epsilon 1e-3
      double sc = (double)g[i] / std::sqrt((double)var[i] + 1e-3);
      pk.h[c.scale + i] = (float)sc;
      pk.h[c.shift + i] = (float)((double)be[i] - (double)mu[i] * sc);
    }
    return c;
  };
  ConvOff encc[3]{}, postc[5]{};
  size_t o_emb = 0, o_kfw = 0, o_bfw = 0, o_kbw = 0, o_bbw = 0, o_pk = 0, o_pb = 0;
  if (tm.count("inputs_embedding") && tm.count("encoder_convolutions/conv_layer_1_encoder_convolutions/conv1d/kernel")) {
    const b200tts_tensor* et = tm["inputs_embedding"];
    REQUIRE(et->ndim == 2, B200TTS_ESHAPE, "inputs_embedding must be 2-D");
    ctx->vocab = (int)et->shape[0]; ctx->emb_dim = (int)et->shape[1];
    o_emb = pk.copy(tm, "inputs_embedding", {ctx->vocab, ctx->emb_dim});
    for (int i = 0; i < 3; ++i) encc[i] = pack_conv("encoder_convolutions/conv_layer_" + std::to_string(i + 1) + "_encoder_convolutions");
    REQUIRE(encc[0].Cin == ctx->emb_dim && encc[2].Cout % 4 == 0 && E % 2 == 0, B200TTS_ESHAPE, "encoder conv shapes");
    const int EU = E / 2, CI = encc[2].Cout;
    REQUIRE(4 * EU == 1024, B200TTS_EINVAL, "encoder LSTM units must be 256");
    const std::string LS = "encoder_LSTM/bidirectional_rnn/";
    o_kfw = pk.copy(tm, LS + "fw/encoder_fw_LSTM/kernel", {CI + EU, 4 * EU}); o_bfw = pk.copy(tm, LS + "fw/encoder_fw_LSTM/bias", {4 * EU});
    o_kbw = pk.copy(tm, LS + "bw/encoder_bw_LSTM/kernel", {CI + EU, 4 * EU}); o_bbw = pk.copy(tm, LS + "bw/encoder_bw_LSTM/bias", {4 * EU});
    ctx->enc_units = EU;
    ctx->has_encoder = true;
  }
  if (tm.count("postnet_projection/projection_postnet_projection/kernel")) {
    for (int i = 0; i < 5; ++i) postc[i] = pack_conv("postnet_convolutions/conv_layer_" + std::to_string(i + 1) + "_postnet_convolutions");
    REQUIRE(postc[0].Cin == M, B200TTS_ESHAPE, "postnet conv 1 must take num_mels channels");
    ctx->post_channels = postc[4].Cout;
    o_pk = pk.copy(tm, "postnet_projection/projection_postnet_projection/kernel", {ctx->post_channels, M});
    o_pb = pk.copy(tm, "postnet_projection/projection_postnet_projection/bias", {M});
    ctx->has_postnet = true;
  }
  ctx->weights.ensure(pk.h.size() * sizeof(float));
  B200_CUDA(cudaMemcpy(ctx->weights.p, pk.h.data(), pk.h.size() * sizeof(float), cudaMemcpyHostToDevice));
  const float* b = ctx->weights.as<float>();
  ctx->tw = o.bind(b, c);
  auto bind = [&](const ConvOff& c0) { return TacoConvW{b + c0.K, b + c0.bias, b + c0.scale, b + c0.shift, c0.k, c0.Cin, c0.Cout}; };
  if (ctx->has_encoder) {
    ctx->embedding = b + o_emb;
    for (int i = 0; i < 3; ++i) ctx->enc_conv[i] = bind(encc[i]);
    ctx->enc_kfw = b + o_kfw; ctx->enc_bfw = b + o_bfw; ctx->enc_kbw = b + o_kbw; ctx->enc_bbw = b + o_bbw;
  }
  if (ctx->has_postnet) {
    for (int i = 0; i < 5; ++i) ctx->post_conv[i] = bind(postc[i]);
    ctx->post_pk = b + o_pk; ctx->post_pb = b + o_pb;
  }
  // ---- per-block weight blobs of the weight-stationary single-sentence decoder (taco_grid.cuh) ----
  int coop = 0;
  B200_CUDA(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, device));
  B200_CUDA(cudaDeviceGetAttribute(&ctx->sm_count, cudaDevAttrMultiProcessorCount, device));
  const std::vector<float> gb = pack_taco_grid_model(o.bind(pk.h.data(), c), ctx->sm_count, coop != 0, ctx->tgm);
  if (!gb.empty()) {
    ctx->tg_blob.ensure(gb.size() * sizeof(float));
    B200_CUDA(cudaMemcpy(ctx->tg_blob.p, gb.data(), gb.size() * sizeof(float), cudaMemcpyHostToDevice));
    ctx->tg_ok = true;
  }
  *out = ctx.release();
  API_END
}

extern "C" void b200tts_taco_destroy(b200tts_taco* ctx) {
  if (!ctx) return;
  DeviceGuard dg(ctx->device, true);
  delete ctx;
}

// Every bias finite and in [-1, 1] (h_mu_bias NULL: none).
static void require_mu_bias(const float* h_mu_bias, int B) {
  if (h_mu_bias)
    for (int b = 0; b < B; ++b)
      REQUIRE(std::isfinite(h_mu_bias[b]) && h_mu_bias[b] >= -1.f && h_mu_bias[b] <= 1.f, B200TTS_EINVAL,
              "mu_bias[" + std::to_string(b) + "] must be finite and in [-1, 1]");
}

static void require_dropout(const b200tts_taco_dropout& d) {
  REQUIRE(d.mode == B200TTS_TACO_DROPOUT_PHILOX || (d.mode == B200TTS_TACO_DROPOUT_EXT && d.d_masks), B200TTS_EINVAL,
          "bad dropout descriptor");
}

// keys[r][:] = memory[r][:] . W_memory for `rows` rows of the encoder output
static void launch_taco_keys(const TacoWeights& w, const float* memory, int rows, float* keys, cudaStream_t st) {
  taco_keys_kernel<<<rows, 128, w.E * sizeof(float), st>>>(memory, w.mem_k, rows, w.E, w.A, keys);
  B200_CUDA(cudaGetLastError());
}

enum class TacoDecoder { kBatch, kBatchBiased, kGta, kGrid, kGridBiased };

// Teacher-forced (GTA) decoding runs one thread block per sentence at every B: it is a batch job, so the single-sentence grid
// decoder is not taught the fed frame.  Otherwise a lone sentence runs on the grid decoder where the model and device allow it.
static TacoDecoder choose_taco_decoder(const b200tts_taco* ctx, int B, bool gta, bool biased) {
  if (gta) return TacoDecoder::kGta;
  if (B == 1 && ctx->tg_ok) return biased ? TacoDecoder::kGridBiased : TacoDecoder::kGrid;
  return biased ? TacoDecoder::kBatchBiased : TacoDecoder::kBatch;
}

// Every b200tts_taco_decode* call once its arguments have been checked: uploads the biases (h_mu_bias: [B] on the host, or
// NULL), computes the keys into `a` and runs the decoder choose_taco_decoder picks.  gta: the recorded mels of a GTA run, or NULL.
static void launch_taco_decoder(b200tts_taco* ctx, TacoArgs a, const TacoGtaArgs* gta, const float* h_mu_bias, cudaStream_t st) {
  DeviceGuard dg(ctx->device);
  const TacoWeights& w = ctx->tw;
  const float* d_mu_bias = nullptr;
  if (h_mu_bias) {
    ctx->mu_bias.ensure((size_t)a.B * sizeof(float));
    B200_CUDA(cudaMemcpyAsync(ctx->mu_bias.p, h_mu_bias, (size_t)a.B * sizeof(float), cudaMemcpyHostToDevice, st));
    d_mu_bias = ctx->mu_bias.as<float>();
  }
  ctx->keys.ensure((size_t)a.B * a.Tx_max * w.A * sizeof(float));
  a.keys = ctx->keys.as<float>();
  launch_taco_keys(w, a.memory, a.B * a.Tx_max, ctx->keys.as<float>(), st);
  const TacoDecoder k = choose_taco_decoder(ctx, a.B, gta != nullptr, h_mu_bias != nullptr);
  if (k == TacoDecoder::kGrid || k == TacoDecoder::kGridBiased) {
    // The sentence length is needed on the host to size the exchange buffers; a.lengths is a device pointer, so Tx_max (the
    // caller's padded length) bounds it and the kernel reads the true length itself.
    const int Txp = (a.Tx_max + 3) & ~3;
    const size_t copy = (size_t)2048 + (size_t)kTgCtas * Txp;
    ctx->tg_vec.ensure(2 * copy * sizeof(float) + 64);
    int* d_err = reinterpret_cast<int*>(ctx->tg_vec.as<float>() + 2 * copy);
    launch_push_init(ctx->tg_vec.as<uint32_t>(), 2 * copy, nullptr, 0, d_err, ctx->sm_count, st);
    TacoGridArgs ga{};
    ga.wblob = ctx->tg_blob.as<float>();
    ga.vec = ctx->tg_vec.as<float>();
    ga.error = d_err;
    ga.memory = a.memory; ga.keys = a.keys;
    ga.lengths = a.lengths;
    ga.Tx = a.Tx_max; ga.Txp = Txp; ga.max_steps = a.max_steps; ga.window = a.window;
    ga.rng_mode = a.rng_mode; ga.seed = a.seed; ga.utt = a.utt_offset; ga.masks = a.masks;
    ga.forced = a.forced; ga.Tx_alloc = a.Tx_max;
    ga.frames = a.frames; ga.stop = a.stop; ga.align = a.align; ga.nsteps = a.nsteps;
    const size_t smem = taco_grid_smem_bytes(ctx->tgm, Txp);
    REQUIRE(smem <= 227 * 1024, B200TTS_EINVAL, "taco_grid_kernel: shared memory budget exceeded");
    const void* kernel = k == TacoDecoder::kGridBiased ? (const void*)taco_grid_biased_kernel : (const void*)taco_grid_kernel;
    B200_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    TacoGridModel gm = ctx->tgm;
    void* args[] = {(void*)&gm, (void*)&ga, (void*)&d_mu_bias};
    B200_CUDA(cudaLaunchCooperativeKernel(kernel, dim3(kTgCtas), dim3(kTgThreads), args, smem, st));
    taco_grid_finish_kernel<<<1, 1, 0, st>>>(d_err, a.nsteps);
    B200_CUDA(cudaGetLastError());
    return;
  }
  // Named in this order, the instantiations of taco_decoder_kernel keep their places in the module, and with them the code ptxas
  // gives the grid kernels.
  const size_t smem = taco_decoder_smem_bytes(w);
  if (k == TacoDecoder::kBatchBiased) {
    B200_CUDA(cudaFuncSetAttribute(taco_decoder_biased_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    taco_decoder_biased_kernel<<<a.B, kTacoThreads, smem, st>>>(w, a, d_mu_bias);
  } else if (k == TacoDecoder::kBatch) {
    B200_CUDA(cudaFuncSetAttribute(taco_decoder_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    taco_decoder_kernel<false><<<a.B, kTacoThreads, smem, st>>>(w, a, TacoGtaArgs{});
  } else {
    B200_CUDA(cudaFuncSetAttribute(taco_decoder_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    taco_decoder_kernel<true><<<a.B, kTacoThreads, smem, st>>>(w, a, *gta);
  }
  B200_CUDA(cudaGetLastError());
}

// free, forced (d_forced: state records) or biased (h_mu_bias: [B] host speaking-rate biases) decoding
static int taco_decode_impl(b200tts_taco* ctx, const float* d_memory, const int32_t* d_lengths, int B, int Tx_max,
                            const b200tts_taco_dropout* dropout, int max_steps, int window, const float* h_mu_bias,
                            const float* d_forced, float* d_frames, float* d_stop, float* d_align, int32_t* d_nsteps, void* stream) {
  API_BEGIN
  REQUIRE(ctx && d_memory && d_lengths && d_frames && d_stop && d_nsteps, B200TTS_EINVAL, "null argument");
  REQUIRE(B >= 1 && Tx_max >= 1 && Tx_max <= kTacoMaxTx && max_steps >= 1, B200TTS_EINVAL, "B, Tx_max (<= 512), max_steps out of range");
  b200tts_taco_dropout d{};
  if (dropout) d = *dropout;
  require_dropout(d);
  require_mu_bias(h_mu_bias, B);
  TacoArgs a{};
  a.memory = d_memory; a.lengths = d_lengths;
  a.B = B; a.Tx_max = Tx_max; a.max_steps = max_steps; a.window = window;
  a.rng_mode = d.mode; a.seed = d.seed; a.utt_offset = d.utterance_offset; a.masks = d.d_masks;
  a.frames = d_frames; a.stop = d_stop; a.align = d_align; a.nsteps = d_nsteps; a.forced = d_forced;
  launch_taco_decoder(ctx, a, nullptr, h_mu_bias, (cudaStream_t)stream);
  API_END
}

extern "C" int b200tts_taco_decode(b200tts_taco* ctx, const float* d_memory, const int32_t* d_lengths, int B, int Tx_max,
                                   const b200tts_taco_dropout* dropout, int max_steps, int window, float* d_frames, float* d_stop,
                                   float* d_align, int32_t* d_nsteps, void* stream) {
  return taco_decode_impl(ctx, d_memory, d_lengths, B, Tx_max, dropout, max_steps, window, nullptr, nullptr, d_frames, d_stop, d_align,
                          d_nsteps, stream);
}

extern "C" int b200tts_taco_decode_biased(b200tts_taco* ctx, const float* d_memory, const int32_t* d_lengths, int B, int Tx_max,
                                          const b200tts_taco_dropout* dropout, int max_steps, int window, const float* h_mu_bias,
                                          const float* d_states, float* d_frames, float* d_stop, float* d_align, int32_t* d_nsteps,
                                          void* stream) {
  if (!h_mu_bias) {
    g_err = "b200tts_taco_decode_biased needs h_mu_bias";
    return B200TTS_EINVAL;
  }
  return taco_decode_impl(ctx, d_memory, d_lengths, B, Tx_max, dropout, max_steps, window, h_mu_bias, d_states, d_frames, d_stop,
                          d_align, d_nsteps, stream);
}

extern "C" int b200tts_taco_state_floats(const b200tts_taco* ctx, int Tx_max) {
  if (!ctx || Tx_max < 1) return B200TTS_EINVAL;
  return taco_state_floats(ctx->cfg.num_mels, ctx->cfg.enc_dim, ctx->cfg.lstm_units, Tx_max);
}

extern "C" int b200tts_taco_decode_forced(b200tts_taco* ctx, const float* d_memory, const int32_t* d_lengths, int B, int Tx_max,
                                          const b200tts_taco_dropout* dropout, int n_steps, int window, const float* d_states,
                                          float* d_frames, float* d_stop, float* d_align, int32_t* d_nsteps, void* stream) {
  if (!d_states) {
    g_err = "b200tts_taco_decode_forced needs d_states";
    return B200TTS_EINVAL;
  }
  return taco_decode_impl(ctx, d_memory, d_lengths, B, Tx_max, dropout, n_steps, window, nullptr, d_states, d_frames, d_stop, d_align,
                          d_nsteps, stream);
}

extern "C" int b200tts_taco_decode_gta(b200tts_taco* ctx, const float* d_memory, const int32_t* d_lengths, int B, int Tx_max,
                                       const b200tts_taco_dropout* dropout, const float* d_targets, const int32_t* d_target_lengths,
                                       int Ty_max, float* d_frames, float* d_align, void* stream) {
  API_BEGIN
  REQUIRE(ctx && d_memory && d_lengths && dropout && d_targets && d_target_lengths && d_frames, B200TTS_EINVAL, "null argument");
  REQUIRE(B >= 1 && Tx_max >= 1 && Tx_max <= kTacoMaxTx && Ty_max >= 1, B200TTS_EINVAL, "B, Tx_max (<= 512), Ty_max out of range");
  const b200tts_taco_dropout d = *dropout;
  require_dropout(d);
  TacoArgs a{};
  a.memory = d_memory; a.lengths = d_lengths;
  a.B = B; a.Tx_max = Tx_max; a.max_steps = Ty_max; a.window = 0;
  a.rng_mode = d.mode; a.seed = d.seed; a.utt_offset = d.utterance_offset; a.masks = d.d_masks;
  a.frames = d_frames; a.align = d_align;
  const TacoGtaArgs g{d_targets, d_target_lengths};
  launch_taco_decoder(ctx, a, &g, nullptr, (cudaStream_t)stream);
  API_END
}

extern "C" int b200tts_taco_philox_masks(int device, uint64_t seed, uint64_t utterance_offset, int B, int steps, int prenet_units,
                                         uint8_t* d_masks, void* stream) {
  API_BEGIN
  REQUIRE(d_masks && B >= 1 && steps >= 1 && prenet_units >= 4 && prenet_units % 4 == 0, B200TTS_EINVAL, "bad argument");
  DeviceGuard dg(device);
  size_t total = (size_t)B * steps * 2 * prenet_units;
  unsigned grid = (unsigned)std::min<size_t>((total + 255) / 256, 132 * 16);
  taco_philox_masks_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(seed, utterance_offset, B, steps, prenet_units, d_masks);
  B200_CUDA(cudaGetLastError());
  API_END
}

// One block per sentence: the first step whose stop token exceeds 0.5.
__global__ void taco_target_lengths_kernel(const float* __restrict__ stop, const int32_t* __restrict__ nsteps, int max_steps,
                                           int32_t* __restrict__ len) {
  __shared__ int first;
  const int b = blockIdx.x, n = min(nsteps[b], max_steps);
  if (threadIdx.x == 0) first = n;
  __syncthreads();
  for (int t = threadIdx.x; t < n; t += blockDim.x)
    if (stop[(size_t)b * max_steps + t] > 0.5f) atomicMin(&first, t);
  __syncthreads();
  if (threadIdx.x == 0) len[b] = first;
}

extern "C" int b200tts_taco_target_lengths(const float* d_stop, const int32_t* d_nsteps, int B, int max_steps, int32_t* d_len,
                                           void* stream) {
  API_BEGIN
  REQUIRE(d_stop && d_nsteps && d_len, B200TTS_EINVAL, "null argument");
  REQUIRE(B >= 1 && max_steps >= 1, B200TTS_EINVAL, "B / max_steps out of range");
  taco_target_lengths_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(d_stop, d_nsteps, max_steps, d_len);
  B200_CUDA(cudaGetLastError());
  API_END
}

// ---- decoder sessions: free runs in slices on taco_decoder_session_kernel -----------------------------------------------------
// Every refusal below comes before the first CUDA call, so a refused call has launched and allocated nothing.
extern "C" int b200tts_taco_session_open_batch(b200tts_taco* ctx, const float* d_memory, const int32_t* h_lengths, int n, int Tx_max,
                                               const b200tts_taco_dropout* dropout, const uint64_t* h_ids, int max_steps, int window,
                                               const float* h_mu_bias, b200tts_taco_session** out, void* stream) {
  API_BEGIN
  REQUIRE(ctx && d_memory && h_lengths && dropout && out, B200TTS_EINVAL, "null argument");
  REQUIRE(n >= 1 && n <= kTacoSessRows, B200TTS_EINVAL, "n must be 1..128 (one wave of thread blocks)");
  REQUIRE(Tx_max >= 1 && Tx_max <= kTacoMaxTx, B200TTS_EINVAL, "Tx_max must be 1..512");
  REQUIRE(max_steps >= 1, B200TTS_EINVAL, "max_steps must be >= 1");
  REQUIRE(dropout->mode == B200TTS_TACO_DROPOUT_PHILOX, B200TTS_EINVAL,
          "decoder sessions take PHILOX dropout keyed by (seed, utterance id); EXT masks are refused");
  for (int i = 0; i < n; ++i) REQUIRE(h_lengths[i] >= 1 && h_lengths[i] <= Tx_max, B200TTS_EINVAL, "every length must be 1..Tx_max");
  require_mu_bias(h_mu_bias, n);
  const TacoWeights& w = ctx->tw;
  const int M = w.mels;
  const size_t mem_f = (size_t)n * Tx_max * w.E, keys_f = (size_t)n * Tx_max * w.A;
  const size_t state_stride = ((size_t)taco_state_floats(M, w.E, w.U, Tx_max) + 3) / 4 * 4;
  const size_t out_stride = (size_t)max_steps * (M + 1);      // frames [max_steps][M], then stop [max_steps]
  const size_t zero_f = (size_t)n * (state_stride + out_stride);
  DeviceGuard dg(ctx->device);
  const cudaStream_t st = (cudaStream_t)stream;
  auto block = std::make_shared<DeviceBuf>();
  block->ensure((mem_f + keys_f + zero_f) * sizeof(float));
  float* base = block->as<float>();
  float* mem = base;
  float* keys = mem + mem_f;
  float* rest = keys + keys_f;
  B200_CUDA(cudaMemcpyAsync(mem, d_memory, mem_f * sizeof(float), cudaMemcpyDeviceToDevice, st));
  B200_CUDA(cudaMemsetAsync(rest, 0, zero_f * sizeof(float), st));
  launch_taco_keys(w, mem, n * Tx_max, keys, st);
  std::vector<std::unique_ptr<b200tts_taco_session>> ss(n);
  for (int i = 0; i < n; ++i) {
    ss[i].reset(new b200tts_taco_session());
    b200tts_taco_session& s = *ss[i];
    s.ctx = ctx;
    s.batch = block;
    s.memory = mem + (size_t)i * Tx_max * w.E;
    s.keys = keys + (size_t)i * Tx_max * w.A;
    s.state = rest + (size_t)i * state_stride;
    s.frames = rest + (size_t)n * state_stride + (size_t)i * out_stride;
    s.stop = s.frames + (size_t)max_steps * M;
    s.seed = dropout->seed;
    s.id = h_ids ? h_ids[i] : dropout->utterance_offset + (uint64_t)i;
    s.mu_bias = h_mu_bias ? h_mu_bias[i] : 0.f;
    s.Tx = h_lengths[i];
    s.max_steps = max_steps;
    s.window = window ? 1 : 0;
  }
  for (int i = 0; i < n; ++i) {
    ctx->sessions.insert(ss[i].get());
    out[i] = ss[i].release();
  }
  API_END
}

// cudaFree waits for the work queued on the device, so no slice still in flight reads the memory freed here.
extern "C" void b200tts_taco_session_destroy(b200tts_taco_session* s) {
  if (!s) return;
  DeviceGuard dg(s->ctx->device, true);
  s->ctx->sessions.erase(s);
  delete s;
}

extern "C" int b200tts_taco_session_info(const b200tts_taco_session* s, int32_t* pos, int32_t* done, int32_t* max_steps) {
  API_BEGIN
  REQUIRE(s, B200TTS_EINVAL, "null argument");
  if (pos) *pos = s->pos;
  if (done) *done = s->done ? 1 : 0;
  if (max_steps) *max_steps = s->max_steps;
  API_END
}

static void require_sessions(const b200tts_taco* ctx, b200tts_taco_session* const* s, int n) {
  REQUIRE(s, B200TTS_EINVAL, "null argument");
  REQUIRE(n >= 1 && n <= kTacoSessRows, B200TTS_EINVAL, "n must be 1..128 sessions");
  for (int i = 0; i < n; ++i) {
    REQUIRE(s[i], B200TTS_EINVAL, "null session");
    REQUIRE(!ctx || s[i]->ctx == ctx, B200TTS_EINVAL, "the session belongs to another context");
    REQUIRE(s[i]->ctx == s[0]->ctx, B200TTS_EINVAL, "the sessions belong to different contexts");
    for (int j = 0; j < i; ++j) REQUIRE(s[j] != s[i], B200TTS_EINVAL, "the same session appears twice in one call");
  }
}

extern "C" int b200tts_taco_session_run(b200tts_taco* ctx, b200tts_taco_session* const* s, int n, int max_steps, void* stream) {
  API_BEGIN
  REQUIRE(ctx, B200TTS_EINVAL, "null argument");
  require_sessions(ctx, s, n);
  REQUIRE(max_steps >= 1, B200TTS_EINVAL, "max_steps must be >= 1");
  // finished sessions take part with 0 steps: they get no thread block
  TacoSessIO io{};
  int rows[kTacoSessRows], m = 0;
  for (int i = 0; i < n; ++i) {
    if (s[i]->done) continue;
    TacoSessRow& r = io.row[m];
    r.memory = s[i]->memory; r.keys = s[i]->keys; r.state = s[i]->state;
    r.frames = s[i]->frames; r.stop = s[i]->stop;
    r.seed = s[i]->seed; r.id = s[i]->id; r.mu_bias = s[i]->mu_bias;
    r.Tx = s[i]->Tx; r.pos = s[i]->pos; r.n = std::min(max_steps, s[i]->max_steps - s[i]->pos); r.window = s[i]->window;
    rows[m++] = i;
  }
  if (m == 0) return B200TTS_OK;
  DeviceGuard dg(ctx->device);
  const cudaStream_t st = (cudaStream_t)stream;
  ctx->sess_status.ensure((size_t)kTacoSessRows * 2 * sizeof(int));
  ctx->h_sess_status.ensure((size_t)kTacoSessRows * 2 * sizeof(int));
  int* d_status = ctx->sess_status.as<int>();
  for (int u = 0; u < m; ++u) io.row[u].status = d_status + 2 * u;
  launch_taco_sessions(ctx->tw, io, m, taco_decoder_smem_bytes(ctx->tw), st);
  // where each decode stopped is decided on the device: wait for the slice and read the positions back
  int* h = static_cast<int*>(ctx->h_sess_status.p);
  B200_CUDA(cudaMemcpyAsync(h, d_status, (size_t)m * 2 * sizeof(int), cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  for (int u = 0; u < m; ++u) {
    b200tts_taco_session& x = *s[rows[u]];
    x.pos = h[2 * u];
    x.done = h[2 * u + 1] != 0 || x.pos >= x.max_steps;
  }
  API_END
}

extern "C" int b200tts_taco_session_outputs(b200tts_taco_session* const* s, int n, int T_max, float* d_frames, float* d_stop,
                                            int32_t* d_nsteps, void* stream) {
  API_BEGIN
  require_sessions(nullptr, s, n);
  REQUIRE(d_frames && d_stop && d_nsteps, B200TTS_EINVAL, "null argument");
  REQUIRE(T_max >= 1, B200TTS_EINVAL, "T_max must be >= 1");
  TacoSessOut g{};
  for (int i = 0; i < n; ++i) {
    REQUIRE(s[i]->pos <= T_max, B200TTS_EINVAL, "T_max is shorter than a session's steps");
    g.frames[i] = s[i]->frames; g.stop[i] = s[i]->stop; g.pos[i] = s[i]->pos;
  }
  b200tts_taco* ctx = s[0]->ctx;
  DeviceGuard dg(ctx->device);
  launch_taco_session_outputs(g, n, T_max, ctx->tw.mels, d_frames, d_stop, d_nsteps, (cudaStream_t)stream);
  API_END
}

static void taco_launch_conv(b200tts_taco* ctx, const TacoConvW& cw, const float* x, const int* ids, const int* lengths, int B, int Tmax,
                             int act, bool clip_in, float lo, float hi, float* y, cudaStream_t st) {
  ConvArgs a{};
  a.x = x; a.ids = ids; a.table = ctx->embedding; a.lengths = lengths;
  a.K = cw.K; a.bias = cw.bias; a.bn_scale = cw.scale; a.bn_shift = cw.shift; a.y = y;
  a.Tmax = Tmax; a.Cin = cw.Cin; a.Cout = cw.Cout; a.k = cw.k; a.act = act; a.clip_in = clip_in ? 1 : 0; a.lo = lo; a.hi = hi;
  size_t smem = (size_t)(kConvTile + cw.k - 1) * cw.Cin * sizeof(float);
  dim3 grid((Tmax + kConvTile - 1) / kConvTile, B);
  taco_conv_bn_kernel<<<grid, 256, smem, st>>>(a);
  B200_CUDA(cudaGetLastError());
}

extern "C" int b200tts_taco_encode(b200tts_taco* ctx, const int32_t* d_ids, const int32_t* d_lengths, int B, int Tx_max, float* d_memory,
                                   void* stream) {
  API_BEGIN
  REQUIRE(ctx && d_ids && d_lengths && d_memory, B200TTS_EINVAL, "null argument");
  REQUIRE(ctx->has_encoder, B200TTS_EMISSING, "this context was created without the encoder variables");
  REQUIRE(B >= 1 && Tx_max >= 1 && Tx_max <= kTacoMaxTx, B200TTS_EINVAL, "B / Tx_max out of range");
  DeviceGuard dg(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  const int C = ctx->enc_conv[0].Cout;
  ctx->act_a.ensure((size_t)B * Tx_max * C * sizeof(float));
  ctx->act_b.ensure((size_t)B * Tx_max * C * sizeof(float));
  float* a = ctx->act_a.as<float>();
  float* bb = ctx->act_b.as<float>();
  taco_launch_conv(ctx, ctx->enc_conv[0], nullptr, d_ids, d_lengths, B, Tx_max, 1, false, 0.f, 0.f, a, st);
  taco_launch_conv(ctx, ctx->enc_conv[1], a, nullptr, d_lengths, B, Tx_max, 1, false, 0.f, 0.f, bb, st);
  taco_launch_conv(ctx, ctx->enc_conv[2], bb, nullptr, d_lengths, B, Tx_max, 1, false, 0.f, 0.f, a, st);
  const int U = ctx->enc_units, Cin = ctx->enc_conv[2].Cout;
  size_t smem = ((size_t)(Cin + U) + 4 * U + U + 4 * 4 * U) * sizeof(float);
  B200_CUDA(cudaFuncSetAttribute(taco_bilstm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  taco_bilstm_kernel<<<dim3(B, 2), kTacoThreads, smem, st>>>(a, d_lengths, Tx_max, Cin, U, ctx->enc_kfw, ctx->enc_bfw, ctx->enc_kbw,
                                                              ctx->enc_bbw, ctx->cfg.zoneout, d_memory);
  B200_CUDA(cudaGetLastError());
  API_END
}

extern "C" int b200tts_taco_postnet(b200tts_taco* ctx, const float* d_frames, const int32_t* d_nsteps, int B, int max_steps, float* d_mel,
                                    void* stream) {
  API_BEGIN
  REQUIRE(ctx && d_frames && d_nsteps && d_mel, B200TTS_EINVAL, "null argument");
  REQUIRE(ctx->has_postnet, B200TTS_EMISSING, "this context was created without the postnet variables");
  REQUIRE(B >= 1 && max_steps >= 1, B200TTS_EINVAL, "B / max_steps out of range");
  DeviceGuard dg(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  const int C = ctx->post_channels, M = ctx->cfg.num_mels;
  const float lo = -4.0f - 0.1f, hi = 4.0f;       // T2_output_range[0] - lower_bound_decay, T2_output_range[1] (tacotron.py:33,111-112)
  ctx->act_a.ensure((size_t)B * max_steps * C * sizeof(float));
  ctx->act_b.ensure((size_t)B * max_steps * C * sizeof(float));
  float* a = ctx->act_a.as<float>();
  float* bb = ctx->act_b.as<float>();
  taco_launch_conv(ctx, ctx->post_conv[0], d_frames, nullptr, d_nsteps, B, max_steps, 2, true, lo, hi, a, st);
  taco_launch_conv(ctx, ctx->post_conv[1], a, nullptr, d_nsteps, B, max_steps, 2, false, 0.f, 0.f, bb, st);
  taco_launch_conv(ctx, ctx->post_conv[2], bb, nullptr, d_nsteps, B, max_steps, 2, false, 0.f, 0.f, a, st);
  taco_launch_conv(ctx, ctx->post_conv[3], a, nullptr, d_nsteps, B, max_steps, 2, false, 0.f, 0.f, bb, st);
  taco_launch_conv(ctx, ctx->post_conv[4], bb, nullptr, d_nsteps, B, max_steps, 0, false, 0.f, 0.f, a, st);
  taco_postnet_proj_kernel<<<dim3(max_steps, B), 128, C * sizeof(float), st>>>(d_frames, a, d_nsteps, max_steps, C, M, ctx->post_pk,
                                                                                 ctx->post_pb, lo, hi, d_mel);
  B200_CUDA(cudaGetLastError());
  API_END
}
