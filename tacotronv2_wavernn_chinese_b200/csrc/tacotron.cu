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
  int64_t launches = 0;
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
  auto copy = [&](const std::string& name, std::initializer_list<int64_t> shape) {
    const b200tts_tensor* t = need(tm, name, shape);
    size_t n = 1;
    for (int64_t s : shape) n *= (size_t)s;
    size_t off = pk.add(n);
    std::memcpy(&pk.h[off], t->data, n * sizeof(float));
    return off;
  };
  const std::string D = "decoder/", L = D + "Location_Sensitive_Attention/";
  size_t o[21];
  o[0] = copy(D + "decoder_prenet/dense_1/kernel", {M, P}); o[1] = copy(D + "decoder_prenet/dense_1/bias", {P});
  o[2] = copy(D + "decoder_prenet/dense_2/kernel", {P, P}); o[3] = copy(D + "decoder_prenet/dense_2/bias", {P});
  o[4] = copy(D + "decoder_LSTM/multi_rnn_cell/cell_0/decoder_LSTM_1/kernel", {P + E + U, 4 * U});
  o[5] = copy(D + "decoder_LSTM/multi_rnn_cell/cell_0/decoder_LSTM_1/bias", {4 * U});
  o[6] = copy(D + "decoder_LSTM/multi_rnn_cell/cell_1/decoder_LSTM_2/kernel", {2 * U, 4 * U});
  o[7] = copy(D + "decoder_LSTM/multi_rnn_cell/cell_1/decoder_LSTM_2/bias", {4 * U});
  o[8] = copy(L + "query_layer/kernel", {U, AD});
  o[9] = copy(L + "location_features_convolution/kernel", {KW, 1, NF}); o[10] = copy(L + "location_features_convolution/bias", {NF});
  o[11] = copy(L + "location_features_layer/kernel", {NF, AD});
  o[12] = copy(L + "attention_variable_projection", {AD}); o[13] = copy(L + "attention_bias", {AD});
  o[14] = copy(D + "dense/kernel", {E + U, 1}); o[15] = copy(D + "dense/bias", {1});
  o[16] = copy(D + "linear_transform_projection/projection_linear_transform_projection/kernel", {U + E, M});
  o[17] = copy(D + "linear_transform_projection/projection_linear_transform_projection/bias", {M});
  o[18] = copy(D + "stop_token_projection/projection_stop_token_projection/kernel", {U + E, 1});
  o[19] = copy(D + "stop_token_projection/projection_stop_token_projection/bias", {1});
  o[20] = copy("memory_layer/kernel", {E, AD});
  // ---- optional run-once neighbours: encoder and postnet ----
  struct ConvOff { size_t K, bias, scale, shift; int k, Cin, Cout; };
  auto pack_conv = [&](const std::string& scope) {
    auto it = tm.find(scope + "/conv1d/kernel");
    REQUIRE(it != tm.end() && it->second->ndim == 3, B200TTS_EMISSING, "missing weight tensor '" + scope + "/conv1d/kernel'");
    const b200tts_tensor* kt = it->second;
    ConvOff c{};
    c.k = (int)kt->shape[0]; c.Cin = (int)kt->shape[1]; c.Cout = (int)kt->shape[2];
    c.K = copy(scope + "/conv1d/kernel", {c.k, c.Cin, c.Cout});
    c.bias = copy(scope + "/conv1d/bias", {c.Cout});
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
    o_emb = copy("inputs_embedding", {ctx->vocab, ctx->emb_dim});
    for (int i = 0; i < 3; ++i) encc[i] = pack_conv("encoder_convolutions/conv_layer_" + std::to_string(i + 1) + "_encoder_convolutions");
    REQUIRE(encc[0].Cin == ctx->emb_dim && encc[2].Cout % 4 == 0 && E % 2 == 0, B200TTS_ESHAPE, "encoder conv shapes");
    const int EU = E / 2, CI = encc[2].Cout;
    REQUIRE(4 * EU == 1024, B200TTS_EINVAL, "encoder LSTM units must be 256");
    const std::string LS = "encoder_LSTM/bidirectional_rnn/";
    o_kfw = copy(LS + "fw/encoder_fw_LSTM/kernel", {CI + EU, 4 * EU}); o_bfw = copy(LS + "fw/encoder_fw_LSTM/bias", {4 * EU});
    o_kbw = copy(LS + "bw/encoder_bw_LSTM/kernel", {CI + EU, 4 * EU}); o_bbw = copy(LS + "bw/encoder_bw_LSTM/bias", {4 * EU});
    ctx->enc_units = EU;
    ctx->has_encoder = true;
  }
  if (tm.count("postnet_projection/projection_postnet_projection/kernel")) {
    for (int i = 0; i < 5; ++i) postc[i] = pack_conv("postnet_convolutions/conv_layer_" + std::to_string(i + 1) + "_postnet_convolutions");
    REQUIRE(postc[0].Cin == M, B200TTS_ESHAPE, "postnet conv 1 must take num_mels channels");
    ctx->post_channels = postc[4].Cout;
    o_pk = copy("postnet_projection/projection_postnet_projection/kernel", {ctx->post_channels, M});
    o_pb = copy("postnet_projection/projection_postnet_projection/bias", {M});
    ctx->has_postnet = true;
  }
  ctx->weights.ensure(pk.h.size() * sizeof(float));
  B200_CUDA(cudaMemcpy(ctx->weights.p, pk.h.data(), pk.h.size() * sizeof(float), cudaMemcpyHostToDevice));
  const float* b = ctx->weights.as<float>();
  TacoWeights& w = ctx->tw;
  w.pre1_k = b + o[0]; w.pre1_b = b + o[1]; w.pre2_k = b + o[2]; w.pre2_b = b + o[3];
  w.l1_k = b + o[4]; w.l1_b = b + o[5]; w.l2_k = b + o[6]; w.l2_b = b + o[7];
  w.q_k = b + o[8]; w.loc_k = b + o[9]; w.loc_b = b + o[10]; w.locl_k = b + o[11]; w.v_a = b + o[12]; w.b_a = b + o[13];
  w.mu_k = b + o[14]; w.mu_b = b + o[15]; w.fr_k = b + o[16]; w.fr_b = b + o[17]; w.st_k = b + o[18]; w.st_b = b + o[19];
  w.mem_k = b + o[20];
  w.mels = M; w.P = P; w.U = U; w.E = E; w.A = AD; w.NF = NF; w.KW = KW; w.zoneout = c.zoneout;
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
  {
    int coop = 0;
    B200_CUDA(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, device));
    B200_CUDA(cudaDeviceGetAttribute(&ctx->sm_count, cudaDevAttrMultiProcessorCount, device));
    if (coop && ctx->sm_count >= kTgCtas && P == 256 && U == 256 && E == 512 && AD == 128 && M <= 96 && KW <= 64) {
      TacoGridModel& g = ctx->tgm;
      g.M = M; g.P = P; g.U = U; g.E = E; g.KW = KW;
      int off = 0;
      auto take = [&](int n) { int o0 = off; off += (n + 3) & ~3; return o0; };
      g.oW1 = take(M * 2); g.oB1 = take(2);
      g.oWfold = take((U + E) * 2); g.oBfold = take(2);
      g.oW2 = take(P * 2); g.oB2 = take(2);
      g.oK1 = take((P + E + U) * 8); g.oBk1 = take(8);
      g.oK2 = take(2 * U * 8); g.oBk2 = take(8);
      g.oWq = take(U);
      g.oFloc = take(KW + 4);
      g.oProj = take((U + E) * 4 + 4);
      g.blob = off;
      const float* H = pk.h.data();
      const float *W1 = H + o[0], *b1 = H + o[1], *W2 = H + o[2], *b2 = H + o[3], *K1 = H + o[4], *bk1 = H + o[5], *K2 = H + o[6],
                  *bk2 = H + o[7], *Wq = H + o[8], *lock = H + o[9], *locb = H + o[10], *locl = H + o[11], *va = H + o[12], *ba = H + o[13],
                  *muk = H + o[14], *mub = H + o[15], *frk = H + o[16], *frb = H + o[17], *stk = H + o[18], *stb = H + o[19];
      // W_f . W_1 and b_f . W_1 + b_1 in float64
      std::vector<double> fold((size_t)(U + E) * P), bfold(P);
      for (int i = 0; i < U + E; ++i)
        for (int p2 = 0; p2 < P; ++p2) {
          double a = 0;
          for (int m = 0; m < M; ++m) a += (double)frk[(size_t)i * M + m] * (double)W1[(size_t)m * P + p2];
          fold[(size_t)i * P + p2] = a;
        }
      for (int p2 = 0; p2 < P; ++p2) {
        double a = b1[p2];
        for (int m = 0; m < M; ++m) a += (double)frb[m] * (double)W1[(size_t)m * P + p2];
        bfold[p2] = a;
      }
      std::vector<float> hb((size_t)kTgCtas * g.blob, 0.f);
      for (int c2 = 0; c2 < kTgCtas; ++c2) {
        float* d = &hb[(size_t)c2 * g.blob];
        for (int j = 0; j < 2; ++j) {
          const int col = 2 * c2 + j;
          for (int m = 0; m < M; ++m) d[g.oW1 + m * 2 + j] = W1[(size_t)m * P + col];
          d[g.oB1 + j] = b1[col];
          for (int i = 0; i < U + E; ++i) d[g.oWfold + i * 2 + j] = (float)fold[(size_t)i * P + col];
          d[g.oBfold + j] = (float)bfold[col];
          for (int k = 0; k < P; ++k) d[g.oW2 + k * 2 + j] = W2[(size_t)k * P + col];
          d[g.oB2 + j] = b2[col];
          for (int gate = 0; gate < 4; ++gate) {
            const int src = gate * U + col, dst = gate * 2 + j;
            for (int k = 0; k < P + E + U; ++k) d[g.oK1 + k * 8 + dst] = K1[(size_t)k * 4 * U + src];
            d[g.oBk1 + dst] = bk1[src];
            for (int k = 0; k < 2 * U; ++k) d[g.oK2 + k * 8 + dst] = K2[(size_t)k * 4 * U + src];
            d[g.oBk2 + dst] = bk2[src];
          }
        }
        for (int u = 0; u < U; ++u) d[g.oWq + u] = Wq[(size_t)u * AD + c2];
        double bl = ba[c2];
        for (int f = 0; f < NF; ++f) bl += (double)locb[f] * (double)locl[(size_t)f * AD + c2];
        for (int k = 0; k < KW; ++k) {
          double a = 0;
          for (int f = 0; f < NF; ++f) a += (double)lock[(size_t)k * NF + f] * (double)locl[(size_t)f * AD + c2];
          d[g.oFloc + k] = (float)a;
        }
        d[g.oFloc + KW] = (float)bl;
        d[g.oFloc + KW + 1] = va[c2];
        d[g.oFloc + KW + 2] = 1.0f - c.zoneout;
        d[g.oFloc + KW + 3] = c.zoneout;
        for (int i = 0; i < U + E; ++i) {
          d[g.oProj + i * 4 + 0] = muk[i < U ? E + i : i - U];          // attention.py:229 concatenates [context, query]
          d[g.oProj + i * 4 + 1] = stk[i];
          d[g.oProj + i * 4 + 2] = c2 < M ? frk[(size_t)i * M + c2] : 0.f;
        }
        d[g.oProj + (U + E) * 4 + 0] = mub[0];
        d[g.oProj + (U + E) * 4 + 1] = stb[0];
        d[g.oProj + (U + E) * 4 + 2] = c2 < M ? frb[c2] : 0.f;
      }
      ctx->tg_blob.ensure(hb.size() * sizeof(float));
      B200_CUDA(cudaMemcpy(ctx->tg_blob.p, hb.data(), hb.size() * sizeof(float), cudaMemcpyHostToDevice));
      ctx->tg_ok = true;
    }
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

// h_mu_bias: NULL for the unbiased kernels, else [B] host speaking-rate biases (b200tts_taco_decode_biased)
static int taco_decode_impl(b200tts_taco* ctx, const float* d_memory, const int32_t* d_lengths, int B, int Tx_max,
                            const b200tts_taco_dropout* dropout, int max_steps, int window, const float* h_mu_bias,
                            const float* d_forced, float* d_frames, float* d_stop, float* d_align, int32_t* d_nsteps, void* stream) {
  API_BEGIN
  REQUIRE(ctx && d_memory && d_lengths && d_frames && d_stop && d_nsteps, B200TTS_EINVAL, "null argument");
  REQUIRE(B >= 1 && Tx_max >= 1 && Tx_max <= kTacoMaxTx && max_steps >= 1, B200TTS_EINVAL, "B, Tx_max (<= 512), max_steps out of range");
  b200tts_taco_dropout d{};
  if (dropout) d = *dropout;
  REQUIRE(d.mode == B200TTS_TACO_DROPOUT_PHILOX || (d.mode == B200TTS_TACO_DROPOUT_EXT && d.d_masks), B200TTS_EINVAL,
          "bad dropout descriptor");
  require_mu_bias(h_mu_bias, B);
  DeviceGuard dg(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  const TacoWeights& w = ctx->tw;
  const float* d_mu_bias = nullptr;
  if (h_mu_bias) {
    ctx->mu_bias.ensure((size_t)B * sizeof(float));
    B200_CUDA(cudaMemcpyAsync(ctx->mu_bias.p, h_mu_bias, (size_t)B * sizeof(float), cudaMemcpyHostToDevice, st));
    d_mu_bias = ctx->mu_bias.as<float>();
  }
  ctx->keys.ensure((size_t)B * Tx_max * w.A * sizeof(float));
  taco_keys_kernel<<<B * Tx_max, 128, w.E * sizeof(float), st>>>(d_memory, w.mem_k, B * Tx_max, w.E, w.A, ctx->keys.as<float>());
  B200_CUDA(cudaGetLastError());
  TacoArgs a{};
  a.memory = d_memory; a.keys = ctx->keys.as<float>(); a.lengths = d_lengths;
  a.B = B; a.Tx_max = Tx_max; a.max_steps = max_steps; a.window = window;
  a.rng_mode = d.mode; a.seed = d.seed; a.utt_offset = d.utterance_offset; a.masks = d.d_masks;
  a.frames = d_frames; a.stop = d_stop; a.align = d_align; a.nsteps = d_nsteps;
  a.forced = d_forced;
  if (B == 1 && ctx->tg_ok) {
    // ONE sentence: the weight-stationary 128-block decoder (taco_grid.cuh).  The sentence length is needed on the host to size
    // the exchange buffers; d_lengths is a device pointer, so Tx_max (the caller's padded length) bounds it and the kernel
    // reads the true length itself.
    const TacoGridModel& g = ctx->tgm;
    const int Txp = (Tx_max + 3) & ~3;
    const size_t copy = (size_t)2048 + (size_t)kTgCtas * Txp;
    ctx->tg_vec.ensure(2 * copy * sizeof(float) + 64);
    int* d_err = reinterpret_cast<int*>(ctx->tg_vec.as<float>() + 2 * copy);
    launch_push_init(ctx->tg_vec.as<uint32_t>(), 2 * copy, nullptr, 0, d_err, ctx->sm_count, st);
    TacoGridArgs ga{};
    ga.wblob = ctx->tg_blob.as<float>();
    ga.vec = ctx->tg_vec.as<float>();
    ga.error = d_err;
    ga.memory = d_memory; ga.keys = ctx->keys.as<float>();
    ga.lengths = d_lengths;
    ga.Tx = Tx_max; ga.Txp = Txp; ga.max_steps = max_steps; ga.window = window;
    ga.rng_mode = d.mode; ga.seed = d.seed; ga.utt = d.utterance_offset; ga.masks = d.d_masks;
    ga.forced = d_forced; ga.Tx_alloc = Tx_max;
    ga.frames = d_frames; ga.stop = d_stop; ga.align = d_align; ga.nsteps = d_nsteps;
    const size_t fl = (size_t)g.blob + (size_t)(w.P + w.E + w.U) + 2 * w.U + (w.U + w.E) + w.P + 128 + 24 * (size_t)Txp + 176;
    const size_t smem = fl * sizeof(float);
    REQUIRE(smem <= 227 * 1024, B200TTS_EINVAL, "taco_grid_kernel: shared memory budget exceeded");
    const void* kernel = d_mu_bias ? (const void*)taco_grid_biased_kernel : (const void*)taco_grid_kernel;
    B200_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    TacoGridModel gm = g;
    void* args[] = {(void*)&gm, (void*)&ga, (void*)&d_mu_bias};
    B200_CUDA(cudaLaunchCooperativeKernel(kernel, dim3(kTgCtas), dim3(kTgThreads), args, smem, st));
    taco_grid_finish_kernel<<<1, 1, 0, st>>>(d_err, d_nsteps);
    B200_CUDA(cudaGetLastError());
    ctx->launches += 4;
    return B200TTS_OK;
  }
  const size_t smem = taco_decoder_smem_bytes(w);
  if (d_mu_bias) {
    B200_CUDA(cudaFuncSetAttribute(taco_decoder_biased_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    taco_decoder_biased_kernel<<<B, kTacoThreads, smem, st>>>(w, a, d_mu_bias);
  } else {
    B200_CUDA(cudaFuncSetAttribute(taco_decoder_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    taco_decoder_kernel<false><<<B, kTacoThreads, smem, st>>>(w, a, TacoGtaArgs{});
  }
  B200_CUDA(cudaGetLastError());
  ctx->launches += 2;
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
  REQUIRE(d.mode == B200TTS_TACO_DROPOUT_PHILOX || (d.mode == B200TTS_TACO_DROPOUT_EXT && d.d_masks), B200TTS_EINVAL,
          "bad dropout descriptor");
  DeviceGuard dg(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  const TacoWeights& w = ctx->tw;
  ctx->keys.ensure((size_t)B * Tx_max * w.A * sizeof(float));
  taco_keys_kernel<<<B * Tx_max, 128, w.E * sizeof(float), st>>>(d_memory, w.mem_k, B * Tx_max, w.E, w.A, ctx->keys.as<float>());
  B200_CUDA(cudaGetLastError());
  // one CTA per sentence at every B: a batch job, so the single-sentence grid decoder is not taught the fed frame
  TacoArgs a{};
  a.memory = d_memory; a.keys = ctx->keys.as<float>(); a.lengths = d_lengths;
  a.B = B; a.Tx_max = Tx_max; a.max_steps = Ty_max; a.window = 0;
  a.rng_mode = d.mode; a.seed = d.seed; a.utt_offset = d.utterance_offset; a.masks = d.d_masks;
  a.frames = d_frames; a.align = d_align;
  TacoGtaArgs g{};
  g.targets = d_targets; g.target_lengths = d_target_lengths;
  const size_t smem = taco_decoder_smem_bytes(w);
  B200_CUDA(cudaFuncSetAttribute(taco_decoder_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  taco_decoder_kernel<true><<<B, kTacoThreads, smem, st>>>(w, a, g);
  B200_CUDA(cudaGetLastError());
  ctx->launches += 2;
  API_END
}

extern "C" int b200tts_taco_philox_masks(int device, uint64_t seed, uint64_t utterance_offset, int B, int steps, int prenet_units,
                                         uint8_t* d_masks, void* stream) {
  API_BEGIN
  REQUIRE(d_masks && B >= 1 && steps >= 1 && prenet_units >= 4, B200TTS_EINVAL, "bad argument");
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
  taco_keys_kernel<<<n * Tx_max, 128, w.E * sizeof(float), st>>>(mem, w.mem_k, n * Tx_max, w.E, w.A, keys);
  B200_CUDA(cudaGetLastError());
  ctx->launches++;
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
  ctx->launches++;
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
  ctx->launches++;
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
  ctx->launches++;
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
  ctx->launches++;
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
  ctx->launches++;
  API_END
}
