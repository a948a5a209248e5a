/*
 * b200tts.h -- C ABI of libb200tts.so: the sm_90a replacement for the hot paths of
 * lturing/tacotronv2_wavernn_chinese.
 *
 * The reference is pure Python and has no FFI of its own (SURVEY.md section 8b); the
 * boundary that a maintainer binds is therefore the body of three Python methods.
 * Each entry point below names the reference interface it replaces
 * (paths relative to the reference root):
 *
 *   b200tts_wavernn_create     <- WaveRNN.__init__ + WaveRNN.load      wavernn/models/fatchord_version.py:93-129, :414-417
 *   b200tts_wavernn_upsample   <- UpsampleNetwork.forward (+pad_tensor) wavernn/models/fatchord_version.py:82-89, :185-186, :281-291
 *   b200tts_wavernn_generate   <- WaveRNN.generate (unbatched branch)   wavernn/models/fatchord_version.py:169-264
 *                                 incl. decode_mu_law                   wavernn/utils/dsp.py:98-103
 *   b200tts_wavernn_generate_host  same, HOST buffers in/out (what wavernn_gen.py:41 sees end to end)
 *   b200tts_wavernn_create_mol / _generate_mol  the same with voc_mode = 'MOL' (wavernn_hparams.py:35): fc3 gives a mixture
 *                                 of 10 logistics, sampled by sample_from_discretized_mix_logistic  wavernn/utils/distribution.py:87-123
 *   gen_opts.fold_target/_overlap  <- fold_with_overlap + xfade_and_unfold  fatchord_version.py:293-405 (--batched)
 *   b200tts_griffin_lim        <- audio.inv_mel_spectrogram (Griffin-Lim) tacotron/datasets/audio.py:122-137, :176-210
 *   b200tts_resample           <- audio.load_wav at another rate (librosa 0.7.2 core.resample, resampy kaiser_best) :14-15
 *
 * Conventions
 *   - plain C types only; no torch / CUDA types in any signature (`stream` is a cudaStream_t passed as void*).
 *   - all `d_*` pointers are DEVICE pointers on the context's device, all `h_*` pointers are HOST pointers;
 *     the caller owns every buffer it passes, the library owns only what *_create allocates.
 *   - every function returns 0 on success or a negative B200TTS_E* code; the message is available from
 *     b200tts_last_error() (thread local).  Nothing aborts or throws across the ABI.
 *   - work is enqueued on `stream` and is asynchronous unless stated; a context is bound to one device and
 *     its calls must be serialised by the caller (one context per GPU per process).
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails with B200TTS_ECUDA.
 */
#ifndef B200TTS_H_
#define B200TTS_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200TTS_ABI_VERSION 3

enum {
  B200TTS_OK = 0,
  B200TTS_EINVAL = -1,   /* bad argument / unsupported configuration            */
  B200TTS_ECUDA = -2,    /* CUDA runtime error (message carries the CUDA string) */
  B200TTS_ENOMEM = -3,   /* device or host allocation failed                    */
  B200TTS_EMISSING = -4, /* a required weight tensor was not supplied           */
  B200TTS_ESHAPE = -5    /* a weight tensor has the wrong shape                 */
};

/* Model dimensions = the constructor arguments of the reference WaveRNN (fatchord_version.py:93-95),
 * filled from wavernn_hparams.py:18-41,50. */
typedef struct {
  int32_t rnn_dims;            /* voc_rnn_dims     512 */
  int32_t fc_dims;             /* voc_fc_dims      512 */
  int32_t bits;                /* bits             10  -> n_classes = 1 << bits */
  int32_t pad;                 /* voc_pad          2   */
  int32_t feat_dims;           /* num_mels         80  */
  int32_t compute_dims;        /* voc_compute_dims 128 */
  int32_t res_out_dims;        /* voc_res_out_dims 128 (aux_dims = res_out_dims / 4) */
  int32_t res_blocks;          /* voc_res_blocks   10  */
  int32_t n_upsample;          /* len(voc_upsample_factors), <= 4 */
  int32_t upsample_factors[4]; /* (5, 5, 11) */
  int32_t hop_length;          /* 275 == prod(upsample_factors) */
} b200tts_wavernn_cfg;

/* One named fp32 weight tensor in HOST memory, contiguous row-major; names are the reference
 * state_dict keys ("I.weight", "rnn1.weight_ih_l0", "upsample.resnet.layers.3.batch_norm1.running_var", ...).
 * The library copies and repacks; the caller may free the data after *_create returns. */
typedef struct {
  const char* name;
  const float* data;
  int32_t ndim;
  int64_t shape[4];
} b200tts_tensor;

/* Sampling noise for `Categorical(softmax(logits)).sample()` (fatchord_version.py:232-235), which the
 * reference evaluates as argmax_i(p_i / q_i), q_i ~ Exp(1).  The kernels evaluate the equivalent
 * argmax_i(logit_i - log q_i). */
enum {
  B200TTS_RNG_PHILOX = 0,          /* q from Philox4x32-10 keyed by (seed, global utterance, step, class) */
  B200TTS_RNG_EXT_EXPONENTIAL = 1, /* q read from d_q[S][B][n_classes] (tests: noise shared with the oracle) */
  B200TTS_RNG_EXT_UNIFORM = 2      /* MOL only: the 11 uniforms of each step read from d_q[S][B][11] (see _generate_mol) */
};
typedef struct {
  int32_t mode;
  uint64_t seed;
  uint64_t utterance_offset; /* global index of row 0 (multi-GPU shards keep results independent of the split) */
  const float* d_q;          /* EXT_EXPONENTIAL only */
  const uint64_t* d_utterance_ids; /* optional [B] (ABI 2): global index of EVERY row, for batches whose rows are not consecutive
                                      utterances (length-sorted chunks of a ragged set, pipeline.py); overrides utterance_offset */
} b200tts_rng;

enum {
  B200TTS_KERNEL_AUTO = 0,
  B200TTS_KERNEL_UTTERANCE = 1, /* one CTA per group of utterances, weights streamed from L2      */
  B200TTS_KERNEL_GRID = 2,      /* weight-stationary persistent cooperative grid, all SMs per step */
  B200TTS_KERNEL_TC = 3         /* layer-stationary tensor-core pipeline (wgmma, split-fp16 operands), 33-256 rows */
};
typedef struct {
  int32_t kernel;             /* B200TTS_KERNEL_*                                                      */
  int32_t mu_law;             /* hp.mu_law (wavernn_hparams.py:28); non-zero -> decode_mu_law          */
  const int16_t* d_teacher;   /* optional [B][S]: fed back instead of the sampled label (teacher forcing) */
  float* d_logits;            /* optional [S][B][n_classes]: fc3 outputs of every step (debug / parity) */
  int32_t max_steps;          /* 0 = all S = T*hop steps; otherwise stop early (no wave is produced)   */
  int32_t fold_target;        /* > 0: fold-with-overlap batched generation of ONE utterance (fatchord_version.py:188-190,
                                 :250-251, :293-405; hp.voc_target).  Then B must be 1, d_labels (if given) is
                                 [n_folds][fold_len] (see b200tts_wavernn_fold_geometry) and d_wave is the cross-faded wave */
  int32_t fold_overlap;       /* hp.voc_overlap                                                          */
  const int32_t* d_utt_frames;/* optional [B]: true frame count of each row of a zero-padded ragged batch; row b of d_wave is then
                                 truncated and faded at (frames_b - 1)*hop like a batch-1 run, and zero beyond      */
  /* PACKED generation of a ragged set (ABI 3; no counterpart in the reference, which is batch-1).  The B utterances of d_mel are
   * not one row each: `pack_rows` (<= 32) kernel rows each run a QUEUE of utterances back to back -- segment k of row r is
   * utterance d_pack_utt[r*pack_segs + k] (< 0: none) and occupies lock-steps [d_pack_start[r*(pack_segs+1) + k],
   * d_pack_start[r*(pack_segs+1) + k + 1]); a row restarts from the zero state (fatchord_version.py:194-196) at every segment
   * start and the noise is keyed by (utterance, step within the utterance), so every utterance gets bit for bit the labels of a
   * stand-alone run.  Lock-steps are spent on samples that are needed instead of on padding.  d_labels stays [B][S], d_wave
   * [B][(T-1)*hop] (give d_utt_frames).  Requires the push kernel (rnn_dims = fc_dims = 512), PHILOX noise, no debug buffers. */
  const int32_t* d_pack_utt;
  const int32_t* d_pack_start;
  int32_t pack_rows, pack_segs, pack_steps;   /* pack_steps = last segment end over all rows */
} b200tts_gen_opts;

typedef struct b200tts_wavernn b200tts_wavernn;

int b200tts_abi_version(void);
const char* b200tts_last_error(void);
/* number of CUDA devices visible, or a negative error */
int b200tts_device_count(void);

int b200tts_wavernn_create(b200tts_wavernn** out, int device, const b200tts_wavernn_cfg* cfg,
                           const b200tts_tensor* weights, int n_weights);
void b200tts_wavernn_destroy(b200tts_wavernn* ctx);

/* d_mel [B][feat][T] (unpadded, as generate() receives it) ->
 *   d_mels_up    [B][T*hop][feat]     (may be NULL)
 *   d_aux_frames [B][T][res_out]      (may be NULL; aux is constant within a hop, so it is kept at frame rate)
 *   d_aux_full   [B][T*hop][res_out]  (may be NULL; the reference's materialised layout) */
int b200tts_wavernn_upsample(b200tts_wavernn* ctx, const float* d_mel, int B, int T, float* d_mels_up,
                             float* d_aux_frames, float* d_aux_full, void* stream);

/* d_mel [B][feat][T] -> d_labels [B][S] (S = T*hop, may be NULL), d_wave [B][(T-1)*hop] float64 mu-law decoded,
 * truncated and faded exactly like fatchord_version.py:243-258 (may be NULL).  Needs T >= 21 when d_wave != NULL. */
int b200tts_wavernn_generate(b200tts_wavernn* ctx, const float* d_mel, int B, int T, const b200tts_rng* rng,
                             const b200tts_gen_opts* opts, int16_t* d_labels, double* d_wave, void* stream);

/* Mixture-of-logistics models (voc_mode = 'MOL').  create_mol takes the same cfg and weights as create, except that cfg.bits
 * is ignored and fc3 must be [30][fc_dims] (B200TTS_ESHAPE otherwise).  A MOL context is refused by _generate and
 * _generate_host, and a RAW context by _generate_mol.
 *
 * generate_mol: per row and step, with p = fc3 output (p[0..9] mixture logits, p[10..19] means, p[20..29] log-scales) and
 * uniforms u[0..10] in [1e-5, 1 - 1e-5], all in fp32 as the reference computes it:
 *     k = argmax_j (p[j] - log(-log(u[j])))          (first maximum)
 *     x = clamp(p[10+k] + exp(max(p[20+k], log(1e-14))) * (log(u[10]) - log(1 - u[10])), -1, 1)
 * x is the sample and the next step's input.  Noise: PHILOX draws u from Philox4x32-10 keyed by (seed, global utterance, step,
 * j = 0..2) (b200tts_philox_mol_uniform dumps it), EXT_UNIFORM reads d_q[S][B][11].
 *   d_samples   [B][S] float32 (may be NULL), [n_folds][fold_len] when folding
 *   d_teacher_x optional [B][S] (or folded): fed back instead of the sample
 *   d_wave      [B][(T-1)*hop] float64 of the samples (no mu-law: the reference turns it off for MOL), truncated and faded like
 *               RAW; the cross-faded wave when folding
 * opts: mu_law is ignored, d_teacher must be NULL, d_logits is [S][B][30], packed rows and kernel = TC are refused.  Kernels as
 * for RAW without the tensor cores: AUTO / GRID take the push kernel up to 32 rows and the wide grid above, UTTERANCE the
 * utterance kernel.  max_steps, fold_target/_overlap, d_utt_frames and d_utterance_ids work as for
 * RAW. */
int b200tts_wavernn_create_mol(b200tts_wavernn** out, int device, const b200tts_wavernn_cfg* cfg,
                               const b200tts_tensor* weights, int n_weights);
int b200tts_wavernn_generate_mol(b200tts_wavernn* ctx, const float* d_mel, int B, int T, const b200tts_rng* rng,
                                 const b200tts_gen_opts* opts, const float* d_teacher_x, float* d_samples, double* d_wave,
                                 void* stream);

/* n_folds and fold_len = target + 2*overlap of fold_with_overlap (fatchord_version.py:319-330) for a T-frame utterance. */
int b200tts_wavernn_fold_geometry(int T, int hop, int target, int overlap, int* n_folds, int* fold_len);

/* Same with HOST buffers: copies h_mel to the device, generates, copies labels / wave back, synchronises. */
int b200tts_wavernn_generate_host(b200tts_wavernn* ctx, const float* h_mel, int B, int T, const b200tts_rng* rng,
                                  const b200tts_gen_opts* opts, int16_t* h_labels, double* h_wave);

/* The Exp(1) noise the PHILOX mode uses for (utterance, step, class): d_q[n_steps][B][n_classes], steps step0 ..
 * step0 + n_steps - 1 with step0 >= 0 and step0 + n_steps <= 2^31 - 1 (else B200TTS_EINVAL, before any CUDA call).
 * Lets a test hand the production noise stream to the oracle. */
int b200tts_philox_exponential(int device, uint64_t seed, uint64_t utterance_offset, int B, int step0, int n_steps,
                               int n_classes, float* d_q, void* stream);

/* The uniforms the PHILOX mode of b200tts_wavernn_generate_mol draws for (utterance, step): d_u[n_steps][B][11], steps as
 * b200tts_philox_exponential takes them. */
int b200tts_philox_mol_uniform(int device, uint64_t seed, uint64_t utterance_offset, int B, int step0, int n_steps, float* d_u,
                               void* stream);

/* Number of kernel launches the library has issued on this context since creation (bench.py: gpu_launches). */
int64_t b200tts_wavernn_launch_count(const b200tts_wavernn* ctx);
/* Milliseconds (CUDA events on the launch stream) spent in the per-sample generation kernel by the most recent
 * generate call; blocks until that kernel has finished.  Negative on error. */
double b200tts_wavernn_last_kernel_ms(b200tts_wavernn* ctx);
/* Which step kernel the last generate call ran: 1 utterance, 2 wide grid, 3 push, 5 tensor-core pipeline, 6 push for a session
 * run, 7 tensor-core pipeline for a session run (0: none yet; 4 is no longer returned).  Instrumentation for bench.py's roofline; no reference counterpart. */
int b200tts_wavernn_last_kernel(const b200tts_wavernn* ctx);

/* Synchronises the device and reports whether the most recent generate call on this context completed: the persistent
 * generation kernels spin on data written by peer thread blocks and give up after ~2 s (B200TTS_ECUDA, the wave of that call
 * is filled with NaN).  The stream-ordered b200tts_wavernn_generate cannot report this itself; callers that hand audio to a
 * user (WaveRNN.generate <- fatchord_version.py:169, wavernn_gen.py:41) call this after their own synchronisation point. */
int b200tts_wavernn_check(b200tts_wavernn* ctx);

/* Generation sessions: one RAW utterance whose sample loop runs in pieces, so audio can be handed out after every run and the
 * set of utterances can change between runs.  A session runs on the kernel it was opened for: the push kernel (<= 32 sessions
 * per launch, any cut) or the tensor-core pipeline (<= 256 sessions per launch, cuts on frame boundaries).  The pieces of a
 * session, concatenated, are bit for bit the labels and wave of a one-shot b200tts_wavernn_generate of that mel with the same
 * seed and utterance id on the same kernel family (kernel = AUTO / GRID at <= 32 rows, or TC), however the steps are cut and
 * whichever sessions share a run.  Refused (B200TTS_EINVAL, before any CUDA call) for a MOL context and a model the push
 * kernel cannot run (rnn_dims = fc_dims = 512 on >= 128 SMs).
 *
 * session_open: a push session (session_open_kernel with kernel = B200TTS_KERNEL_AUTO).
 * session_open_kernel: d_mel [feat][T], T >= 21.  kernel: B200TTS_KERNEL_AUTO (push) or B200TTS_KERNEL_TC (tensor cores; refused
 *   where kernel=tc cannot run).  rng: PHILOX only, rng->utterance_offset is the utterance id (d_utterance_ids must be NULL).
 *   A one-row b200tts_wavernn_session_open_batch of the mel (layout B200TTS_MEL_FEAT_T, T_max = T; T x max(feat_dims,
 *   res_out_dims) must stay below 2^31): the conditioning tables are computed once, on `stream`, in three launches, into one
 *   allocation of the session's table and state.
 * session_destroy: null-safe; waits for the runs still queued.  b200tts_wavernn_destroy frees the sessions still open.
 * session_info: next step, steps of the utterance (T*hop) and samples of its wave ((T-1)*hop); any pointer may be NULL.
 * session_run: n distinct sessions of ctx advance by min(max_steps, steps - pos) steps each in one launch (a finished session
 *   takes part with 0 steps): 1..32 push sessions, or 1..256 tensor-core sessions with max_steps a multiple of hop_length, never
 *   a mix of the two.  d_labels [n][max_steps] int16 and d_wave [n][max_steps] float64 (either may
 *   be NULL) receive each session's steps from its old position: wave entry i is sample pos + i of the one-shot wave (0 from
 *   (T-1)*hop on) and entries past the session's count are 0.  Positions advance on the host at enqueue.  Poll timeouts are
 *   reported by b200tts_wavernn_check as for generate. */
typedef struct b200tts_wavernn_session b200tts_wavernn_session;
int b200tts_wavernn_session_open(b200tts_wavernn* ctx, const float* d_mel, int T, const b200tts_rng* rng, int mu_law,
                                 b200tts_wavernn_session** out, void* stream);
int b200tts_wavernn_session_open_kernel(b200tts_wavernn* ctx, const float* d_mel, int T, const b200tts_rng* rng, int mu_law,
                                        int kernel, b200tts_wavernn_session** out, void* stream);
void b200tts_wavernn_session_destroy(b200tts_wavernn_session* s);
int b200tts_wavernn_session_info(const b200tts_wavernn_session* s, int64_t* pos, int64_t* steps, int64_t* wave_len);
int b200tts_wavernn_session_run(b200tts_wavernn* ctx, b200tts_wavernn_session* const* s, int n, int max_steps,
                                int16_t* d_labels, double* d_wave, void* stream);
/* The most sessions one session_run takes on ctx: 256 where the tensor-core pipeline runs (kernel=tc), else 32. */
int b200tts_wavernn_session_max_rows(const b200tts_wavernn* ctx);

/* Batched open: n sessions in three launches whatever n is (mel preparation, MelResNet and the conditioning tables, each over the
 * rows' own frame counts), with no host copy of the mels; b200tts_wavernn_session_open_kernel is its one-row case.  Session i is
 * bit for bit the session b200tts_wavernn_session_open_kernel opens from row i's mel in [0, 1], zero-padded to max(h_frames[i], 21)
 * frames, with the same seed, id, mu_law and kernel: its pieces concatenate to that one-shot run.
 *   d_mel, layout B200TTS_MEL_FEAT_T: [n][feat][T_max], in [0, 1].
 *          layout B200TTS_MEL_TACO:   [n][T_max][feat], the Tacotron postnet output, mapped on the device with the float32
 *          statements of the reference's synthesizer: m = clip(m, -max_abs_value, max_abs_value), clip((m + a) / (2a), 0, 1).
 *   h_frames [n] (host): frames of each row, 1..T_max; rows shorter than 21 frames get zero frames (in [0, 1]) up to 21.
 *   n: 1..b200tts_wavernn_session_max_rows(ctx).  rng: PHILOX; session i's utterance id is d_utterance_ids[i] (device memory,
 *   read back in stream order, which synchronises `stream`) or utterance_offset + i.  kernel: B200TTS_KERNEL_AUTO (push) or
 *   B200TTS_KERNEL_TC.  out[n] receives the sessions, on success only.
 * The sessions of one call share one allocation, freed when the last of them is destroyed.  Bad arguments return B200TTS_EINVAL
 * before any CUDA call, with the refusals of session_open_kernel. */
enum { B200TTS_MEL_FEAT_T = 0, B200TTS_MEL_TACO = 1 };
int b200tts_wavernn_session_open_batch(b200tts_wavernn* ctx, const float* d_mel, int layout, float max_abs_value,
                                       const int32_t* h_frames, int n, int T_max, const b200tts_rng* rng, int mu_law, int kernel,
                                       b200tts_wavernn_session** out, void* stream);

/* Measured fp32 CUDA-core ceiling of `device` in TFLOP/s (register-only packed FFMA2 loop on every SM): the denominator
 * of bench.py's FLOP-form roofline. */
int b200tts_debug_fp32_peak(int device, double* tflops);

/* ------------------------------------------------------------------------------------------------------------------
 * Tacotron-2 forward-attention decoder loop (secondary hot path).
 *   b200tts_taco_create  <- the decoder-side variables tf.train.Saver restores (tacotron_synthesize.py:76-78), by their
 *                           checkpoint names minus the "Tacotron_model/inference/" prefix
 *   b200tts_taco_decode  <- dynamic_decode(CustomDecoder(TacotronDecoderCell, TacoTestHelper)) tacotron/models/tacotron.py:99-103
 *                           = Architecture_wrappers.py:175-218 + attention.py:119-231 + modules.py:114-142,240-251,304,334-342
 *                           + custom_decoder.py:105-135 + helpers.py:36-66
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct {
  int32_t num_mels;         /* 80   tacotron_hparams.py num_mels                */
  int32_t prenet_units;     /* 256  prenet_layers = [256, 256]                  */
  int32_t lstm_units;       /* 256  decoder_lstm_units (checkpoint kernels are [768+256,1024] and [512,1024]) */
  int32_t enc_dim;          /* 512  2 * encoder_lstm_units                      */
  int32_t attn_dim;         /* 128  attention_dim                               */
  int32_t attn_filters;     /* 32   attention_filters (at most 32: location features of 512 tokens x 32 fill the decoder's buffer) */
  int32_t attn_kernel;      /* 31   attention_kernel                            */
  float zoneout;            /* 0.1  tacotron_zoneout_rate                       */
} b200tts_taco_cfg;

enum { B200TTS_TACO_DROPOUT_PHILOX = 0, B200TTS_TACO_DROPOUT_EXT = 1 };
typedef struct {
  int32_t mode;
  uint64_t seed;
  uint64_t utterance_offset;
  const uint8_t* d_masks;   /* EXT: keep flags [B][max_steps][2][prenet_units]; prenet dropout is ON at inference (modules.py:249) */
} b200tts_taco_dropout;

typedef struct b200tts_taco b200tts_taco;

int b200tts_taco_create(b200tts_taco** out, int device, const b200tts_taco_cfg* cfg, const b200tts_tensor* weights, int n_weights);
void b200tts_taco_destroy(b200tts_taco* ctx);

/* d_memory [B][Tx_max][enc_dim] encoder outputs, d_lengths [B] (<= Tx_max <= 512).  Every sentence runs until its own
 * stop token exceeds 0.5 or max_steps.  window != 0 enables the inference attention window of forward_attention.py:171-215.
 * Outputs: d_frames [B][max_steps][num_mels] raw decoder outputs (before the clip of tacotron.py:111), d_stop [B][max_steps],
 * d_align [B][max_steps][Tx_max] (may be NULL), d_nsteps [B] = frames produced (the last one is the frame whose stop fired). */
int b200tts_taco_decode(b200tts_taco* ctx, const float* d_memory, const int32_t* d_lengths, int B, int Tx_max,
                        const b200tts_taco_dropout* dropout, int max_steps, int window, float* d_frames, float* d_stop,
                        float* d_align, int32_t* d_nsteps, void* stream);

/* Parity aid (teacher forcing): the same loop, but the COMPLETE recurrent state is reloaded from d_states before every step and
 * the stop rule is ignored, so exactly n_steps steps run.  d_states [B][n_steps][b200tts_taco_state_floats(ctx, Tx_max)], one
 * record per step:  x[num_mels] | context[enc_dim] | c1 | h1 | c2 | h2 [lstm_units each] | mu | max_attention | pos_rec | 0 |
 * cumulated alignments[Tx_max] | alpha[Tx_max]   (the loop state of Architecture_wrappers.py:136-173 + attention.py:112-117).
 * Lets a test compare EVERY step of a long, numerically chaotic run against the oracle fed with the oracle's own state. */
int b200tts_taco_state_floats(const b200tts_taco* ctx, int Tx_max);
int b200tts_taco_decode_forced(b200tts_taco* ctx, const float* d_memory, const int32_t* d_lengths, int B, int Tx_max,
                               const b200tts_taco_dropout* dropout, int n_steps, int window, const float* d_states,
                               float* d_frames, float* d_stop, float* d_align, int32_t* d_nsteps, void* stream);

/* Speaking-rate control: the forward-attention speed bias of attention.py:163-165 / forward_attention.py:163-165 (the branch the
 * reference ships switched off with `and False`), one bias per sentence.  Sentence b's recursion (attention.py:167) uses
 *   mu' = clip(mu + h_mu_bias[b], 0, 1)      (fp32 add rounded once, then tf.clip_by_value: min with 1, max with 0)
 * instead of mu at every step, the first (mu = 0.5) included; the carried mu, the fresh sigmoid of [context | query]
 * (attention.py:229), stays unbiased, and the window (window != 0) acts on the biased recursion.  Positive biases move attention
 * on sooner: faster speech, shorter mels; a bias of 0 gives exactly b200tts_taco_decode.  h_mu_bias [B] host floats, each finite
 * and in [-1, 1] (anything else returns B200TTS_EINVAL before any launch); the library uploads them on `stream`.  d_states NULL
 * is a free run; otherwise it holds the teacher-forcing records of b200tts_taco_decode_forced with n_steps = max_steps (their mu
 * is the unbiased one).  Kernel selection, outputs and the remaining arguments are those of b200tts_taco_decode. */
int b200tts_taco_decode_biased(b200tts_taco* ctx, const float* d_memory, const int32_t* d_lengths, int B, int Tx_max,
                               const b200tts_taco_dropout* dropout, int max_steps, int window, const float* h_mu_bias,
                               const float* d_states, float* d_frames, float* d_stop, float* d_align, int32_t* d_nsteps, void* stream);

/* Ground-truth-aligned (GTA) decoding, the teacher-forced loop of wavernn_preprocess.py (TacoTrainingHelper, helpers.py:111-151):
 * the step-t input is d_targets[b][t-1] (the zero GO frame at t = 0) instead of the previous output, and exactly
 * clamp(d_target_lengths[b], 0, Ty_max) steps run.  No stop rule, no inference window (the reference builds this attention with
 * is_training = True), no stop output; prenet dropout stays on and draws the same stream as b200tts_taco_decode, so fed a free
 * run's own raw frames with the same dropout descriptor this replays that run.  One thread block per sentence at every B.
 * d_targets [B][Ty_max][num_mels] used as given (the reference clips them to +-max_abs_value first); d_frames
 * [B][Ty_max][num_mels] raw decoder outputs; d_align [B][Ty_max][Tx_max] or NULL; EXT masks [B][Ty_max][2][prenet_units].
 * Rows at or beyond a sentence's step count are left untouched.  Bad arguments return B200TTS_EINVAL and launch nothing. */
int b200tts_taco_decode_gta(b200tts_taco* ctx, const float* d_memory, const int32_t* d_lengths, int B, int Tx_max,
                            const b200tts_taco_dropout* dropout, const float* d_targets, const int32_t* d_target_lengths,
                            int Ty_max, float* d_frames, float* d_align, void* stream);

/* Run-once neighbours of the decoder loop (available when b200tts_taco_create also received the encoder / postnet
 * variables):
 *   b200tts_taco_encode   <- embedding lookup + EncoderConvolutions + EncoderRNN   tacotron.py:44-57, modules.py:145-217
 *   b200tts_taco_postnet  <- clip + Postnet + postnet_projection + residual + clip  tacotron.py:111-129, modules.py:345-376
 * d_ids [B][Tx_max] symbol ids (tacotron/utils/text.py:18-31; each id below its sentence's length must be < the vocabulary size),
 * d_lengths [B], d_memory [B][Tx_max][enc_dim] (rows >= length are zero);
 * d_frames [B][max_steps][num_mels] raw decoder outputs, d_nsteps [B], d_mel [B][max_steps][num_mels] (rows >= nsteps untouched).
 * Like the decoders, both clamp each length to [0, Tx_max] / [0, max_steps]: a length <= 0 is an empty sentence. */
int b200tts_taco_encode(b200tts_taco* ctx, const int32_t* d_ids, const int32_t* d_lengths, int B, int Tx_max, float* d_memory,
                        void* stream);
int b200tts_taco_postnet(b200tts_taco* ctx, const float* d_frames, const int32_t* d_nsteps, int B, int max_steps, float* d_mel,
                         void* stream);

/* The reference synthesizer's cut of a free run (tacotron_synthesize.py:104-105): d_len[b] = the first step t < nsteps[b] whose
 * np.round(stop) is 1, i.e. stop > 0.5 (np.round(0.5) is 0), else nsteps[b].  d_stop [B][max_steps], d_nsteps [B] as
 * b200tts_taco_decode writes them; nsteps is clamped to max_steps, and a negative nsteps (a failed decode) is passed through. */
int b200tts_taco_target_lengths(const float* d_stop, const int32_t* d_nsteps, int B, int max_steps, int32_t* d_len, void* stream);

/* Decoder sessions: free runs decoded in slices of at most k steps, so a service can bound the decoder work it does between two
 * vocoder runs, and decodes opened at different times can share a slice (continuous batching).  The frames, stop values and step
 * count of a session, however its steps are cut and whichever sessions share its slices, are bit for bit those of
 * b200tts_taco_decode_biased with B >= 2 (taco_decoder_kernel, one thread block per sentence) on the same encoder output, with the
 * same seed, utterance id, bias, window flag and max_steps.  A slice is one launch of 1..128 thread blocks: one wave of the SMs.
 * Refusals return B200TTS_EINVAL before any CUDA call.
 *
 * session_open_batch: n (1..128) sessions from d_memory [n][Tx_max][enc_dim] (Tx_max <= 512) with h_lengths [n] (host, each
 *   1..Tx_max).  dropout: PHILOX only (EXT masks are refused); session i's utterance id is h_ids[i] (host; NULL: utterance_offset
 *   + i).  h_mu_bias [n] host speaking-rate biases, each finite and in [-1, 1] (NULL: 0).  The memory is copied and its keys
 *   computed once, on `stream`, into memory the sessions own; each starts at position 0.  The sessions of one call share one
 *   allocation, freed when the last of them is destroyed.  out[n] receives the sessions, on success only.
 * session_destroy: null-safe; waits for the work still queued.  b200tts_taco_destroy frees the sessions still open.
 * session_info: steps decoded so far (the position of the next slice), whether the decode is done (its stop token fired, or
 *   it reached max_steps), and its max_steps; any pointer may be NULL.
 * session_run: n (1..128) distinct sessions of ctx advance by up to max_steps (>= 1) steps each in one launch; a session stops
 *   early at the step whose stop token exceeds 0.5, and a finished session takes part with 0 steps.  Where a decode stops is known
 *   on the device only, so the call waits for the slice (it synchronises `stream`) and returns with every position updated.
 * session_outputs: the decoded steps of n (1..128) sessions of one context in the batch layout b200tts_taco_decode writes, ready
 *   for b200tts_taco_postnet and b200tts_taco_target_lengths: d_frames [n][T_max][num_mels], d_stop [n][T_max] (zeros from each
 *   session's position on) and d_nsteps [n] = the positions.  T_max must be at least every position.  One launch on `stream`. */
typedef struct b200tts_taco_session b200tts_taco_session;
int b200tts_taco_session_open_batch(b200tts_taco* ctx, const float* d_memory, const int32_t* h_lengths, int n, int Tx_max,
                                    const b200tts_taco_dropout* dropout, const uint64_t* h_ids, int max_steps, int window,
                                    const float* h_mu_bias, b200tts_taco_session** out, void* stream);
void b200tts_taco_session_destroy(b200tts_taco_session* s);
int b200tts_taco_session_info(const b200tts_taco_session* s, int32_t* pos, int32_t* done, int32_t* max_steps);
int b200tts_taco_session_run(b200tts_taco* ctx, b200tts_taco_session* const* s, int n, int max_steps, void* stream);
int b200tts_taco_session_outputs(b200tts_taco_session* const* s, int n, int T_max, float* d_frames, float* d_stop,
                                 int32_t* d_nsteps, void* stream);

/* The keep flags the PHILOX dropout mode draws: d_masks [B][steps][2][prenet_units], prenet_units a multiple of 4 as
 * b200tts_taco_create requires. */
int b200tts_taco_philox_masks(int device, uint64_t seed, uint64_t utterance_offset, int B, int steps, int prenet_units,
                              uint8_t* d_masks, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Griffin-Lim mel inversion (the preview wav of tacotron_synthesize.py:110-112).
 *   b200tts_griffin_lim  <- audio.inv_mel_spectrogram(mel.T, hparams)  tacotron/datasets/audio.py:122-137
 *                           = _denormalize :297-309, _db_to_amp :277-278, _mel_to_linear :256-260, _griffin_lim :176-186,
 *                           _stft / _istft (librosa 0.7.2 stft / istft) :203-210, inv_preemphasis :52-55
 * Symmetric mels clipped to +-max_abs_value (signal_normalization, allow_clipping_in_normalization) and librosa's stft with
 * center=True and constant padding are assumed.  T frames give exactly hop * (T - 1) samples.
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct {
  int32_t n_fft;            /* 2048 (the only size implemented)  */
  int32_t hop_size;         /* 275                               */
  int32_t win_size;         /* 1100 (<= n_fft), periodic Hann    */
  int32_t num_mels;         /* 80 (<= 128)                       */
  float max_abs_value;      /* 4                                 */
  float min_level_db;       /* -100                              */
  float ref_level_db;       /* 20                                */
  float magnitude_power;    /* 2                                 */
  float power;              /* 1.5                               */
  float preemphasis;        /* 0.97; 0 when preemphasize is off  */
} b200tts_gl_cfg;

enum { B200TTS_GL_PHASE_PHILOX = 0, B200TTS_GL_PHASE_EXT = 1 };
/* Initial phase e^{2 pi i u} of _griffin_lim (:181, np.random.rand): u from Philox4x32-10 keyed by (seed, utterance_offset + row,
 * frame, bin), or read from d_u[B][T_max][n_fft/2 + 1] (EXT; tests share the phase with the oracle). */
typedef struct {
  int32_t mode;
  uint64_t seed;
  uint64_t utterance_offset;
  const float* d_u;
} b200tts_gl_phase;

typedef struct b200tts_gl b200tts_gl;

/* h_inv_mel_basis [n_fft/2 + 1][num_mels]: pinv of the mel filterbank (librosa.filters.mel(sample_rate, n_fft, num_mels, fmin,
 * fmax), _build_mel_basis :268-271), computed by the caller (in float64) and rounded to fp32. */
int b200tts_gl_create(b200tts_gl** out, int device, const b200tts_gl_cfg* cfg, const float* h_inv_mel_basis);
void b200tts_gl_destroy(b200tts_gl* ctx);

/* d_mel [B][T_max][num_mels] (frames x mels, the decoder's layout) -> d_wave [B][hop * (T_max - 1)] float32 after n_iters
 * iterations.  d_frames [B] (may be NULL = T_max for every row): true frame count of each row of a zero-padded ragged batch;
 * row b is then computed exactly as a stand-alone run of d_frames[b] frames and is zero from hop * (d_frames[b] - 1) on (values
 * above T_max count as T_max; rows with fewer than 2 frames come back all zero).  d_u_out [B][T_max][n_fft/2 + 1] (may be NULL):
 * the phase, as angle / 2 pi mod 1, of the last stft (of `init` when n_iters = 0) -- with init = EXT and n_iters = 1 this
 * teacher-forces a single iteration.  Rows beyond a row's frame count are left untouched in d_u_out. */
int b200tts_griffin_lim(b200tts_gl* ctx, const float* d_mel, const int32_t* d_frames, int B, int T_max, const b200tts_gl_phase* init,
                        int n_iters, float* d_wave, float* d_u_out, void* stream);

/* The uniforms the PHILOX phase mode draws: d_u[B][T][n_bins]. */
int b200tts_gl_philox_uniform(int device, uint64_t seed, uint64_t utterance_offset, int B, int T, int n_bins, float* d_u, void* stream);

/* Number of kernel launches issued on this context since creation. */
int64_t b200tts_gl_launch_count(const b200tts_gl* ctx);

/* ------------------------------------------------------------------------------------------------------------------
 * Mel analysis (the reference's feature extraction, tacotron/datasets/preprocessor.py:52-121 _process_utterance_v1).
 *   flags = 0                               <- audio.melspectrogram(wav, hparams)       tacotron/datasets/audio.py:95-102
 *   flags = TRIM | PREEMPHASIS | RESCALE    <- _process_utterance_v1 without the file I/O: trim_silence :71-77 (librosa 0.7.2
 *                                              effects.trim), preemphasis :47-50, rescale preprocessor.py:70-72,
 *                                              melspectrogram of the pre-emphasised signal, and the padded audio :100-111
 * librosa's stft with center=True and constant padding, symmetric clipped normalisation.  A signal of n samples gives
 * T = 1 + n / hop frames.  The float parameters preemphasis and rescaling_max enter the fp64 steps as the shortest decimal
 * that rounds to them (0.97f -> 0.97), which is what a Python caller passed.
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct {
  int32_t n_fft;            /* 2048 (the only size implemented)       */
  int32_t hop_size;         /* 275                                    */
  int32_t win_size;         /* 1100 (<= n_fft), periodic Hann         */
  int32_t num_mels;         /* 80 (<= 128)                            */
  float max_abs_value;      /* 4                                      */
  float min_level_db;       /* -100                                   */
  float ref_level_db;       /* 20                                     */
  float magnitude_power;    /* 2                                      */
  float preemphasis;        /* 0.97                                   */
  float rescaling_max;      /* 0.999                                  */
  int32_t trim_fft_size;    /* 2048: trim frame length                */
  int32_t trim_hop_size;    /* 512                                    */
  float trim_top_db;        /* 25                                     */
} b200tts_mel_cfg;

enum { B200TTS_MEL_TRIM = 1, B200TTS_MEL_PREEMPHASIS = 2, B200TTS_MEL_RESCALE = 4 };

typedef struct b200tts_mel b200tts_mel;

/* h_mel_basis [num_mels][n_fft/2 + 1]: the fp32 Slaney filterbank (librosa.filters.mel(sample_rate, n_fft, num_mels, fmin,
 * fmax), _build_mel_basis :268-271), computed by the caller. */
int b200tts_mel_create(b200tts_mel** out, int device, const b200tts_mel_cfg* cfg, const float* h_mel_basis);
void b200tts_mel_destroy(b200tts_mel* ctx);

/* d_wav [B][L_max] float32 signals, d_len [B] their lengths (clamped to [0, L_max]).  Outputs, with T_max = 1 + L_max / hop:
 *   d_mel    [B][T_max][num_mels]  frames x mels, zero beyond each row's frame count
 *   d_frames [B]                   frame count T of each row (0 for a row that TRIM empties, a row shorter than
 *                                  trim_fft_size when trimming, and an empty row)
 *   d_bounds [B][2] (may be NULL)  [start, end) of the kept samples (the whole row without TRIM)
 *   d_audio  [B][T_max * hop] (may be NULL)  the (rescaled) kept samples, zero-padded from end - start on
 * Each row is computed exactly as a stand-alone run of that row.  TRIM: a frame is non-silent when its mean square is within
 * trim_top_db of the loudest frame's; a row whose frames are all exactly zero has none. */
int b200tts_mel_analyze(b200tts_mel* ctx, const float* d_wav, const int32_t* d_len, int B, int L_max, int flags, float* d_mel,
                        int32_t* d_frames, int32_t* d_bounds, float* d_audio, void* stream);

/* Number of kernel launches issued on this context since creation. */
int64_t b200tts_mel_launch_count(const b200tts_mel* ctx);

/* ------------------------------------------------------------------------------------------------------------------
 * Resampling (what the reference's audio.load_wav does to a recording at another rate: librosa 0.7.2
 * core.load(path, sr=22050) -> core.resample(y, sr_native, sr, res_type='kaiser_best') = resampy 0.2.2 resample, then
 * util.fix_length).  One context per rate pair.  With ratio = (double)sr_new / sr_orig, a row of n samples gives
 * int(n * ratio) resampled samples (resampy's length; the caller refuses rows where that is 0, as resampy does), zero-padded
 * to ceil(n * ratio) (librosa's length).  The arithmetic is resampy's, bit for bit: fp64 weights and products, each partial
 * sum rounded to fp32, the time register a sequential fp64 sum.
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct b200tts_resampler b200tts_resampler;

/* h_half_window [nwin] float64: the filter's right half (resampy's kaiser_best: nwin = 64 * 512 + 1, num_table = 512),
 * unscaled; the context multiplies it by ratio when ratio < 1 and tabulates its differences, as resampy does.  sr_orig ==
 * sr_new is refused (there is nothing to compute: librosa returns the input). */
int b200tts_resample_create(b200tts_resampler** out, int device, int sr_orig, int sr_new, const double* h_half_window, int nwin,
                            int num_table);
void b200tts_resample_destroy(b200tts_resampler* ctx);

/* d_x [B][L_max] float32 signals, d_len [B] their lengths (clamped to [0, L_max]).  Outputs, with Y_max = ceil(L_max * ratio):
 *   d_y       [B][Y_max]  the resampled rows, zero from int(len * ratio) on
 *   d_out_len [B]         ceil(len * ratio)
 * int(L_max * ratio) must be >= 1.  The first call that needs a longer time register than the context holds extends it on the
 * host and synchronises `stream`.  Each row is computed exactly as a stand-alone run of that row. */
int b200tts_resample(b200tts_resampler* ctx, const float* d_x, const int32_t* d_len, int B, int L_max, float* d_y,
                     int32_t* d_out_len, void* stream);

/* Number of kernel launches issued on this context since creation. */
int64_t b200tts_resample_launch_count(const b200tts_resampler* ctx);

/* Debug aid: mean SM cycles per CTA spent in {compute, barrier} of each of the 6 phases of the last grid-kernel
 * launch; only recorded when the environment variable B200TTS_GRID_PROF is set while generating. */
int b200tts_wavernn_debug_phase_cycles(b200tts_wavernn* ctx, double* out12);

#ifdef __cplusplus
}
#endif
#endif /* B200TTS_H_ */
