// WaveRNN per-sample recurrence, "push" kernel: the small-batch (B <= 32 rows per GPU) form of the weight-stationary grid.
//
// Same decomposition as wavernn_grid.cuh -- 128 co-resident CTAs (cooperative launch), CTA c keeps the rows of every layer
// that produce hidden units / fc rows [4c, 4c+4) and classes [8c, 8c+8) in shared memory for the whole launch -- but the
// five exchanges of a sample step (reference loop wavernn/models/fatchord_version.py:201-237) no longer go through a
// grid barrier followed by a load of the activations.  At B <= 32 a step is pure latency, and on the GPU this kernel was
// first written for the barrier round (bar.sync + red.release + spin on ld.acquire + bar.sync) plus the L2 pull after it
// took about three quarters of a step of the grid kernel.  Here:
//
//   * FLAG-IN-DATA exchange.  Every exchanged activation vector lives in L2 as [producer CTA][row][4 units] fp32, two
//     parity copies, pre-filled with a sentinel bit pattern (0xFFFFFFFF, a NaN no arithmetic here can produce).  A
//     producer simply stores its 4 x G values; a consumer thread loads the float4 it needs straight into registers with
//     ld.relaxed.gpu and re-polls until none of the four words is the sentinel -- the data IS the flag, one L2 round trip
//     instead of fence + flag + poll + load.  A producer re-arms the OTHER parity copy of its own entries (sentinel stores +
//     __threadfence) right after it has seen every CTA's winner of the previous step, i.e. when every consumer of that
//     copy is provably done and long before anybody can poll it again (proof at `rearm` below).
//   * The sampled label travels the same way: every CTA publishes its local Gumbel-max winner per row as one 64-bit word
//     (ordered key | inverted class | 22-bit step tag -- 8-byte stores are single-copy atomic) and every CTA reduces the
//     128 winners itself; no atomics, no barrier.
//   * No shared-memory staging: thread (row lane, k queue) loads exactly the float4s it multiplies (G/4 per vector), all
//     rows of the phase are accumulated in registers, k queues are reduced by shuffles + one 16-warp pass through shared
//     memory.
//   * CONDITIONING HOISTED (SURVEY 7.1-5): the 112 conditioning columns of the I layer / GRU-1 and the 32 aux columns of
//     GRU-2, fc1, fc2 never enter the serial path.  push_cond_table_kernel computes, once per utterance and FRAME,
//     W.mel[f] (FIR linearity: W.(sum_j fir[ph][j] mel[f_j]) = sum_j fir[ph][j] (W.mel[f_j])) and W.aux[f] + bias for
//     the 52 conditioned rows of every CTA; the kernel combines <= 6 table rows per output row for step t+1 while it
//     waits for fc2's exchange of step t.  This also removes the [S][80][B] sample-rate mel buffer of the round-1 path.
//   * The two recurrent projections W_hh1.h1(t), W_hh2.h2(t) (42 % of the MACs) do not depend on the sample drawn at
//     step t: they run in the shadow of the NEXT exchange (after GRU-2 / fc1 have published) and are consumed one step later.
//
// Per step and CTA:  P01 winners(t-1) -> x, GRU-1 gate math (all matrix work precomputed) -> publish h1, x1
//                    P2  x1 -> W_ih2 (12 x 512) -> gate math -> publish h2, x2      | shadow: W_hh1.h1(t)
//                    P3  x2 -> fc1 (4 x 512)  -> publish f1                          | shadow: W_hh2.h2(t)
//                    P4  f1 -> fc2 (4 x 512)  -> publish f2                          | shadow: conditioning of step t+1
//                    P5  f2 -> fc3 (8 x 512)  -> Gumbel-max over the CTA's 8 classes -> publish winner
#pragma once
#include "common.cuh"
#include "exchange.cuh"
#include "wavernn_upsample.cuh"
#include "wavernn_grid.cuh"

namespace b200tts {

constexpr int kPushThreads = 512;
constexpr int kPushWarps = kPushThreads / 32;
constexpr int kPushMaxRows = 32;    // rows of the widest variant, wavernn_push_kernel<32>; larger batches run other kernels
constexpr int kPushCondRows = 52;   // per CTA and frame: 16 mel projections | 16 + 12 + 4 + 4 aux projections (+ bias)
constexpr int kPushVecs = 6;        // h1, x1, h2, x2, f1, f2
enum { PV_H1 = 0, PV_X1, PV_H2, PV_X2, PV_F1, PV_F2 };

struct PushModel {          // layout of one CTA's weight blob (offsets in floats, 16-byte aligned)
  int ncta, R, F, NC;
  int ohh1, oih2, ohh2;     // [12][R]  row = gate*4 + unit ; W_ih2 without its aux columns
  int ofc1, ofc2, ofc3;     // [4][R], [4][F], [8][F]
  int oAx;                  // [16]: coefficient of the fed-back sample x in the 4 I rows and the 12 folded GRU-1 rows
  int obhh1, obhh2, obfc3;  // [12], [12], [8]
  int blob;
  int ok;
};

struct PushArgs {
  const float* wblob;            // [ncta][blob]
  float* vec;                    // [6][2][ncta][G][4]   exchanged activations (sentinel pre-filled)
  unsigned long long* best;      // [ncta][G]            winners, tagged with the step
  int* error;                    // set non-zero when a poll timed out
  const float* tab;              // [n_src][T+1][ncta][52] conditioning tables (push_cond_table_kernel)
  const float* fir;              // [hop][NT] composite polyphase FIR of the upsampling network
  int NT;
  int B, S, T, hop, steps;
  int reserved;                  // unused; it keeps the offsets of the fields below, and ptxas's register allocation of the
                                 // push kernels follows those offsets
  int row_stride;                // 0: row u is utterance u.  > 0 (fold-with-overlap): row u = samples [u*row_stride, ...) of utterance 0
  int S_src;                     // samples of the source utterance (conditioning is ZERO beyond, fatchord_version.py:315-317)
  int rng_mode;
  unsigned long long seed, utt_offset;
  const unsigned long long* utt_ids;   // optional [B]: global utterance index of every row (overrides utt_offset + row)
  const float* q;                // [S][B][NC]
  const int16_t* teacher;        // [B][S]
  float* logits_out;             // [S][B][NC]
  int16_t* labels;               // [B][S]
  long long* prof;               // optional [ncta][16] cycle counters of thread 0
  // PACKED rows (ragged sets, pipeline.py): row u runs a QUEUE of utterances back to back -- segment k of row u is utterance
  // pack_utt[u*pack_segs + k] from step pack_start[u*(pack_segs+1) + k] (next entry = its end; utt < 0 = no more work) -- and
  // restarts from the zero state at every segment start, so every utterance gets exactly the arithmetic of a stand-alone run.
  // B then counts UTTERANCES (labels [B][S], tables [B][T+1]...), the kernel runs G rows for `steps` lock-steps.
  const int* pack_utt;           // [pack_rows][pack_segs]
  const int* pack_start;         // [pack_rows][pack_segs + 1]
  int pack_segs, pack_rows;      // kernel rows >= pack_rows are idle
};

// GENERATION SESSIONS (b200tts_wavernn_session_*, wavernn_push_session_kernel): row u of a launch resumes session u at its
// position `pos` and runs `n` steps, a segment from lock-step 0 to n whose step within the utterance is pos + t; then it is idle.
// At the end of its run a row saves what makes its next step exactly the one-shot run's next step: both GRU states, the two
// recurrent projections W_hh . h as this CTA reduced them for the next step (12 rows per CTA) and the last label (the next x).
// Saving the reduced projections instead of recomputing them keeps the summation order, hence the bits.  Needs R = 512 and
// 128 CTAs (pm.ok).
constexpr int kSessH1 = 0, kSessH2 = 512, kSessGh1 = 1024, kSessGh2 = kSessGh1 + 128 * 12, kSessLabel = kSessGh2 + 128 * 12;
constexpr int kSessStateFloats = kSessLabel + 4;
struct SessRow {
  const float* tab;                 // [T+1][ncta][52] the session's conditioning tables
  float* state;                     // [kSessStateFloats]; the label is stored as an int
  unsigned long long seed, id;      // Philox key of the one-shot run: (seed, utterance id, step within the utterance)
  int T, pos, n, mu_law;            // frames; first step of this run; steps of this run (0: idle row); wave decoding
};
struct SessIO {                     // passed by value, next to PushArgs (whose field offsets are left alone)
  SessRow row[kPushMaxRows];
  int16_t* labels;                  // [rows][ld]: the label of step pos + i of row u at labels[u * ld + i]
  int ld;
};

struct PushRowState {            // per-row bookkeeping in shared memory (normal mode: row u == utterance u from step 0, forever)
  // current segment: utterance (-1 idle), first step, first step of the NEXT segment, index
  int utt[kPushMaxRows], t0[kPushMaxRows], end[kPushMaxRows], k[kPushMaxRows];
  int putt[kPushMaxRows], pn[kPushMaxRows];   // (utterance, local step) the row was at in the PREVIOUS step (whose winner P01 collects)
  int rst[kPushMaxRows];                      // the current step is the first of a segment: x = 0, h1 = h2 = 0
};
// (utterance, local step) of row u at step t+1, seen from step t
__device__ __forceinline__ void push_row_next(const PushArgs& A, const PushRowState& R, int u, int t1, int& utt, int& n) {
  if (t1 < R.end[u]) { utt = R.utt[u]; n = t1 - R.t0[u]; return; }
  const int k1 = R.k[u] + 1;
  utt = (A.pack_utt && u < A.pack_rows && k1 < A.pack_segs) ? A.pack_utt[u * A.pack_segs + k1] : -1;
  n = t1 - R.end[u];
}

// ---- exchange protocol ------------------------------------------------------------------------------------------
// Compared in isolation on the previous GPU (tools/exchange_bench.cu; all-to-all exchange of a [128][G][4] vector by 128
// CTAs): every thread spinning on its own entries beat a counter barrier followed by loads and a canary warp releasing the
// block through a barrier -- detection and delivery are the same L2 round trip.  Not re-measured on the H100.  Every
// thread issues ALL its loads first and re-polls only what still carries a sentinel.
template <int NL>
__device__ __forceinline__ void poll_entries(const float* base, const int (&off)[NL], float4 (&a)[NL], PollGuard& g) {
#pragma unroll
  for (int i = 0; i < NL; ++i) a[i] = ld_relaxed_f4(base + off[i]);
  // Then each entry in turn until it carries no sentinel.  (Written as one loop per entry: the earlier form with a bit mask
  // of pending entries was compiled by nvcc 12.9 for sm_90a, at two entries per thread, into a test that skipped the re-poll
  // exactly when BOTH entries were still pending -- stale sentinels went on as data, without a timeout.)
  g.begin();
#pragma unroll
  for (int i = 0; i < NL; ++i) {
    while (!f4_ready(a[i]) && !g.aborted) {
      if (g.expired()) break;
      a[i] = ld_relaxed_f4(base + off[i]);
    }
  }
}

// winner word: ordered-float key (32) | 1023 - class (10) | step tag (22)
__device__ __forceinline__ unsigned long long push_pack(float key, uint32_t cls, uint32_t tag) {
  uint32_t u = __float_as_uint(key);
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ((unsigned long long)u << 32) | ((unsigned long long)(1023u - cls) << 22) | (unsigned long long)(tag & 0x3FFFFFu);
}
__device__ __forceinline__ uint32_t push_cls(unsigned long long p) { return 1023u - (uint32_t)((p >> 22) & 1023u); }

template <int G> struct PushTraits {
  static constexpr int UT = (G >= 16) ? 2 : 1;             // rows per thread in the GEMMs
  static constexpr int NU = G / UT;                        // row lanes
  static constexpr int NKQ = kPushThreads / NU;            // k queues
  static constexpr int NKB = 128 / NKQ;                    // producer blocks (float4 columns) per thread and row
  static constexpr int NL = NKB * UT;                      // float4 loads per thread and vector = G/4
  static constexpr int kPartFloats = kPushWarps * 16 * G;        // up to 16 rows per pass (W_ih2 12 + fc1 4 on x1)
  static_assert(G <= kPushMaxRows && NU >= 8 && NU <= 32 && NKQ * NKB == 128 && NL * 4 == G && (32 / NU) * NKB == 8 && (NKB == 2 || NKB == 4),
                "mapping");
  // shared memory after the weight blob (floats)
  static constexpr int oPartX = 0;
  static constexpr int oPartY = oPartX + kPartFloats;
  static constexpr int oCond = oPartY + kPartFloats;       // [2][36][G]
  static constexpr int oGh1 = oCond + 2 * 36 * G;          // [12][G]
  static constexpr int oGh2 = oGh1 + 12 * G;               // [12][G]
  static constexpr int oSmax = oGh2 + 12 * G;              // u64 [16][G]
  static constexpr int oKeys = oSmax + 2 * kPushWarps * G; // u64 [8][G]
  static constexpr int oXs = oKeys + 2 * 8 * G;            // [G] fed-back sample
  static constexpr int oFir = oXs + ((G + 3) & ~3);        // [hop*NT]
  static constexpr int scratch_floats(int hop, int NT) { return oFir + ((hop * NT + 3) & ~3); }
};

// ---- one GEMM pass over this thread's NKB producer blocks x UT rows.  The 128 four-term dot products of an output (one
//      per producer block kb) are combined in ONE fixed order for every G: pairwise by bit 0, 1, 2 of kb (inside the thread
//      while it owns the pair, by warp shuffle otherwise; 8 consecutive kb per warp for every G), then the 16 warps in
//      sequence (push_part_sum).  A row's result is therefore bit-identical whatever batch it is generated in (G = 8 ... 32),
//      which is what lets N ranks reproduce the single-rank labels exactly.  Partials to part[(warp*ROWS + r)*G + u]. -------
template <int G>
__device__ __forceinline__ void push_load(const float* vecbase, float4 (&a)[PushTraits<G>::NL], int ul, int kq, PollGuard& pg) {
  using PT = PushTraits<G>;
  constexpr int UT = PT::UT, NU = PT::NU, NKB = PT::NKB, NL = PT::NL;
  int off[NL];
#pragma unroll
  for (int i = 0; i < NKB; ++i)
#pragma unroll
    for (int j = 0; j < UT; ++j) off[i * UT + j] = ((kq * NKB + i) * G + ul + NU * j) * 4;
  poll_entries<NL>(vecbase, off, a, pg);
}
// (settling and multiplying block by block, so that the FMAs of block i overlap the loads of block i+1, was measured slower
//  on the previous GPU: the per-block leaves no longer fit the register file)
template <int G, int ROWS>
__device__ __forceinline__ void push_mma(const float* __restrict__ W /*[ROWS][512] smem*/, const float4 (&a)[PushTraits<G>::NL], float* part,
                                         int ul, int kq, int warp, int lane) {
  using PT = PushTraits<G>;
  constexpr int UT = PT::UT, NU = PT::NU, NKB = PT::NKB;
  float acc[ROWS][UT];
  const float4* W4 = reinterpret_cast<const float4*>(W);
#pragma unroll
  for (int r = 0; r < ROWS; ++r) {
    float leaf[NKB][UT];
#pragma unroll
    for (int i = 0; i < NKB; ++i) {
      const float4 w = W4[r * 128 + kq * NKB + i];
      if constexpr (UT == 2) {
        // packed fp32: both rows of this thread against one broadcast weight (bit-identical to two scalar FMA chains)
        const float4 v0 = a[i * 2], v1 = a[i * 2 + 1];
        float2 s2 = fma2_rn(make_float2(v0.x, v1.x), make_float2(w.x, w.x), make_float2(0.f, 0.f));
        s2 = fma2_rn(make_float2(v0.y, v1.y), make_float2(w.y, w.y), s2);
        s2 = fma2_rn(make_float2(v0.z, v1.z), make_float2(w.z, w.z), s2);
        s2 = fma2_rn(make_float2(v0.w, v1.w), make_float2(w.w, w.w), s2);
        leaf[i][0] = s2.x; leaf[i][1] = s2.y;
      } else {
        const float4 v = a[i];
        float s1 = fmaf(w.x, v.x, 0.f);
        s1 = fmaf(w.y, v.y, s1); s1 = fmaf(w.z, v.z, s1); s1 = fmaf(w.w, v.w, s1);
        leaf[i][0] = s1;
      }
    }
#pragma unroll
    for (int j = 0; j < UT; ++j) {
      if constexpr (NKB == 4) acc[r][j] = (leaf[0][j] + leaf[1][j]) + (leaf[2][j] + leaf[3][j]);
      else acc[r][j] = leaf[0][j] + leaf[1][j];
    }
  }
  // the remaining levels of the 8-block tree: k queues that share the warp sit at lanes ul + NU*m
#pragma unroll
  for (int o = NU; o < 32; o <<= 1)
#pragma unroll
    for (int r = 0; r < ROWS; ++r)
#pragma unroll
      for (int j = 0; j < UT; ++j) acc[r][j] += __shfl_xor_sync(0xffffffffu, acc[r][j], o);
  if (lane < NU) {
#pragma unroll
    for (int r = 0; r < ROWS; ++r)
#pragma unroll
      for (int j = 0; j < UT; ++j) part[(warp * ROWS + r) * G + ul + NU * j] = acc[r][j];
  }
}
template <int G, int ROWS>
__device__ __forceinline__ void push_gemm(const float* __restrict__ W /*[ROWS][512] smem*/, const float* vecbase, float* part,
                                          int ul, int kq, int warp, int lane, PollGuard& pg) {
  float4 a[PushTraits<G>::NL];
  push_load<G>(vecbase, a, ul, kq, pg);
  push_mma<G, ROWS>(W, a, part, ul, kq, warp, lane);
}

template <int G, int ROWS>
__device__ __forceinline__ float push_part_sum(const float* part, int r, int u) {
  float v = 0.f;
#pragma unroll
  for (int w = 0; w < kPushWarps; ++w) v += part[(w * ROWS + r) * G + u];
  return v;
}

// Conditioning of step `t`.  Rows 0-15 (I rows 0-3 and the folded GRU-1 rows: FIR-combined mel projections + aux projection
// + bias) change every sample -> push_cond16, one (row, cond row) item per thread at 32 rows, all (<= 1 + kMaxTaps) table
// loads of an item in flight at once.  Rows 16-35 (GRU-2 12, fc1 4, fc2 4: aux projection + bias) are constant within a
// frame -> push_cond20, refreshed only when the next step starts a new frame (every step in fold mode, where rows sit at
// different phases).
// SESS: the tables and frame count of row u are those of session u (SessIO).
template <int G, bool SESS>
__device__ __forceinline__ void push_cond16(const PushArgs& A, const PushRowState& R, const SessIO& sio, const float* fir_s, float* cdst,
                                            int c, int ncta, int t, int tid) {
  const size_t fstride = (size_t)ncta * kPushCondRows;
  const int fr0 = t / A.hop, ph0 = t - fr0 * A.hop;                   // plain batch: every row is at the same frame / phase
  // items start at thread 4G: the gate threads (0 ... 4G-1) are busy with the fc2 gate, the re-arm and its fence at this point
  for (int it = (tid + kPushThreads - 4 * G) % kPushThreads; it < 16 * G; it += kPushThreads) {
    const int u = it >> 4, r = it & 15;
    int src = u, fr = fr0, ph = ph0;
    bool beyond = false;
    if (A.row_stride) {
      const long long n = (long long)u * A.row_stride + t;
      src = 0;
      beyond = n >= A.S_src;                                           // past the source utterance: zero mel and aux -> bias only
      fr = beyond ? A.T : (int)(n / A.hop);
      ph = beyond ? 0 : (int)(n - (long long)fr * A.hop);
    } else if (SESS || A.pack_utt) {
      int n;
      push_row_next(A, R, u, t, src, n);
      if (src < 0) { cdst[r * G + u] = 0.f; continue; }                // idle row
      fr = n / A.hop;
      ph = n - fr * A.hop;
    }
    const int T = SESS ? sio.row[src].T : A.T;
    const float* row = SESS ? sio.row[src].tab + ((size_t)fr * ncta + c) * kPushCondRows
                            : A.tab + (((size_t)src * (A.T + 1) + fr) * ncta + c) * kPushCondRows;
    float v = __ldg(row + 16 + r);
    float pm[kMaxTaps];
#pragma unroll
    for (int j = 0; j < kMaxTaps; ++j) {
      const int f = fr + j - A.NT / 2;
      pm[j] = (!beyond && j < A.NT && f >= 0 && f < T) ? __ldg(row + ((ptrdiff_t)(f - fr)) * (ptrdiff_t)fstride + r) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < kMaxTaps; ++j)
      if (j < A.NT) v = fmaf(fir_s[ph * A.NT + j], pm[j], v);          // an absent frame contributes fir * 0 = 0 exactly
    cdst[r * G + u] = v;
  }
}
template <int G, bool SESS>
__device__ __forceinline__ void push_cond20(const PushArgs& A, const PushRowState& R, const SessIO& sio, float* cdst, int c, int ncta, int t,
                                            int tid) {
  const int fr0 = t / A.hop;
  for (int it = tid; it < 20 * G; it += kPushThreads) {
    const int u = it / 20, r = it - u * 20;
    int src = u, fr = fr0;
    if (A.row_stride) {
      const long long n = (long long)u * A.row_stride + t;
      src = 0;
      fr = n >= A.S_src ? A.T : (int)(n / A.hop);
    } else if (SESS || A.pack_utt) {
      int n;
      push_row_next(A, R, u, t, src, n);
      if (src < 0) { cdst[r * G + u] = 0.f; continue; }
      fr = n / A.hop;
    }
    cdst[r * G + u] = SESS ? __ldg(sio.row[src].tab + ((size_t)fr * ncta + c) * kPushCondRows + 32 + r)
                           : __ldg(A.tab + (((size_t)src * (A.T + 1) + fr) * ncta + c) * kPushCondRows + 32 + r);
  }
}

// The whole kernel; MOL selects the sampler.  MOL models are packed with fc3 parameter j as class 8j (create_context, wavernn.cu), so CTA j < 30
// computes parameter j as its first class and publishes it, with the step tag, in its winner word; the other CTAs publish the
// tag alone.  The words and the exchange protocol are RAW's; P01 gathers the 30 parameters instead of reducing the winners.
template <int G>
__global__ void __launch_bounds__(kPushThreads, 1) wavernn_push_kernel(PushModel M, PushArgs A) {
  constexpr bool MOL = false, SESS = false;
  [[maybe_unused]] const MolIO io{};
  [[maybe_unused]] const SessIO sio{};
#include "wavernn_push_step.cuh"
}

template <int G>
__global__ void __launch_bounds__(kPushThreads, 1) wavernn_push_mol_kernel(PushModel M, PushArgs A, MolIO io) {
  constexpr bool MOL = true, SESS = false;
  [[maybe_unused]] const SessIO sio{};
#include "wavernn_push_step.cuh"
}

// RAW generation sessions: row u resumes session u of `sio` (see SessRow); A carries the shared buffers and B = rows.
template <int G>
__global__ void __launch_bounds__(kPushThreads, 1) wavernn_push_session_kernel(PushModel M, PushArgs A, SessIO sio) {
  constexpr bool MOL = false, SESS = true;
  [[maybe_unused]] const MolIO io{};
#include "wavernn_push_step.cuh"
}

// The wave of one run of each session: samples [pos, pos + n) of its one-shot wave (finish_wave_kernel), i.e. mu-law decoded,
// zero from (T-1)*hop on and faded over the 20 hops before; entries past n are zero.  wave [rows][ld].
__global__ void session_wave_kernel(SessIO sio, int hop, int fade_len, int ncls, const int* __restrict__ gen_error,
                                    double* __restrict__ wave) {
  const int b = blockIdx.y;
  const SessRow& r = sio.row[b];
  const LabelSamples sample{sio.labels + (size_t)b * sio.ld, (double)(ncls - 1), ncls, r.mu_law};
  const int wave_len = (r.T - 1) * hop;
  finish_wave_range(sample, r.pos, r.n, wave_len, fade_len, gen_error, sio.ld, wave + (size_t)b * sio.ld);
}

// ---- conditioning tables: tab[u][f][c][52] for f in [0, T]; frame T carries the bias only (zero conditioning) ------------
// cw: per CTA [16][feat] mel rows | [36][aux] aux rows | [36] bias   (floats; packed by pack_push_model below)
struct PushCondW {
  const float* wm;      // [ncta][16][feat]
  const float* wa;      // [ncta][36][aux]
  const float* bias;    // [ncta][36]
  int ncta, feat, aux;
};
// Frames [f0, f0 + FT) of table row u (rows u >= B are zero).
template <int FT>
__device__ __forceinline__ void push_cond_table_tile(const PushCondW& W, const float* __restrict__ mel /*[B][feat][T]*/,
                                                     const float* __restrict__ aux_frames /*[B][T][4*aux]*/, int B, int T, int u,
                                                     int f0, float* __restrict__ tab /*[Brows][T+1][ncta][52]*/) {
  extern __shared__ float sm[];
  float* sm_mel = sm;                          // [feat][FT]
  float* sm_aux = sm + W.feat * FT;            // [4*aux][FT]
  const int O = 4 * W.aux;
  const bool real = u < B;
  for (int i = threadIdx.x; i < W.feat * FT; i += blockDim.x) {
    const int k = i / FT, ff = f0 + i % FT;
    sm_mel[i] = (real && ff < T) ? mel[((size_t)u * W.feat + k) * T + ff] : 0.f;
  }
  for (int i = threadIdx.x; i < O * FT; i += blockDim.x) {
    const int k = i / FT, ff = f0 + i % FT;
    sm_aux[i] = (real && ff < T) ? aux_frames[((size_t)u * T + ff) * O + k] : 0.f;
  }
  __syncthreads();
  const int nout = W.ncta * kPushCondRows;
  for (int o = threadIdx.x; o < nout; o += blockDim.x) {
    const int c = o / kPushCondRows, row = o % kPushCondRows;
    float acc[FT];
    if (row < 16) {
#pragma unroll
      for (int i = 0; i < FT; ++i) acc[i] = 0.f;
      const float* w = W.wm + ((size_t)c * 16 + row) * W.feat;
      for (int k = 0; k < W.feat; ++k) {
        const float wk = __ldg(w + k);
#pragma unroll
        for (int i = 0; i < FT; ++i) acc[i] = fmaf(wk, sm_mel[k * FT + i], acc[i]);
      }
    } else {
      const int pr = row - 16;                                      // 0-15 a1 | 16-27 a2 | 28-31 a3 | 32-35 a4
      const int seg = pr < 16 ? 0 : (pr < 28 ? 1 : (pr < 32 ? 2 : 3));
      const float* w = W.wa + ((size_t)c * 36 + pr) * W.aux;
      const float b = __ldg(W.bias + (size_t)c * 36 + pr);
#pragma unroll
      for (int i = 0; i < FT; ++i) acc[i] = 0.f;
      for (int k = 0; k < W.aux; ++k) {
        const float wk = __ldg(w + k);
#pragma unroll
        for (int i = 0; i < FT; ++i) acc[i] = fmaf(wk, sm_aux[(seg * W.aux + k) * FT + i], acc[i]);
      }
#pragma unroll
      for (int i = 0; i < FT; ++i) acc[i] += b;
      if (!real) {
#pragma unroll
        for (int i = 0; i < FT; ++i) acc[i] = 0.f;
      }
      // frame T (and padding frames of the last tile): zero conditioning -> bias only
#pragma unroll
      for (int i = 0; i < FT; ++i)
        if (f0 + i >= T) acc[i] = real ? b : 0.f;
    }
#pragma unroll
    for (int i = 0; i < FT; ++i) {
      const int ff = f0 + i;
      if (ff <= T) tab[(((size_t)u * (T + 1) + ff) * W.ncta + c) * kPushCondRows + row] = (row < 16 && ff >= T) ? 0.f : acc[i];
    }
  }
}

template <int FT>
__global__ void push_cond_table_kernel(PushCondW W, const float* __restrict__ mel /*[B][feat][T]*/,
                                       const float* __restrict__ aux_frames /*[B][T][4*aux]*/, int B, int T,
                                       float* __restrict__ tab /*[Brows][T+1][ncta][52]*/) {
  push_cond_table_tile<FT>(W, mel, aux_frames, B, T, blockIdx.y, blockIdx.x * FT, tab);
}

// fills the exchange buffers with the sentinel pattern and clears the winner slots and, if given, the error flag
__global__ void push_init_kernel(uint32_t* __restrict__ vec, size_t nvec, unsigned long long* __restrict__ best, size_t nbest,
                                 int* __restrict__ error) {
  const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x, st = (size_t)gridDim.x * blockDim.x;
  for (size_t i = i0; i < nvec; i += st) vec[i] = kPushSentinel;
  for (size_t i = i0; i < nbest; i += st) best[i] = 0ull;
  if (i0 == 0 && error) *error = 0;
}

// ---- host: the per-CTA blobs [ncta][blob] and the conditioning weights (PushCondW: [ncta][16][feat] mel rows | [ncta][36][aux]
//      aux rows | [ncta][36] bias), cut from the grid kernel's blobs `gb` (pack_grid_model): the recurrent / feed-forward rows
//      stay, the conditioned columns become the weights of the tables.  Fills the layout `pm`; pm.ok says whether the model can
//      run this kernel with a [hop][NT] FIR table, and both vectors are empty when it cannot. ------------------------------------
inline std::vector<float> pack_push_model(const GridModel& g, const std::vector<float>& gb, int hop, int NT, PushModel& pm,
                                          std::vector<float>& condw) {
  const int R = g.R, F = g.F, NC = g.NC, FEAT = g.FEAT, AUX = g.AUX;
  pm = PushModel{};
  pm.ncta = g.ncta; pm.R = R; pm.F = F; pm.NC = NC;
  int off = 0;
  auto take = [&](int n) { int o = off; off += (n + 3) & ~3; return o; };
  // W_ih2 (12 rows) | fc1 (4 rows) | W_hh2 (12 rows) are contiguous: x1 is multiplied by the first 16 rows in one pass, h2 by the
  // last 16 (fc1, then W_hh2) from one set of registers
  pm.ohh1 = take(12 * R); pm.oih2 = take(12 * R); pm.ofc1 = take(4 * R); pm.ohh2 = take(12 * R);
  pm.ofc2 = take(4 * F); pm.ofc3 = take(8 * F);
  pm.oAx = take(16); pm.obhh1 = take(12); pm.obhh2 = take(12); pm.obfc3 = take(8);
  pm.blob = off;
  const size_t smem = ((size_t)pm.blob + (size_t)PushTraits<32>::scratch_floats(hop, NT)) * sizeof(float) + 1024;
  pm.ok = (g.ok && R == 512 && F == 512 && g.ncta == 128 && NC <= 1024 && smem <= 227 * 1024) ? 1 : 0;
  condw.clear();
  if (!pm.ok) return {};

  std::vector<float> pb((size_t)g.ncta * pm.blob, 0.f);
  condw.assign((size_t)g.ncta * (16 * FEAT + 36 * AUX + 36), 0.f);
  float* wm = condw.data();
  float* wa = wm + (size_t)g.ncta * 16 * FEAT;
  float* cb = wa + (size_t)g.ncta * 36 * AUX;
  for (int cta = 0; cta < g.ncta; ++cta) {
    const float* b = &gb[(size_t)cta * g.blob];
    float* d = &pb[(size_t)cta * pm.blob];
    for (int r = 0; r < 12; ++r) {
      std::memcpy(d + pm.ohh1 + (size_t)r * R, b + g.ohh1 + (size_t)r * R, sizeof(float) * R);
      std::memcpy(d + pm.oih2 + (size_t)r * R, b + g.oih2 + (size_t)r * g.ldX, sizeof(float) * R);
      std::memcpy(d + pm.ohh2 + (size_t)r * R, b + g.ohh2 + (size_t)r * R, sizeof(float) * R);
      d[pm.obhh1 + r] = b[g.obhh1 + r];
      d[pm.obhh2 + r] = b[g.obhh2 + r];
      std::memcpy(wa + ((size_t)cta * 36 + 16 + r) * AUX, b + g.oih2 + (size_t)r * g.ldX + R, sizeof(float) * AUX);
      cb[(size_t)cta * 36 + 16 + r] = b[g.obih2 + r];
    }
    for (int j = 0; j < 4; ++j) {
      std::memcpy(d + pm.ofc1 + (size_t)j * R, b + g.ofc1 + (size_t)j * g.ldX, sizeof(float) * R);
      std::memcpy(d + pm.ofc2 + (size_t)j * F, b + g.ofc2 + (size_t)j * g.ldF, sizeof(float) * F);
      std::memcpy(wa + ((size_t)cta * 36 + 28 + j) * AUX, b + g.ofc1 + (size_t)j * g.ldX + R, sizeof(float) * AUX);
      std::memcpy(wa + ((size_t)cta * 36 + 32 + j) * AUX, b + g.ofc2 + (size_t)j * g.ldF + F, sizeof(float) * AUX);
      cb[(size_t)cta * 36 + 28 + j] = b[g.obfc1 + j];
      cb[(size_t)cta * 36 + 32 + j] = b[g.obfc2 + j];
    }
    for (int r = 0; r < 8; ++r) {
      std::memcpy(d + pm.ofc3 + (size_t)r * F, b + g.ofc3 + (size_t)r * F, sizeof(float) * F);
      d[pm.obfc3 + r] = b[g.obfc3 + r];
    }
    for (int r = 0; r < 16; ++r) {          // I rows 0-3, folded GRU-1 rows 4-15: [mel | a1] columns, x coefficient, bias
      d[pm.oAx + r] = b[g.oA_x + r];
      std::memcpy(wm + ((size_t)cta * 16 + r) * FEAT, b + g.oA_w + (size_t)r * g.ldC, sizeof(float) * FEAT);
      std::memcpy(wa + ((size_t)cta * 36 + r) * AUX, b + g.oA_w + (size_t)r * g.ldC + FEAT, sizeof(float) * AUX);
      cb[(size_t)cta * 36 + r] = b[g.oA_b + r];
    }
  }
  return pb;
}

}  // namespace b200tts
