// WaveRNN per-sample recurrence, "grid" kernel: weight-stationary, persistent, cooperative.
//
// The 17.4 MB of fp32 step weights cannot live in one SM (228 KB), but they fit the chip: the grid is NCTA = R/4 = 128
// co-resident CTAs (one per SM, cooperative launch), CTA c permanently holds in SHARED MEMORY the rows of every layer
// that produce hidden units / fc rows [4c, 4c+4) and classes [8c, 8c+8) (117 KB), and all B utterances advance in
// lock step.  Per step each layer is a skinny GEMM  out[B, rows_c] = act[B, K] . W_c[rows_c, K]^T : the activations
// ([K][Bp] fp32, K-major, L2-resident, 2 KB per utterance per layer) are the only thing that moves; weights never do.
// Phases are separated by a grid-wide barrier (monotonic counter in L2, release/acquire).
//
// Replaces the hot loop of WaveRNN.generate, reference wavernn/models/fatchord_version.py:201-237, phase by phase:
//   P01 I (:208-209) + GRU rnn1 (:210,:212): the I layer is FOLDED into the GRU's input projection,
//       W_ih1.(W_I.[x|m_t|a1] + b_I) + b_ih1 = (W_ih1.W_I).[x|m_t|a1] + (W_ih1.b_I + b_ih1)   (product formed in fp64 on the
//       host), so one phase computes Iout rows (4 x 113), gi (12 x 113), gh (12 x 512), h1' and x1 = Iout + h1'.
//       This removes a grid barrier, 14 % of the MACs and the Iout round trip through L2.
//   P2  GRU rnn2 (:213-216)  x1|a2,h2 -> h2', x2 = x1 + h2'          12 x 544 + 12 x 512
//   P3  fc1+relu (:217-218)  x2|a3 -> f1                              4 rows x 544
//   P4  fc2+relu (:220-221)  f1|a4 -> f2                              4 rows x 544
//   P5  fc3      (:223) + sampling (:232-235): every CTA owns 8 logits per utterance and joins a distributed
//       argmax of (logit - log q), q ~ Exp(1), through one 64-bit atomicMax per (CTA, utterance)  [Gumbel-max ==
//       Categorical(softmax(logits)).sample()]; the winner is read back by everybody at the next P0 (:235-237).
// Two thread mappings: "wide" for B >= 5 -- lanes = utterances, register tile 4 utterances x 6 rows, 16 warps factored as
// (GEMM x utterance warp x row slice x k slice), k-slice partial sums through shared memory, two independent utterance
// groups per CTA above 128 utterances (own named barrier + grid-barrier counter each) so one group computes while the
// other sits in a barrier -- and "narrow" for B <= 4 (activation vector staged into shared memory in one L2 round trip,
// lanes = k, warp-shuffle reductions) where the step is pure latency.
#pragma once
#include "common.cuh"

namespace b200tts {

constexpr int kGridWarpsWide = 16;     // wide mapping: warps per CTA.  Measured at B=256: 8 warps (255 regs, 4x12 tiles) 80.5 us,
                                       // 12 warps (168 regs) spill, 16 warps (128 regs, 4x6 tiles via row slices) 73.5 us
constexpr int kGridWarpsNarrow = 8;
constexpr int kUPC = 4;   // hidden units (and fc1/fc2 rows) per CTA
constexpr int kCPC = 8;   // classes (fc3 rows) per CTA

struct GridModel {        // layout of one CTA's weight blob (offsets in floats, every array 16-byte aligned)
  int ncta, R, F, AUX, FEAT, NC;
  int ldC;                // feat + aux   (cond columns of I, multiple of 4)
  int ldX;                // R + aux
  int ldF;                // F + aux
  int oA_w, oA_x, oA_b;                            // [16][ldC], [16], [16]: rows 0-3 = I, rows 4-15 = W_ih1.W_I (gate*4 + unit)
  int ohh1, oih2, ohh2;                            // [12][R], [12][ldX], [12][R]   row = gate*4 + unit
  int ofc1, ofc2, ofc3;                            // [4][ldX], [4][ldF], [8][F]
  int obhh1, obih2, obhh2, obfc1, obfc2, obfc3;
  int blob;                                        // floats per CTA
  int ok;                                          // model fits this kernel
};

struct GridArgs {
  const float* wblob;          // [ncta][blob]
  float* h1;                   // [2][R][Bp]
  float* h2;                   // [2][R][Bp]
  float* x1;                   // [R][Bp]
  float* x2;                   // [R][Bp]
  float* f1;                   // [F][Bp]
  float* f2;                   // [F][Bp]
  unsigned long long* best;    // [2][Bp]   packed argmax per utterance, ping-pong by step parity
  unsigned int* barrier;       // monotonic arrival counter
  int* error;                  // set non-zero if a barrier wait timed out
  const float* mels_T;         // [S][FEAT][Bp]
  const float* aux_T;          // [T][4*AUX][Bp]
  int B, Bp, S, T, hop, steps;
  int rng_mode;
  unsigned long long seed, utt_offset;
  const unsigned long long* utt_ids;   // optional [B]: global utterance index of every row (overrides utt_offset + row)
  const float* q;              // [S][B][NC]
  const int16_t* teacher;      // [B][S]
  float* logits_out;           // [S][B][NC]
  int16_t* labels;             // [B][S]
  long long* prof;             // optional [ncta][12]: cycles spent in compute / barrier of each phase (debug)
};

// ---- grid-wide barrier --------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned int ld_acquire_u32(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_add_u32(unsigned int* p, unsigned int v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// Group-local block barrier: the CTA may host two independent utterance groups (warps [0,NWG) and [NWG,2*NWG)); each
// synchronises on its own named barrier so that one group can sit in a grid barrier while the other computes.
template <int GROUPS, int NTG>
__device__ __forceinline__ void group_sync(int grp) {
  if constexpr (GROUPS == 1) __syncthreads();
  else asm volatile("bar.sync %0, %1;" ::"r"(grp + 1), "r"(NTG) : "memory");
}

// The grid barrier in two halves so that work which does not depend on the other CTAs can sit between them.
// `grid_arrive`: all threads of the group call, after their last global write of the phase.
// `grid_wait`:   all threads of the group call; `target` = (number of barriers arrived at so far) * gridDim.x.  False on
//                timeout (a co-resident CTA is gone): the caller returns instead of hanging the GPU.
template <int GROUPS, int NTG>
__device__ __forceinline__ void grid_arrive(unsigned int* ctr, int grp, int gtid) {
  group_sync<GROUPS, NTG>(grp);
  if (gtid == 0) red_release_add_u32(ctr, 1u);    // release: orders this group's prior global writes (cumulative via bar.sync)
}
__device__ __forceinline__ int grid_spin(const unsigned int* ctr, unsigned int target, int* error) {
  long long t0 = clock64();
  while (ld_acquire_u32(ctr) < target) {
    if (clock64() - t0 > 4000000000LL) {          // ~2 s: a peer CTA is gone; bail out instead of hanging the GPU
      atomicExch(error, 1);
      return 0;
    }
  }
  return 1;
}
template <int GROUPS, int NTG>
__device__ __forceinline__ bool grid_wait(unsigned int* ctr, unsigned int target, int* error, int grp, int gtid, int* s_ok) {
  if (gtid == 0) s_ok[grp] = grid_spin(ctr, target, error);
  group_sync<GROUPS, NTG>(grp);
  return s_ok[grp] != 0;
}
template <int GROUPS, int NTG>
__device__ __forceinline__ bool grid_barrier(unsigned int* ctr, unsigned int target, int* error, int grp, int gtid, int* s_ok) {
  grid_arrive<GROUPS, NTG>(ctr, grp, gtid);
  return grid_wait<GROUPS, NTG>(ctr, target, error, grp, gtid, s_ok);
}
// Only the first `NSUB` threads of the group wait (named barrier 3 + grp); the rest of the group carries on and meets
// them at the next group_sync.  The outcome is left in s_ok[grp] for everybody to read after that group_sync.
template <int NSUB>
__device__ __forceinline__ void grid_wait_sub(unsigned int* ctr, unsigned int target, int* error, int grp, int gtid, int* s_ok) {
  if (gtid == 0) s_ok[grp] = grid_spin(ctr, target, error);
  asm volatile("bar.sync %0, %1;" ::"r"(grp + 3), "r"(NSUB) : "memory");
}

// ---- activation loads (L2 only: these buffers are rewritten by other SMs every step) ----------------------------------
template <int U> struct ActLoad;
template <> struct ActLoad<1> {
  static __device__ __forceinline__ void ld(const float* p, float (&a)[1]) { a[0] = __ldcg(p); }
  static __device__ __forceinline__ void st(float* p, const float (&a)[1]) { p[0] = a[0]; }
};
template <> struct ActLoad<2> {
  static __device__ __forceinline__ void ld(const float* p, float (&a)[2]) {
    float2 v = __ldcg(reinterpret_cast<const float2*>(p)); a[0] = v.x; a[1] = v.y;
  }
  static __device__ __forceinline__ void st(float* p, const float (&a)[2]) { *reinterpret_cast<float2*>(p) = make_float2(a[0], a[1]); }
};
template <> struct ActLoad<4> {
  static __device__ __forceinline__ void ld(const float* p, float (&a)[4]) {
    float4 v = __ldcg(reinterpret_cast<const float4*>(p)); a[0] = v.x; a[1] = v.y; a[2] = v.z; a[3] = v.w;
  }
  static __device__ __forceinline__ void st(float* p, const float (&a)[4]) {
    *reinterpret_cast<float4*>(p) = make_float4(a[0], a[1], a[2], a[3]);
  }
};

struct Seg {            // a run of activation rows: act[4*n4][Bp], matching 4*n4 consecutive weight columns
  const float* act;
  int n4;
};
struct Gemm {           // rows x (sum of segs) weight block in shared memory
  const float* W;
  int ldw;              // floats, multiple of 4
  Seg seg[2];
  int nseg;
};

// acc[r][u] += sum_{c4 in [lo,hi)} W[r][4*(col4+c4) .. +3] . act[4*c4 .. +3][u0 .. u0+U)
template <int U, int RT>
__device__ __forceinline__ void wide_fma4(float (&acc)[RT][U], const float4* __restrict__ W4, int ldw4, int c4,
                                          const float (&a)[4][U]) {
#pragma unroll
  for (int r = 0; r < RT; ++r) {
    float4 w = W4[r * ldw4 + c4];
    if constexpr (U % 2 == 0) {
      // two utterances against ONE weight register per step (fma2_rn: two scalar FFMAs on Hopper, which has no packed
      // fp32 FMA) -- bit-identical to the scalar loop below (same rounding, same summation order per lane).
#pragma unroll
      for (int u = 0; u < U; u += 2) {
        float2 s = make_float2(acc[r][u], acc[r][u + 1]);
        s = fma2_rn(make_float2(a[0][u], a[0][u + 1]), make_float2(w.x, w.x), s);
        s = fma2_rn(make_float2(a[1][u], a[1][u + 1]), make_float2(w.y, w.y), s);
        s = fma2_rn(make_float2(a[2][u], a[2][u + 1]), make_float2(w.z, w.z), s);
        s = fma2_rn(make_float2(a[3][u], a[3][u + 1]), make_float2(w.w, w.w), s);
        acc[r][u] = s.x; acc[r][u + 1] = s.y;
      }
    } else {
#pragma unroll
      for (int u = 0; u < U; ++u) {
        acc[r][u] = fmaf(w.x, a[0][u], acc[r][u]);
        acc[r][u] = fmaf(w.y, a[1][u], acc[r][u]);
        acc[r][u] = fmaf(w.z, a[2][u], acc[r][u]);
        acc[r][u] = fmaf(w.w, a[3][u], acc[r][u]);
      }
    }
  }
}
template <int U>
__device__ __forceinline__ void wide_ld4(float (&a)[4][U], const float* __restrict__ p, unsigned Bp) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) ActLoad<U>::ld(p + kk * Bp, a[kk]);
}
// n float4 weight columns starting at W4 (row stride ldw4), activation rows starting at `ap` (row stride Bp floats).
// The activation loads come from L2 (about a microsecond under load), so they are software pipelined: the loads of the
// NEXT PD columns are issued before the PD x 4*RT*U FMAs of the current ones (ping-pong register buffers, 4*PD LDG.128 in
// flight per thread), addresses advance by pointer bumps.
template <int U, int RT, int PD>
__device__ __forceinline__ void wide_accumulate_pd(float (&acc)[RT][U], const float* __restrict__ W, int ldw, int col4,
                                                   const float* __restrict__ act, int Bp_, int u0, int lo, int hi) {
  const unsigned Bp = (unsigned)Bp_;
  const int ldw4 = ldw >> 2;
  const float4* W4 = reinterpret_cast<const float4*>(W) + col4 + lo;
  const float* p = act + (size_t)(4 * lo) * Bp + u0;
  const size_t step = (size_t)4 * Bp;
  const int n = hi - lo;
  const int nmain = n - n % (2 * PD);          // every shape of this model gives n % 4 == 0; the tail loop is only a safety net
  float c[PD][4][U], nb[PD][4][U];
  // ONE copy of the unrolled body (2*PD blocks of 4*RT*U FMAs): the look-ahead loads of the last trip are predicated
  // instead of peeling prologue / epilogue variants (the fully peeled version made the kernel 288 KB of SASS).
  if (nmain > 0) {
#pragma unroll
    for (int j = 0; j < PD; ++j) wide_ld4<U>(c[j], p + j * step, Bp);
    p += PD * step;
#pragma unroll 1
    for (int i = 0; i < nmain; i += 2 * PD) {
#pragma unroll
      for (int j = 0; j < PD; ++j) wide_ld4<U>(nb[j], p + j * step, Bp);
      p += PD * step;
#pragma unroll
      for (int j = 0; j < PD; ++j) wide_fma4<U, RT>(acc, W4, ldw4, i + j, c[j]);
      if (i + 2 * PD < nmain) {
#pragma unroll
        for (int j = 0; j < PD; ++j) wide_ld4<U>(c[j], p + j * step, Bp);
        p += PD * step;
      }
#pragma unroll
      for (int j = 0; j < PD; ++j) wide_fma4<U, RT>(acc, W4, ldw4, i + PD + j, nb[j]);
    }
  }
#pragma unroll 1
  for (int i = nmain; i < n; ++i) {
    wide_ld4<U>(c[0], p, Bp); p += step;
    wide_fma4<U, RT>(acc, W4, ldw4, i, c[0]);
  }
}
template <int U, int RT>
__device__ __forceinline__ void wide_accumulate(float (&acc)[RT][U], const float* __restrict__ W, int ldw, int col4,
                                                const float* __restrict__ act, int Bp, int u0, int lo, int hi) {
  // one column of look-ahead: the 16-warp build leaves 128 registers per thread, and on the previous GPU 3-4 columns ahead
  // was slower also on the 4/8-row tiles, which have registers to spare
  wide_accumulate_pd<U, RT, 1>(acc, W, ldw, col4, act, Bp, u0, lo, hi);
}

// Wide mapping: NG GEMMs of RT rows each; 8 warps = NG x UW (utterance warps) x KS (k slices).
// Partial sums land in part[((g*KS + ks)*RT + r)*BT + ul].
// (Measured on the previous GPU: sharing one __noinline__ copy of this body between phases to shrink the ~65 KB kernel is
// slower -- the call/stack traffic costs more than the instruction-fetch stalls it removes.)
template <int NW, int U, int UW, int RT, int NG, int RS = 1>
__device__ __forceinline__ void wide_partials(float* part, const Gemm& g0, const Gemm& g1, int tile_base, int Bp, int warp,
                                              int lane) {
  // warps = NG GEMMs x UW utterance warps x RS row slices x KS k slices; a thread owns U utterances x RT/RS rows
  constexpr int KS = NW / (NG * UW * RS);
  constexpr int BT = 32 * U * UW;
  constexpr int RTT = RT / RS;
  static_assert(KS >= 1 && KS * NG * UW * RS == NW && RTT * RS == RT, "warps must factor as NG x UW x RS x KS");
  const int g = warp / (UW * RS * KS), rem = warp % (UW * RS * KS), uw = rem / (RS * KS), rs = (rem / KS) % RS, ks = rem % KS;
  const Gemm& G = (NG == 2 && g == 1) ? g1 : g0;
  const int ul = uw * 32 * U + lane * U;
  float acc[RTT][U];
#pragma unroll
  for (int r = 0; r < RTT; ++r)
#pragma unroll
    for (int u = 0; u < U; ++u) acc[r][u] = 0.f;
  int N4 = G.seg[0].n4 + (G.nseg > 1 ? G.seg[1].n4 : 0);
  const int lo = N4 * ks / KS, hi = N4 * (ks + 1) / KS;
  const float* Wr = G.W + (size_t)rs * RTT * G.ldw;
  int col = 0;
  if constexpr (NG == 2) {                        // the big 2-GEMM phase: segments unrolled (measured faster for P2)
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      if (s < G.nseg) {
        const int a = max(lo, col), b = min(hi, col + G.seg[s].n4);
        if (a < b) wide_accumulate<U, RTT>(acc, Wr, G.ldw, col, G.seg[s].act, Bp, tile_base + ul, a - col, b - col);
        col += G.seg[s].n4;
      }
    }
  } else {
#pragma unroll 1
    for (int s = 0; s < G.nseg; ++s) {            // runtime loop: one copy of the GEMM body per call site
      const int a = max(lo, col), b = min(hi, col + G.seg[s].n4);
      if (a < b) wide_accumulate<U, RTT>(acc, Wr, G.ldw, col, G.seg[s].act, Bp, tile_base + ul, a - col, b - col);
      col += G.seg[s].n4;
    }
  }
  float* dst = part + (size_t)((g * KS + ks) * RT + rs * RTT) * BT + ul;
#pragma unroll
  for (int r = 0; r < RTT; ++r) ActLoad<U>::st(dst + r * BT, acc[r]);
}

// Narrow mapping (Bp == G == 4): the whole activation vector of the phase is first staged into shared memory by all
// threads (ONE L2 round trip), then lanes stride over float4 columns, RT rows per warp pass, shuffle reduction.
// Warps [wbeg, wbeg+wcnt) take part.  Result in out[(gslot*nrows + r)*G + u].
template <int G>
__device__ __forceinline__ void smem_ld(const float* p, float (&a)[G]) {
  static_assert(G == 4, "one float4 per activation row");
  const float4 v = *reinterpret_cast<const float4*>(p);
  a[0] = v.x; a[1] = v.y; a[2] = v.z; a[3] = v.w;
}
template <int NT>
__device__ __forceinline__ void stage_rows(float* dst, const float* __restrict__ src, int nfloats, int tid) {
  for (int i = tid; i < nfloats / 4; i += NT)
    reinterpret_cast<float4*>(dst)[i] = __ldcg(reinterpret_cast<const float4*>(src) + i);
}
template <int G, int RT>
__device__ __forceinline__ void narrow_rows(float* out, int gslot, const float* __restrict__ W, int ldw, const float* act,
                                            int n4, int nrows, int wbeg, int wcnt, int warp, int lane) {
  if (warp < wbeg || warp >= wbeg + wcnt) return;
  const int ldw4 = ldw >> 2;
  for (int r0 = (warp - wbeg) * RT; r0 < nrows; r0 += wcnt * RT) {
    float acc[RT][G];
#pragma unroll
    for (int r = 0; r < RT; ++r)
#pragma unroll
      for (int u = 0; u < G; ++u) acc[r][u] = 0.f;
    const float4* W4 = reinterpret_cast<const float4*>(W) + (size_t)r0 * ldw4;
    for (int c4 = lane; c4 < n4; c4 += 32) {
      float a[4][G];
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) smem_ld<G>(act + (size_t)(4 * c4 + kk) * G, a[kk]);
#pragma unroll
      for (int r = 0; r < RT; ++r) {
        float4 w = W4[r * ldw4 + c4];
#pragma unroll
        for (int u = 0; u < G; ++u) {
          acc[r][u] = fmaf(w.x, a[0][u], acc[r][u]);
          acc[r][u] = fmaf(w.y, a[1][u], acc[r][u]);
          acc[r][u] = fmaf(w.z, a[2][u], acc[r][u]);
          acc[r][u] = fmaf(w.w, a[3][u], acc[r][u]);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < RT; ++r)
#pragma unroll
      for (int u = 0; u < G; ++u) {
        float v = warp_sum(acc[r][u]);
        if (lane == 0) out[(size_t)(gslot * nrows + r0 + r) * G + u] = v;
      }
  }
}

// Mapping traits.  U == 0 selects the narrow mapping with G = UW utterances.  GROUPS = independent utterance groups
// per CTA (wide only): with 2, warps 0-3 and 4-7 run the same phase sequence on disjoint utterance ranges, each with its
// own named barrier and grid-barrier counter, sharing the resident weights -- stalls of one group (L2 latency, barrier
// wait) are filled by the other (one warp of each group per scheduler).
template <int U, int UW, int GROUPS> struct MapTraits {
  static constexpr bool kWide = true;
  static constexpr int NW = kGridWarpsWide;                                // warps per CTA
  static constexpr int NWG = NW / GROUPS;                                  // warps per group
  static constexpr int BT = 32 * U * UW;                                   // utterances per group tile
  static constexpr int RS12 = (UW == 1) ? 2 : 1;                           // row slices of the 12-row GRU tiles (16-warp build:
                                                                           // 128 registers/thread -> 4 utterances x 6 rows)
  static constexpr int KS1 = NWG / UW;                                     // k slices of the 4/8-row 1-GEMM phases (fc1/fc2/fc3)
  static constexpr int KSB = NWG / (UW * RS12);                            // ... of the 12-row 1-GEMM pass of P01 (W_hh1)
  static constexpr int RS2 = RS12;                                         // row slices in the 2-GEMM phase (GRU 2)
  static constexpr int KS2 = NWG / (2 * UW * RS2);                         // ... of the 2-GEMM phase (GRU 2)
  static constexpr int kPartRows = KSB * 12 > KS1 * 8 ? KSB * 12 : KS1 * 8;
  static constexpr int kPartFloats = (kPartRows > 2 * KS2 * 12 ? kPartRows : 2 * KS2 * 12) * BT;   // largest partial-sum footprint
  static constexpr int KSA = NWG / (UW * 4);                               // k slices of P01's 16 cond rows (4 row slices of 4)
  static constexpr int kCondOff = KSB * 12 * BT;                           // P01: cond-row partials sit behind the W_hh1 partials
  static constexpr int kGroupScratch = kPartFloats > kCondOff + KSA * 16 * BT ? kPartFloats : kCondOff + KSA * 16 * BT;
  static_assert(KSA >= 1 && KSA * UW * 4 == NWG, "group warps must factor as UW x 4 x KSA");
  static constexpr int kScratchFloats = GROUPS * kGroupScratch;
  static_assert(KS2 >= 1 && KS2 * 2 * UW * RS2 == NWG, "group warps must factor as 2 x UW x RS2 x KS2");
};
template <int G> struct MapTraits<0, G, 1> {
  static constexpr bool kWide = false;
  static constexpr int NW = kGridWarpsNarrow;
  static constexpr int NWG = NW;
  static constexpr int BT = G;
  static constexpr int RS12 = 1;
  static constexpr int RS2 = 1;
  static constexpr int KS1 = 1;
  static constexpr int KSB = 1;
  static constexpr int KS2 = 1;
  static constexpr int KSA = 1;
  static constexpr int kPartFloats = 0;
  static constexpr int kGroupScratch = 640 * G + 512 * G + 32 * G + 64;   // staged act A | act B | row results (16 + 12 rows)
  static constexpr int kScratchFloats = kGroupScratch;
};

// sum over k slices of one output: gemm slot g, row r (of RT), local utterance ul
template <int KS, int RT, int BT>
__device__ __forceinline__ float part_sum(const float* part, int g, int r, int ul) {
  float v = 0.f;
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) v += part[(size_t)((g * KS + ks) * RT + r) * BT + ul];
  return v;
}

__device__ __forceinline__ float gru_update(float gir, float giz, float gin, float ghr, float ghz, float ghn, float hold) {
  const float r = sigmoidf_acc(gir + ghr), z = sigmoidf_acc(giz + ghz);
  const float n = tanhf(gin + r * ghn);
  return (1.0f - z) * n + z * hold;
}

template <int U, int UW, int GROUPS>
__global__ void __launch_bounds__(MapTraits<U, UW, GROUPS>::NW * 32, 1) wavernn_grid_kernel(GridModel M, GridArgs A) {
  using MT = MapTraits<U, UW, GROUPS>;
  constexpr int BT = MT::BT, NWG = MT::NWG, NT = NWG * 32;   // NT = threads of one group
  constexpr int KS1 = MT::KS1, KS2 = MT::KS2, KSB = MT::KSB, KSA = MT::KSA, RS12 = MT::RS12;
  constexpr int G = MT::kWide ? 4 : UW;               // narrow: utterances per row; (unused value in wide mode)
  extern __shared__ __align__(16) float smem[];
  float* Wb = smem;                                   // this CTA's weights, resident for the whole kernel
  __shared__ float xs_all[GROUPS * (BT > 32 ? BT : 32)];

  const int lane = threadIdx.x & 31;
  const int grp = (GROUPS == 1) ? 0 : (int)(threadIdx.x >> 5) / NWG;   // utterance group of this warp
  const int warp = (int)(threadIdx.x >> 5) - grp * NWG;                // warp index within the group
  const int tid = (int)threadIdx.x - grp * NT;                         // thread index within the group
  float* part = smem + M.blob + grp * MT::kGroupScratch;               // wide: partial sums; narrow: staged act + results
  float* xs = xs_all + grp * (BT > 32 ? BT : 32);                      // fed-back sample of the tile's utterances
  const int c = blockIdx.x, Bp = A.Bp;
  const int tb_lo = grp * (Bp / GROUPS), tb_hi = (grp + 1) * (Bp / GROUPS);   // this group's utterance columns
  unsigned int* bar_ctr = A.barrier + grp * 32;
  const int R = M.R, F = M.F, AUX = M.AUX;
  const float ncls_m1 = (float)(M.NC - 1);
  {
    // one-time load of this CTA's 117 KB weight blob: TMA bulk copies (UBLKCP) signalled through an mbarrier
    __shared__ __align__(8) unsigned long long wbar;
    const char* src = reinterpret_cast<const char*>(A.wblob + (size_t)c * M.blob);
    const unsigned total = (unsigned)M.blob * 4u;
    if (threadIdx.x == 0) mbar_init(&wbar, 1);
    __syncthreads();
    if (threadIdx.x == 0) {
      mbar_expect_tx(&wbar, total);
      for (unsigned off = 0; off < total; off += 32768u)
        tma_bulk_g2s(reinterpret_cast<char*>(Wb) + off, src + off, min(32768u, total - off), &wbar);
    }
    mbar_wait(&wbar, 0);
  }
  __syncthreads();
  unsigned int nbar = 0;
  const unsigned int ncta = gridDim.x;
  __shared__ int s_ok[2];                             // outcome of the group's last barrier wait
  // Split barriers.  0: plain barriers; 1: P01's GEMMs run before the wait on P5's barrier; 2: also GRU-2's W_hh pass starts
  // before the wait on P01's barrier.  They paid off on the previous GPU when ONE group owns the SM (B <= 128); with two groups
  // the other group already fills the barrier bubble and the split was slower, so it is off there.  Not re-measured on the H100.
  constexpr int kSplit = (GROUPS == 1) ? 2 : 0;
  bool pending = false;                               // arrived at the sampling barrier of the previous step, not yet waited
  unsigned int pend_target = 0;
  const size_t RB = (size_t)R * Bp;
  // narrow-mode scratch views
  float* stA = part;
  float* stB = part + (MT::kWide ? 0 : 640 * G);
  float* nout = part + (MT::kWide ? 0 : 640 * G + 512 * G);
  const float* res = MT::kWide ? part : nout;         // where part_sum() reads

  long long pf[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) pf[i] = 0;
  long long tmark = clock64();
#define PROF_MARK(slot)                                   \
  do {                                                    \
    if (A.prof && grp == 0) {                             \
      long long now_ = clock64();                         \
      pf[slot] += now_ - tmark;                           \
      tmark = now_;                                       \
    }                                                     \
  } while (0)
  for (int t = 0; t < A.steps; ++t) {
    const int cur = t & 1, fr = t / A.hop;
    const float* auxT = A.aux_T + (size_t)fr * 4 * AUX * Bp;
    const float* h1c = A.h1 + cur * RB;
    float* h1n = A.h1 + (cur ^ 1) * RB;
    const float* h2c = A.h2 + cur * RB;
    float* h2n = A.h2 + (cur ^ 1) * RB;

    // ================= P01: read back the previous step's winner; I layer folded into GRU 1 =================
    for (int tb = tb_lo; tb < tb_hi; tb += BT) {
      const float* melT = A.mels_T + (size_t)t * M.FEAT * Bp;
      const float* rA;        // [16][BT]: cond part of the 4 I rows and the 12 folded gi rows
      const float* rB;        // gh partial sums (k slices) / rows
      if constexpr (MT::kWide) {
        float* resA = part + MT::kCondOff;
        Gemm ga{};
        ga.W = Wb + M.oA_w; ga.ldw = M.ldC; ga.nseg = 2; ga.seg[0] = Seg{melT, M.FEAT / 4}; ga.seg[1] = Seg{auxT, AUX / 4};
        wide_partials<NWG, U, UW, 16, 1, 4>(resA, ga, ga, tb, Bp, warp, lane);
        Gemm gh{};
        gh.W = Wb + M.ohh1; gh.ldw = R; gh.nseg = 1; gh.seg[0] = Seg{h1c, R / 4};
        wide_partials<NWG, U, UW, 3 * kUPC, 1, RS12>(part, gh, gh, tb, Bp, warp, lane);
        rA = resA; rB = part;
      } else {
        stage_rows<NT>(stA, melT, M.FEAT * G, tid);
        stage_rows<NT>(stA + M.FEAT * G, auxT, AUX * G, tid);
        stage_rows<NT>(stB, h1c, R * G, tid);
        group_sync<GROUPS, NT>(grp);
        narrow_rows<G, 4>(nout, 0, Wb + M.oA_w, M.ldC, stA, M.ldC / 4, 16, 0, NWG / 2, warp, lane);
        narrow_rows<G, 3>(nout + 16 * G, 0, Wb + M.ohh1, R, stB, R / 4, 3 * kUPC, NWG / 2, NWG / 2, warp, lane);
        rA = nout; rB = nout + 16 * G;
      }
      // Everything above reads only the conditioning and h1(t-1).  The fed-back sample needs the sampling barrier of
      // step t-1, which this group arrived at before starting the GEMMs: its latency and skew hide behind them.
      if (pending) {
        PROF_MARK(0);
        if (!grid_wait<GROUPS, NT>(bar_ctr, pend_target, A.error, grp, tid, s_ok)) return;
        pending = false;
        PROF_MARK(11);
      }
      for (int ul = tid; ul < BT; ul += NT) {       // read back the previous step's winner
        const int u = tb + ul;
        float x = 0.f;
        if (t > 0 && u < A.B) {
          unsigned long long pk = __ldcg(A.best + (size_t)((t - 1) & 1) * Bp + u);
          int label = (int)unpack_idx(pk);
          if (c == 0) A.labels[(size_t)u * A.S + (t - 1)] = (int16_t)label;
          int fb = A.teacher ? (int)A.teacher[(size_t)u * A.S + (t - 1)] : label;
          x = label_to_float(fb, ncls_m1);
        }
        xs[ul] = x;
      }
      group_sync<GROUPS, NT>(grp);
      const float* wAx = Wb + M.oA_x; const float* bA = Wb + M.oA_b; const float* bhh = Wb + M.obhh1;
      for (int idx = tid; idx < BT * kUPC; idx += NT) {
        const int ul = idx % BT, j = idx / BT;
        const size_t o = (size_t)(c * kUPC + j) * Bp + tb + ul;
        const float x = xs[ul];
        float hold;
        if constexpr (MT::kWide) hold = __ldcg(h1c + o);
        else hold = stB[(c * kUPC + j) * G + ul];
        const float iout = fmaf(wAx[j], x, part_sum<KSA, 16, BT>(rA, 0, j, ul)) + bA[j];
        const float gir = fmaf(wAx[4 + j], x, part_sum<KSA, 16, BT>(rA, 0, 4 + j, ul)) + bA[4 + j];
        const float giz = fmaf(wAx[4 + kUPC + j], x, part_sum<KSA, 16, BT>(rA, 0, 4 + kUPC + j, ul)) + bA[4 + kUPC + j];
        const float gin = fmaf(wAx[4 + 2 * kUPC + j], x, part_sum<KSA, 16, BT>(rA, 0, 4 + 2 * kUPC + j, ul)) + bA[4 + 2 * kUPC + j];
        float h = gru_update(gir, giz, gin, part_sum<KSB, 3 * kUPC, BT>(rB, 0, j, ul) + bhh[j],
                             part_sum<KSB, 3 * kUPC, BT>(rB, 0, kUPC + j, ul) + bhh[kUPC + j],
                             part_sum<KSB, 3 * kUPC, BT>(rB, 0, 2 * kUPC + j, ul) + bhh[2 * kUPC + j], hold);
        h1n[o] = h;
        A.x1[o] = iout + h;
      }
      if (tb + BT < tb_hi) group_sync<GROUPS, NT>(grp);
    }
    PROF_MARK(0);
    constexpr bool kEarlyHH = kSplit >= 2;                    // GRU-2's W_hh pass reads only h2(t-1): it need not wait for x1
    if constexpr (kEarlyHH) {
      grid_arrive<GROUPS, NT>(bar_ctr, grp, tid);
      ++nbar;
    } else {
      if (!grid_barrier<GROUPS, NT>(bar_ctr, (++nbar) * ncta, A.error, grp, tid, s_ok)) return;
      PROF_MARK(1);
    }

    // ================= P2: GRU 2 =================
    for (int tb = tb_lo; tb < tb_hi; tb += BT) {
      const bool first_tile = (tb == tb_lo);
      if constexpr (MT::kWide) {
        Gemm gi{}, gh{};
        gi.W = Wb + M.oih2; gi.ldw = M.ldX; gi.nseg = 2; gi.seg[0] = Seg{A.x1, R / 4};
        gi.seg[1] = Seg{auxT + (size_t)AUX * Bp, AUX / 4};
        gh.W = Wb + M.ohh2; gh.ldw = R; gh.nseg = 1; gh.seg[0] = Seg{h2c, R / 4};
        if constexpr (kEarlyHH) {
          // warps [0, NWG/2) own the W_ih GEMM (x1 from the other CTAs): only they wait; the W_hh warps start at once
          if (first_tile && warp < NWG / 2) {
            grid_wait_sub<NT / 2>(bar_ctr, nbar * ncta, A.error, grp, tid, s_ok);
            PROF_MARK(1);
          }
        }
        wide_partials<NWG, U, UW, 3 * kUPC, 2, MT::RS2>(part, gi, gh, tb, Bp, warp, lane);
      } else {
        stage_rows<NT>(stA + R * G, auxT + (size_t)AUX * Bp, AUX * G, tid);
        stage_rows<NT>(stB, h2c, R * G, tid);
        if constexpr (kEarlyHH) {
          if (first_tile) {
            if (!grid_wait<GROUPS, NT>(bar_ctr, nbar * ncta, A.error, grp, tid, s_ok)) return;
            PROF_MARK(1);
          }
        }
        stage_rows<NT>(stA, A.x1, R * G, tid);
        group_sync<GROUPS, NT>(grp);
        narrow_rows<G, 3>(nout, 0, Wb + M.oih2, M.ldX, stA, M.ldX / 4, 3 * kUPC, 0, NWG / 2, warp, lane);
        narrow_rows<G, 3>(nout, 1, Wb + M.ohh2, R, stB, R / 4, 3 * kUPC, NWG / 2, NWG / 2, warp, lane);
      }
      group_sync<GROUPS, NT>(grp);
      if constexpr (kEarlyHH && MT::kWide) {
        if (first_tile && !s_ok[grp]) return;       // the sub-group wait timed out: every thread of the group leaves here
      }
      const float* bih = Wb + M.obih2; const float* bhh = Wb + M.obhh2;
      for (int idx = tid; idx < BT * kUPC; idx += NT) {
        const int ul = idx % BT, j = idx / BT;
        const size_t o = (size_t)(c * kUPC + j) * Bp + tb + ul;
        float hold, resid;
        if constexpr (MT::kWide) { hold = __ldcg(h2c + o); resid = __ldcg(A.x1 + o); }
        else { hold = stB[(c * kUPC + j) * G + ul]; resid = stA[(c * kUPC + j) * G + ul]; }
        float h = gru_update(part_sum<KS2, 3 * kUPC, BT>(res, 0, j, ul) + bih[j],
                             part_sum<KS2, 3 * kUPC, BT>(res, 0, kUPC + j, ul) + bih[kUPC + j],
                             part_sum<KS2, 3 * kUPC, BT>(res, 0, 2 * kUPC + j, ul) + bih[2 * kUPC + j],
                             part_sum<KS2, 3 * kUPC, BT>(res, 1, j, ul) + bhh[j],
                             part_sum<KS2, 3 * kUPC, BT>(res, 1, kUPC + j, ul) + bhh[kUPC + j],
                             part_sum<KS2, 3 * kUPC, BT>(res, 1, 2 * kUPC + j, ul) + bhh[2 * kUPC + j], hold);
        h2n[o] = h;
        A.x2[o] = resid + h;
      }
      if (tb + BT < tb_hi) group_sync<GROUPS, NT>(grp);
    }
    PROF_MARK(4);
    if (!grid_barrier<GROUPS, NT>(bar_ctr, (++nbar) * ncta, A.error, grp, tid, s_ok)) return;
    PROF_MARK(5);

    // ================= P3: fc1 + relu  (CTA 0 also recycles the argmax slot the NEXT step will use) =================
    if (c == 0)
      for (int u = tb_lo + tid; u < tb_hi; u += NT) A.best[(size_t)((t + 1) & 1) * Bp + u] = 0ull;
    for (int tb = tb_lo; tb < tb_hi; tb += BT) {
      if constexpr (MT::kWide) {
        Gemm g{};
        g.W = Wb + M.ofc1; g.ldw = M.ldX; g.nseg = 2; g.seg[0] = Seg{A.x2, R / 4};
        g.seg[1] = Seg{auxT + (size_t)2 * AUX * Bp, AUX / 4};
        wide_partials<NWG, U, UW, kUPC, 1>(part, g, g, tb, Bp, warp, lane);
      } else {
        stage_rows<NT>(stA, A.x2, R * G, tid);
        stage_rows<NT>(stA + R * G, auxT + (size_t)2 * AUX * Bp, AUX * G, tid);
        group_sync<GROUPS, NT>(grp);
        narrow_rows<G, 1>(nout, 0, Wb + M.ofc1, M.ldX, stA, M.ldX / 4, kUPC, 0, NWG, warp, lane);
      }
      group_sync<GROUPS, NT>(grp);
      const float* b = Wb + M.obfc1;
      for (int idx = tid; idx < BT * kUPC; idx += NT) {
        const int ul = idx % BT, j = idx / BT;
        A.f1[(size_t)(c * kUPC + j) * Bp + tb + ul] = fmaxf(part_sum<KS1, kUPC, BT>(res, 0, j, ul) + b[j], 0.f);
      }
      if (tb + BT < tb_hi) group_sync<GROUPS, NT>(grp);
    }
    PROF_MARK(6);
    if (!grid_barrier<GROUPS, NT>(bar_ctr, (++nbar) * ncta, A.error, grp, tid, s_ok)) return;
    PROF_MARK(7);

    // ================= P4: fc2 + relu =================
    for (int tb = tb_lo; tb < tb_hi; tb += BT) {
      if constexpr (MT::kWide) {
        Gemm g{};
        g.W = Wb + M.ofc2; g.ldw = M.ldF; g.nseg = 2; g.seg[0] = Seg{A.f1, F / 4};
        g.seg[1] = Seg{auxT + (size_t)3 * AUX * Bp, AUX / 4};
        wide_partials<NWG, U, UW, kUPC, 1>(part, g, g, tb, Bp, warp, lane);
      } else {
        stage_rows<NT>(stA, A.f1, F * G, tid);
        stage_rows<NT>(stA + F * G, auxT + (size_t)3 * AUX * Bp, AUX * G, tid);
        group_sync<GROUPS, NT>(grp);
        narrow_rows<G, 1>(nout, 0, Wb + M.ofc2, M.ldF, stA, M.ldF / 4, kUPC, 0, NWG, warp, lane);
      }
      group_sync<GROUPS, NT>(grp);
      const float* b = Wb + M.obfc2;
      for (int idx = tid; idx < BT * kUPC; idx += NT) {
        const int ul = idx % BT, j = idx / BT;
        A.f2[(size_t)(c * kUPC + j) * Bp + tb + ul] = fmaxf(part_sum<KS1, kUPC, BT>(res, 0, j, ul) + b[j], 0.f);
      }
      if (tb + BT < tb_hi) group_sync<GROUPS, NT>(grp);
    }
    PROF_MARK(8);
    if (!grid_barrier<GROUPS, NT>(bar_ctr, (++nbar) * ncta, A.error, grp, tid, s_ok)) return;
    PROF_MARK(9);

    // ================= P5: fc3 + distributed Gumbel-max sampling =================
    for (int tb = tb_lo; tb < tb_hi; tb += BT) {
      if constexpr (MT::kWide) {
        Gemm g{};
        g.W = Wb + M.ofc3; g.ldw = F; g.nseg = 1; g.seg[0] = Seg{A.f2, F / 4};
        wide_partials<NWG, U, UW, kCPC, 1>(part, g, g, tb, Bp, warp, lane);
      } else {
        stage_rows<NT>(stA, A.f2, F * G, tid);
        group_sync<GROUPS, NT>(grp);
        narrow_rows<G, 1>(nout, 0, Wb + M.ofc3, F, stA, F / 4, kCPC, 0, NWG, warp, lane);
      }
      group_sync<GROUPS, NT>(grp);
      const float* b = Wb + M.obfc3;
      for (int ul = tid; ul < BT; ul += NT) {
        const int u = tb + ul;
        if (u < A.B) {
          unsigned long long bestp = 0ull;
#pragma unroll
          for (int r4 = 0; r4 < kCPC / 4; ++r4) {
            float q[4];
            const int cls0 = c * kCPC + r4 * 4;
            if (A.rng_mode == 0) {
              philox_exp4(A.seed, A.utt_ids ? A.utt_ids[u] : A.utt_offset + (unsigned long long)u, (uint32_t)t, (uint32_t)(cls0 >> 2), q);
            } else {
              float4 qv = __ldg(reinterpret_cast<const float4*>(A.q + ((size_t)t * A.B + u) * M.NC + cls0));
              q[0] = qv.x; q[1] = qv.y; q[2] = qv.z; q[3] = qv.w;
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const int r = r4 * 4 + k;
              float l = part_sum<KS1, kCPC, BT>(res, 0, r, ul) + b[r];
              if (A.logits_out) A.logits_out[((size_t)t * A.B + u) * M.NC + cls0 + k] = l;
              unsigned long long p = pack_key(l - logf(q[k]), (uint32_t)(cls0 + k));
              bestp = p > bestp ? p : bestp;
            }
          }
          atomicMax(A.best + (size_t)(t & 1) * Bp + u, bestp);
        }
      }
      if (tb + BT < tb_hi) group_sync<GROUPS, NT>(grp);
    }
    PROF_MARK(10);
    if constexpr (kSplit >= 1) {                      // the wait sits in the next step's P01, after its GEMMs
      grid_arrive<GROUPS, NT>(bar_ctr, grp, tid);
      pend_target = (++nbar) * ncta;
      pending = true;
    } else {
      if (!grid_barrier<GROUPS, NT>(bar_ctr, (++nbar) * ncta, A.error, grp, tid, s_ok)) return;
      PROF_MARK(11);
    }
  }
  if (pending && !grid_wait<GROUPS, NT>(bar_ctr, pend_target, A.error, grp, tid, s_ok)) return;
  if (A.prof && grp == 0 && tid == 0)
    for (int i = 0; i < 12; ++i) A.prof[(size_t)c * 12 + i] = pf[i];
#undef PROF_MARK
  // the last step's winner
  if (c == 0 && A.steps > 0) {
    const int t = A.steps;
    for (int u = tb_lo + tid; u < tb_hi && u < A.B; u += NT) {
      unsigned long long pk = __ldcg(A.best + (size_t)((t - 1) & 1) * Bp + u);
      A.labels[(size_t)u * A.S + (t - 1)] = (int16_t)unpack_idx(pk);
    }
  }
}

// Instantiated here, ahead of wavernn_tc.cuh, so that this kernel is the module's first user of `smem`.  ptxas aligns an
// extern shared array to the largest alignment among those the module declares before it; declaring `smem` ahead of
// wavernn_tc_kernel's 1024-byte aligned `tsm` lets the grid and push kernels' weight blobs start right behind their static
// shared variables.
template __global__ void wavernn_grid_kernel<0, 4, 1>(GridModel, GridArgs);

// conditioning in the K-major layout the grid kernel streams: mels_T[t][c][u], aux_T[fr][o][u]
__global__ void mel_fir_T_kernel(const float* __restrict__ mel /*[B][feat][T]*/, const float* __restrict__ fir, int B, int Bp,
                                 int T, int feat, int hop, int pad, int NT, float* __restrict__ mels_T /*[S][feat][Bp]*/) {
  const size_t S = (size_t)T * hop, total = S * feat * Bp;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    int u = (int)(e % Bp);
    size_t rest = e / Bp;
    int c = (int)(rest % feat);
    size_t n = rest / feat;
    float acc = 0.f;
    if (u < B) {
      size_t np = n + (size_t)pad * hop;
      int fr = (int)(np / hop), ph = (int)(np % hop);
      for (int j = 0; j < NT; ++j) {
        int f = fr + j - NT / 2 - pad;
        if (f >= 0 && f < T) acc = fmaf(fir[ph * NT + j], mel[((size_t)u * feat + c) * T + f], acc);
      }
    }
    mels_T[e] = acc;
  }
}

__global__ void aux_T_kernel(const float* __restrict__ aux_frames /*[B][T][O]*/, int B, int Bp, int T, int O,
                             float* __restrict__ aux_T /*[T][O][Bp]*/) {
  const size_t total = (size_t)T * O * Bp;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    int u = (int)(e % Bp);
    size_t rest = e / Bp;
    int o = (int)(rest % O);
    size_t f = rest / O;
    aux_T[e] = u < B ? aux_frames[((size_t)u * T + f) * O + o] : 0.f;
  }
}

}  // namespace b200tts
