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
#include <algorithm>
#include <cstring>
#include <vector>
#include "common.cuh"
#include "wavernn_utt.cuh"

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

// MOL: the sample of row u at step n from the 30 parameters P5 stored (sample_from_discretized_mix_logistic, distribution.py:87-123);
// `out` stores it.  Returns the value fed back.
__device__ __forceinline__ float grid_mol_sample(const GridArgs& A, const MolIO& io, int u, int n, bool out) {
  const float* pp = io.par + ((size_t)(n & 1) * A.Bp + u) * 32;
  float p[kMolParams], uu[kMolU];
#pragma unroll
  for (int j = 0; j < kMolParams; ++j) p[j] = __ldcg(pp + j);
  if (A.rng_mode == 0) {
    philox_mol_u(A.seed, A.utt_ids ? A.utt_ids[u] : A.utt_offset + (unsigned long long)u, (uint32_t)n, uu);
  } else {
#pragma unroll
    for (int j = 0; j < kMolU; ++j) uu[j] = __ldg(A.q + ((size_t)n * A.B + u) * kMolU + j);
  }
  const float xs = mol_sample(p, uu);
  if (out) io.samples[(size_t)u * A.S + n] = xs;
  return io.teacher_x ? io.teacher_x[(size_t)u * A.S + n] : xs;
}

// The whole kernel; MOL selects the sampler.  MOL models are packed with fc3 parameter j as class 8j (create_context, wavernn.cu): in P5,
// CTA j < 30 stores parameter j of every row to io.par instead of joining the argmax race, and after the barrier every CTA
// reads the 30 parameters back and samples.
template <int U, int UW, int GROUPS>
__global__ void __launch_bounds__(MapTraits<U, UW, GROUPS>::NW * 32, 1) wavernn_grid_kernel(GridModel M, GridArgs A) {
  constexpr bool MOL = false;
  [[maybe_unused]] const MolIO io{};
#include "wavernn_grid_step.cuh"
}

template <int U, int UW, int GROUPS>
__global__ void __launch_bounds__(MapTraits<U, UW, GROUPS>::NW * 32, 1) wavernn_grid_mol_kernel(GridModel M, GridArgs A, MolIO io) {
  constexpr bool MOL = true;
#include "wavernn_grid_step.cuh"
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

// ---- host: the per-CTA weight blobs [ncta][blob], cut from the step weights in their original layouts (`w` points to host
//      memory).  Fills the layout `g`; g.ok says whether the model and device can run this kernel, and the blobs are empty
//      when they cannot. --------------------------------------------------------------------------------------------------
inline std::vector<float> pack_grid_model(const StepWeights& w, int sm_count, bool coop, GridModel& g) {
  const int R = w.R, F = w.F, AUX = w.aux, FEAT = w.feat, NC = w.NC, ldI = w.ldI;
  g = GridModel{};
  g.R = R; g.F = F; g.AUX = AUX; g.FEAT = FEAT; g.NC = NC;
  g.ldC = FEAT + AUX; g.ldX = R + AUX; g.ldF = F + AUX;
  g.ncta = R / kUPC;
  g.ok = (R == F) && (R % kUPC == 0) && (NC == g.ncta * kCPC) && (FEAT % 4 == 0) && (g.ncta <= sm_count) && coop;
  // the narrow mapping stages [x1|aux], [f1|aux], [mel|aux] in a 640*G-float area and h in a 512*G-float area
  if (R + AUX > 640 || F + AUX > 640 || FEAT + AUX > 640 || R > 512) g.ok = 0;
  int off = 0;
  auto take = [&](int n) { int o = off; off += (n + 3) & ~3; return o; };
  g.oA_w = take(16 * g.ldC); g.oA_x = take(16); g.oA_b = take(16);
  g.ohh1 = take(3 * kUPC * R); g.oih2 = take(3 * kUPC * g.ldX); g.ohh2 = take(3 * kUPC * R);
  g.ofc1 = take(kUPC * g.ldX); g.ofc2 = take(kUPC * g.ldF); g.ofc3 = take(kCPC * F);
  g.obhh1 = take(3 * kUPC); g.obih2 = take(3 * kUPC); g.obhh2 = take(3 * kUPC);
  g.obfc1 = take(kUPC); g.obfc2 = take(kUPC); g.obfc3 = take(kCPC);
  g.blob = off;
  constexpr int kMaxScratch = std::max({MapTraits<0, 4, 1>::kScratchFloats, MapTraits<1, 1, 1>::kScratchFloats,
                                        MapTraits<2, 1, 1>::kScratchFloats, MapTraits<4, 1, 1>::kScratchFloats,
                                        MapTraits<4, 1, 2>::kScratchFloats});   // every variant launch_grid can dispatch
  size_t smem_need = ((size_t)g.blob + (size_t)kMaxScratch) * sizeof(float) + 2048;
  if (smem_need > 227 * 1024) g.ok = 0;
  if (!g.ok) return {};

  std::vector<float> hb((size_t)g.ncta * g.blob, 0.f);
  std::vector<double> fold_acc(1 + g.ldC);
  for (int cta = 0; cta < g.ncta; ++cta) {
    float* b = &hb[(size_t)cta * g.blob];
    for (int j = 0; j < kUPC; ++j) {
      const int row = cta * kUPC + j;
      const float* src = w.I_w + (size_t)row * ldI;          // [x | feat | aux] padded
      b[g.oA_x + j] = src[0];
      std::memcpy(b + g.oA_w + (size_t)j * g.ldC, src + 1, sizeof(float) * g.ldC);
      b[g.oA_b + j] = w.I_b[row];
      std::memcpy(b + g.ofc1 + (size_t)j * g.ldX, w.fc1_w + (size_t)row * g.ldX, sizeof(float) * g.ldX);
      std::memcpy(b + g.ofc2 + (size_t)j * g.ldF, w.fc2_w + (size_t)row * g.ldF, sizeof(float) * g.ldF);
      b[g.obfc1 + j] = w.fc1_b[row];
      b[g.obfc2 + j] = w.fc2_b[row];
      for (int gate = 0; gate < 3; ++gate) {
        const int srow = gate * R + row, drow = gate * kUPC + j;
        // folded input projection of GRU 1: row srow of W_ih1.W_I (x column | cond columns) and W_ih1.b_I + b_ih1, in double
        const float* wr = w.ih1_w + (size_t)srow * R;
        double bacc = (double)w.ih1_b[srow];
        std::fill(fold_acc.begin(), fold_acc.end(), 0.0);
        for (int k = 0; k < R; ++k) {
          const double wk = (double)wr[k];
          const float* irow = w.I_w + (size_t)k * ldI;
          for (int col = 0; col < 1 + g.ldC; ++col) fold_acc[col] += wk * (double)irow[col];
          bacc += wk * (double)w.I_b[k];
        }
        b[g.oA_x + 4 + drow] = (float)fold_acc[0];
        for (int col = 0; col < g.ldC; ++col) b[g.oA_w + (size_t)(4 + drow) * g.ldC + col] = (float)fold_acc[1 + col];
        b[g.oA_b + 4 + drow] = (float)bacc;
        std::memcpy(b + g.ohh1 + (size_t)drow * R, w.hh1_w + (size_t)srow * R, sizeof(float) * R);
        std::memcpy(b + g.oih2 + (size_t)drow * g.ldX, w.ih2_w + (size_t)srow * g.ldX, sizeof(float) * g.ldX);
        std::memcpy(b + g.ohh2 + (size_t)drow * R, w.hh2_w + (size_t)srow * R, sizeof(float) * R);
        b[g.obhh1 + drow] = w.hh1_b[srow];
        b[g.obih2 + drow] = w.ih2_b[srow]; b[g.obhh2 + drow] = w.hh2_b[srow];
      }
    }
    for (int r = 0; r < kCPC; ++r) {
      const int row = cta * kCPC + r;
      std::memcpy(b + g.ofc3 + (size_t)r * F, w.fc3_w + (size_t)row * F, sizeof(float) * F);
      b[g.obfc3 + r] = w.fc3_b[row];
    }
  }
  return hb;
}

}  // namespace b200tts
