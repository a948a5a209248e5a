// WaveRNN per-sample recurrence on the Hopper tensor cores (wgmma, fp32 accumulators in registers): the large-batch
// (33 ... 256 rows per GPU) form of the reference loop wavernn/models/fatchord_version.py:201-237.
//
// LAYER-STATIONARY decomposition.  128 co-resident CTAs (one per SM; H100 has 132), each keeps a [N x 512] slice of ONE
// layer's weights in shared memory for the whole launch as the B operand of the MMA (K-major, no swizzle):
//     CTAs   0- 31  GRU-1 recurrent  W_hh1, 16 hidden units x (r, z, n) = 48 columns
//     CTAs  32- 95  GRU-2            W_ih2 and W_hh2, 8 units x (r, z, n) (+ 8 zero columns) = 32 + 32 columns
//     CTAs  96-103  fc1, 64 units    CTAs 104-111  fc2, 64 units    CTAs 112-127  fc3, 64 classes
// The batch is cut into groups of 128 rows; a group's activation vector [128 x 512] is the A operand.  Two consumer
// warpgroups per CTA each own 64 rows of a group (one M = 64 wgmma) and hold that slice of the accumulators in registers, so
// the thread that issues the MMA also does the gate math of the rows it accumulated.  The two groups of a 256-row batch flow
// through the layers as a pipeline: while group 0 is in fc1, group 1 is in GRU-2, and so on -- a CTA works on whichever group
// has reached its layer.
//
// EXACTNESS.  The tensor core has no fp32 operands; every fp32 value v (weights on the host, activations by the thread that
// produces them) is split into two fp16 planes, v = hi + lo' / 2048 with hi = fp16(v), lo' = fp16((v - hi) * 2048) (the scaling
// keeps lo' out of the fp16 subnormals), 22 mantissa bits in all.  a.w = hi.hi + (hi.lo' + lo'.hi) / 2048 (+ lo'.lo' / 2^22,
// dropped: below fp32 resolution): three f16 wgmma per k-step with fp32 accumulation.  The tensor-core accumulator does not
// round to nearest on every add, so the dominant hi.hi product is accumulated only over 8 k-steps (K = 128) at a time; the four
// chunk sums and the cross-term accumulator are added in fp32 registers (round to nearest).
//
// DATA FLOW.  A consumer thread owns two batch rows and a quarter of the CTA's columns (the wgmma accumulator fragment: rows
// r, r + 8, column pairs 8i + 2(lane % 4)).  After the gate math it stores its results ALREADY SPLIT and ALREADY in the
// canonical K-major layout into the vector's image in global memory (L2): [K/32 stages][plane][k-step][k half][16 row groups]
// [8 rows][8 halves] -- rows of a warp are contiguous.  Every consumer warp then releases one arrival on the per-(vector, group)
// counter (red.release.gpu, cumulative over the warp barrier; no block barrier on the critical path).  A consumer CTA's loader
// thread spins on the counter (ld.acquire.gpu), executes fence.proxy.async, and streams the 256 KB image through a ring of
// 16 KB shared-memory stages with cp.async.bulk; the two warpgroups issue six wgmma per stage and release the stage through
// its mbarrier once their products are done.  Vectors are double-buffered by step parity; the dependency chain of the
// recurrence itself guarantees that a buffer is rewritten only after every reader of its previous content has finished:
// parity p of a vector is rewritten at step t+2, and its producer reaches step t+2 only through the winner of step t+1, which
// needs every layer of step t+1 -- including each consumer of parity p, which finished its GEMM of step t first.
//
// What stays off the tensor cores, as in the push kernels (wavernn_push.cuh): the conditioning (per-frame tables, FIR linearity;
// GRU-1's 64 values per row come from 3 dedicated warps in blocks of <= 8 steps through a ring in L2), the sampled-label column of
// the I layer / GRU-1 (rank 1), the Gumbel-max race.  W_hh1.h1(t) and W_hh2.h2(t) run one step ahead, right after the
// CTA has published its own part of step t, and wait in registers for the gate math of step t+1.  Every wait is bounded
// (PollGuard, ~2 s) and raises the launch's error flag instead of hanging; a warpgroup that gave up keeps issuing its
// (meaningless) MMAs to the end of the GEMM so that the warps of a wgmma never diverge, and the consumers leave together.
#pragma once
#include <cuda_fp16.h>
#include <utility>
#include <vector>
#include "common.cuh"
#include "wavernn_push.cuh"

namespace b200tts {

constexpr int kTcConsumerWarps = 8;         // warps 0-3 / 4-7: the warpgroups of rows 0-63 / 64-127 of a group
constexpr int kTcLoaderWarp = 8;
constexpr int kTcCondWarp0 = 9;             // warps 9-11: conditioning (GRU-1 CTAs)
constexpr int kTcCondWarps = 3;
constexpr int kTcThreads = 12 * 32;         // 3 warps per SM sub-partition: 168 registers per thread at launch, then
constexpr int kTcConsumerRegs = 232;        // warpgroups 0-1 take what warpgroup 2 gives back (setmaxnreg):
constexpr int kTcOtherRegs = 40;            // 2 x 128 x (232 - 168) = 128 x (168 - 40)
constexpr int kTcRows = 128;                // rows per group
constexpr int kTcMaxGroups = 2;
constexpr int kTcStageBytes = 16384;        // K = 32 of one vector: [plane 2][k-step 2][k half 2][row group 16][8 rows][8 halves]
constexpr int kTcStagesPerVec = 16;
constexpr int kTcVecBytes = kTcStagesPerVec * kTcStageBytes;
constexpr int kTcCtas = 128;
constexpr int kTcWimgBytes = 131072;        // per-CTA weight image slot
constexpr int kTcPrm = 128;                 // per-CTA fp32 parameters
constexpr int kTcStages = 6;                // shared-memory ring (fc3: 4, its 32 KB of noise take the room of two stages)
constexpr int kTcWinCopies = 8;             // the winner words are written 8 times: 32 GRU-1 CTAs x 256 threads read them at the same moment
constexpr int kTcCondBlk = 8;               // GRU-1 conditioning is produced in blocks of <= 8 consecutive steps of one frame
constexpr int kTcCondSlot = kTcRows * 64;   // floats of one (step, group) of the conditioning ring
constexpr int kTcSmemBytes = kTcWimgBytes + kTcStages * kTcStageBytes + kTcPrm * 4;   // GRU-2 / fc CTAs (largest); GRU-1: 96 KB + stages + FIR
constexpr int kTcFirMaxBytes = kTcSmemBytes - (98304 + kTcStages * kTcStageBytes + kTcPrm * 4);
enum { TV_H1 = 0, TV_X1, TV_H2, TV_X2, TV_F1, TV_F2, TV_COUNT };
enum { TCN_C1 = 0, TCN_C2, TCN_F1, TCN_F2, TCN_W, TCN_COUNT = 8 };
enum { TC_ROLE_G1 = 0, TC_ROLE_G2, TC_ROLE_F1, TC_ROLE_F2, TC_ROLE_F3 };

struct TcArgs {
  const uint8_t* wimg;           // [128][kTcWimgBytes] fp16 B-operand images (packed by pack_tc_images below)
  const float* prm;              // [128][128]
  uint8_t* vec;                  // [TV_COUNT][ng][2][kTcVecBytes]
  float* x1f;                    // [ng][2][128][512] fp32 copy of x1 (GRU-2 CTAs add their h2 to it: x2 = x1 + h2)
  unsigned long long* winners;   // [ng][2][kTcWinCopies][128][16]
  unsigned* cnt;                 // [ng][TCN_COUNT][32] arrival counters (one 128-byte line each, one arrival per consumer WARP), zeroed before the launch
  float* condg;                  // [32 GRU-1 CTAs][2 block buffers][ng][kTcCondBlk][128 rows][64] conditioning ring (stays in L2)
  int* error;
  const float* tab;              // [B][T+1][128][52] conditioning tables (push_cond_table_kernel)
  const float* fir;              // [hop][NT]
  int NT, B, S, T, hop, steps, ng, NC;
  int rng_mode;
  unsigned long long seed, utt_offset;
  const unsigned long long* utt_ids;
  const float* q;                // [S][B][NC]
  const int16_t* teacher;        // [B][S]
  float* logits_out;             // [S][B][NC]
  int16_t* labels;               // [B][S]
  long long* prof;               // optional [128][12] cycle counters (B200TTS_GRID_PROF): slots 3 (role - 1) + {exchange wait,
                                 // GEMM, epilogue} of one job per (step, group) -- GRU-2's x1 job, fc1, fc2, fc3 -- summed by thread 0
};

// ---- small PTX wrappers ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t tc_smem(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ unsigned tc_ld_acquire(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void tc_red_release(unsigned* p, unsigned v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void tc_mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(tc_smem(bar)) : "memory");
}
// bounded wait: false when the launch has been aborted (a peer timed out) or after ~2 s
__device__ __forceinline__ bool tc_mbar_wait(unsigned long long* bar, unsigned parity, PollGuard& pg) {
  if (pg.aborted) return false;
  const uint32_t a = tc_smem(bar);
  pg.begin();
  while (true) {
    unsigned done;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
                 : "=r"(done) : "r"(a), "r"(parity) : "memory");
    if (done) return true;
    if (pg.expired()) return false;
  }
}
__device__ __forceinline__ bool tc_cnt_wait(const unsigned* p, unsigned need, PollGuard& pg) {
  if (pg.aborted) return false;
  pg.begin();
  while (true) {
    if (tc_ld_acquire(p) >= need) return true;
    if (pg.expired()) return false;
  }
}
// the same for a whole (converged) warp: lane 0 polls, the warp barrier passes the acquired view on -- 32x fewer requests on
// the counter's L2 line (thousands of threads wait on the same few lines at the same moment)
__device__ __forceinline__ bool tc_cnt_wait_warp(const unsigned* p, unsigned need, PollGuard& pg, int lane) {
  bool ok = true;
  if (lane == 0) ok = tc_cnt_wait(p, need, pg);
  ok = __shfl_sync(0xffffffffu, ok ? 1 : 0, 0) != 0;
  __syncwarp();                             // memory ordering among the lanes: they read (ld.cg) what lane 0 acquired
  if (!ok) pg.aborted = true;
  return ok;
}
// wgmma shared-memory matrix descriptor, K-major, no swizzle: core matrix = 8 rows x 16 bytes; LBO = stride between the two
// K halves of one k-step, SBO = stride between 8-row groups (PTX ISA, "Matrix Descriptor Format" of wgmma)
__device__ __forceinline__ uint64_t tc_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)(lbo_bytes >> 4) << 16;
  d |= (uint64_t)(sbo_bytes >> 4) << 32;
  return d;
}
// D[64 x N] (+)= A[64 x 16] . B[16 x N], f16 operands from shared memory, fp32 accumulators in registers (ACC = 0 overwrites
// D).  Fragment of a thread: D[4i + 2h + e] = (row 16 * (warp % 4) + lane / 4 + 8h, column 8i + 2 (lane % 4) + e).
// The descriptors are da + AOFF and db + BOFF, added inside the asm: as plain C++ sums of loop-invariant bases the 64 B-operand
// descriptors of a GEMM would be hoisted out of the step loop and held in registers for the whole launch.
// Operands: DREGS, then da, db, AOFF, BOFF, ACC (I0 ... I0 + 4).
#define TC_WGMMA_ASM(SHAPE, DREGS, A, B, AO, BO, ACC)                                                                            \
  "{\n\t.reg .pred p;\n\t.reg .b64 da, db;\n\tsetp.ne.b32 p, " ACC ", 0;\n\t"                                                \
  "add.s64 da, " A ", " AO ";\n\tadd.s64 db, " B ", " BO ";\n\t"                                                                 \
  "wgmma.mma_async.sync.aligned." SHAPE ".f32.f16.f16 {" DREGS "}, da, db, p, 1, 1, 0, 0;\n\t}\n"
template <int AOFF, int BOFF, int ACC>
__device__ __forceinline__ void tc_wgmma32(float (&d)[16], uint64_t da, uint64_t db) {
  asm volatile(TC_WGMMA_ASM("m64n32k16", "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15",
                            "%16", "%17", "%18", "%19", "%20")
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "n"(AOFF), "n"(BOFF), "n"(ACC));
}
template <int AOFF, int BOFF, int ACC>
__device__ __forceinline__ void tc_wgmma48(float (&d)[24], uint64_t da, uint64_t db) {
  asm volatile(TC_WGMMA_ASM("m64n48k16", "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23",
                            "%24", "%25", "%26", "%27", "%28")
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
      : "l"(da), "l"(db), "n"(AOFF), "n"(BOFF), "n"(ACC));
}
template <int AOFF, int BOFF, int ACC>
__device__ __forceinline__ void tc_wgmma64(float (&d)[32], uint64_t da, uint64_t db) {
  asm volatile(TC_WGMMA_ASM("m64n64k16", "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31",
                            "%32", "%33", "%34", "%35", "%36")
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "n"(AOFF), "n"(BOFF), "n"(ACC));
}
#undef TC_WGMMA_ASM
template <int R>
__device__ __forceinline__ void tc_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int N, int AOFF, int BOFF, int ACC>
__device__ __forceinline__ void tc_wgmma(float (&d)[N / 2], uint64_t da, uint64_t db) {
  if constexpr (N == 32) tc_wgmma32<AOFF, BOFF, ACC>(d, da, db);
  else if constexpr (N == 48) tc_wgmma48<AOFF, BOFF, ACC>(d, da, db);
  else tc_wgmma64<AOFF, BOFF, ACC>(d, da, db);
}
__device__ __forceinline__ void tc_wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void tc_wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int P>
__device__ __forceinline__ void tc_wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(P) : "memory"); }

// fp32 -> (hi, lo') fp16 planes, 8 values -> one 16-byte word per plane
__device__ __forceinline__ void tc_split8(const float* v, uint4& hi, uint4& lo) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const __half a = __float2half_rn(v[2 * i]), b = __float2half_rn(v[2 * i + 1]);
    const __half al = __float2half_rn((v[2 * i] - __half2float(a)) * 2048.0f);
    const __half bl = __float2half_rn((v[2 * i + 1] - __half2float(b)) * 2048.0f);
    h[i] = (uint32_t)__half_as_ushort(a) | ((uint32_t)__half_as_ushort(b) << 16);
    l[i] = (uint32_t)__half_as_ushort(al) | ((uint32_t)__half_as_ushort(bl) << 16);
  }
  hi = make_uint4(h[0], h[1], h[2], h[3]);
  lo = make_uint4(l[0], l[1], l[2], l[3]);
}
// where the 8 halves k = 8*k8 ... 8*k8+7 of row `row` live inside a vector image (bytes); plane 1 is + 8192
__device__ __forceinline__ uint32_t tc_img_off(int k8, int row) {
  const int kstep = k8 >> 1, ki = k8 & 1;
  return (uint32_t)(kstep >> 1) * kTcStageBytes + (uint32_t)(kstep & 1) * 4096u + (uint32_t)ki * 2048u + (uint32_t)(row >> 3) * 128u +
         (uint32_t)(row & 7) * 16u;
}
// units k0, k0 + 1 (k0 even) of row `row`: one 32-bit word per plane
__device__ __forceinline__ void tc_store2(uint8_t* img, int k0, int row, float v0, float v1) {
  const __half a = __float2half_rn(v0), b = __float2half_rn(v1);
  const __half al = __float2half_rn((v0 - __half2float(a)) * 2048.0f);
  const __half bl = __float2half_rn((v1 - __half2float(b)) * 2048.0f);
  uint8_t* p = img + tc_img_off(k0 >> 3, row) + (uint32_t)(k0 & 7) * 2u;
  *reinterpret_cast<uint32_t*>(p) = (uint32_t)__half_as_ushort(a) | ((uint32_t)__half_as_ushort(b) << 16);
  *reinterpret_cast<uint32_t*>(p + 8192) = (uint32_t)__half_as_ushort(al) | ((uint32_t)__half_as_ushort(bl) << 16);
}

struct TcRoleInfo {
  int role, ci;            // role, index inside the role
  int njobs;               // GEMMs per (step, group)
  int nstage;              // shared-memory stages
  int wbytes;              // weight image bytes
};
__host__ __device__ __forceinline__ TcRoleInfo tc_role(int cta) {
  TcRoleInfo r;
  if (cta < 32) { r.role = TC_ROLE_G1; r.ci = cta; r.njobs = 1; r.nstage = kTcStages; r.wbytes = 98304; }
  else if (cta < 96) { r.role = TC_ROLE_G2; r.ci = cta - 32; r.njobs = 2; r.nstage = kTcStages; r.wbytes = 131072; }
  else if (cta < 104) { r.role = TC_ROLE_F1; r.ci = cta - 96; r.njobs = 1; r.nstage = kTcStages; r.wbytes = 131072; }
  else if (cta < 112) { r.role = TC_ROLE_F2; r.ci = cta - 104; r.njobs = 1; r.nstage = kTcStages; r.wbytes = 131072; }
  else { r.role = TC_ROLE_F3; r.ci = cta - 112; r.njobs = 1; r.nstage = 4; r.wbytes = 131072; }
  return r;
}
// job j of a role: which vector it multiplies, which counter announces it, how many arrivals (8 consumer warps per producer CTA) fill it
__device__ __forceinline__ void tc_job(int role, int j, int& vec, int& cnt, int& nprod) {
  switch (role) {
    case TC_ROLE_G1: vec = TV_H1; cnt = TCN_C1; nprod = 32 * kTcConsumerWarps; break;
    case TC_ROLE_G2: if (j == 0) { vec = TV_X1; cnt = TCN_C1; nprod = 32 * kTcConsumerWarps; } else { vec = TV_H2; cnt = TCN_C2; nprod = 64 * kTcConsumerWarps; } break;
    case TC_ROLE_F1: vec = TV_X2; cnt = TCN_C2; nprod = 64 * kTcConsumerWarps; break;
    case TC_ROLE_F2: vec = TV_F1; cnt = TCN_F1; nprod = 8 * kTcConsumerWarps; break;
    default: vec = TV_F2; cnt = TCN_F2; nprod = 8 * kTcConsumerWarps; break;
  }
}

// OR of `flag` over the 8 consumer warps (named barrier 1): they all leave a loop at the same point
__device__ __forceinline__ bool tc_consumers_any(bool flag) {
  unsigned any;
  asm volatile("{\n\t.reg .pred p, q;\n\tsetp.ne.u32 q, %1, 0;\n\tbar.red.or.pred p, 1, %2, q;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
               : "=r"(any) : "r"(flag ? 1u : 0u), "n"(kTcConsumerWarps * 32) : "memory");
  return any != 0;
}

// The stage ring as one consumer warp sees it: the slot of its next stage, that slot's fill parity, the slot it consumed last.
struct TcRing {
  unsigned long long* full;
  unsigned long long* empty;
  unsigned nstage, slot, parity, prev;
  int lane;
  // each consumer warp releases a stage (one of kTcConsumerWarps arrivals) once its products are done
  __device__ __forceinline__ void release(unsigned sl) const {
    __syncwarp();
    if (lane == 0) tc_mbar_arrive(&empty[sl]);
  }
};
// Stage KS (K = 32, k-steps 2 KS and 2 KS + 1) of tc_gemm.  Everything that depends on KS -- the accumulate flags, the fold at the
// end of a K = 128 chunk, which waits and releases follow -- is fixed at compile time: the code between a wgmma and its wait
// has no branch, so the MMAs stay asynchronous (the previous stage's products overlap this stage's wait and issue).
template <int N, int KS>
__device__ __forceinline__ void tc_gemm_stage(float (&out)[N / 2], float (&acc)[N / 2], float (&crs)[N / 2], uint64_t dA0, uint64_t dB, TcRing& r,
                                              PollGuard& pg) {
  constexpr int K0 = 2 * KS, BT = N * 2;                // B tile of one k-step: N * 32 bytes = N * 2 descriptor units
  const unsigned sl = r.slot;
  tc_mbar_wait(&r.full[sl], r.parity, pg);              // after an abort: no wait, the MMAs below still run (on stale data)
  const uint64_t dA = dA0 + (uint64_t)(sl * (unsigned)(kTcStageBytes >> 4));
  tc_fence_regs(acc);
  tc_fence_regs(crs);
  tc_wg_fence();
  // A: hi plane at + 0, lo plane at + 8192 bytes, k half h at + 4096 h;  B: hi k-step K at K * N * 32, lo at (32 + K) * N * 32
  tc_wgmma<N, 0, K0 * BT, (K0 & 7) ? 1 : 0>(acc, dA, dB);
  tc_wgmma<N, 0, (32 + K0) * BT, K0 ? 1 : 0>(crs, dA, dB);
  tc_wgmma<N, 512, K0 * BT, 1>(crs, dA, dB);
  tc_wgmma<N, 256, (K0 + 1) * BT, 1>(acc, dA, dB);
  tc_wgmma<N, 256, (33 + K0) * BT, 1>(crs, dA, dB);
  tc_wgmma<N, 768, (K0 + 1) * BT, 1>(crs, dA, dB);
  tc_wg_commit();
  if constexpr ((KS & 3) == 3) {                        // end of a K = 128 chunk: fold its hi.hi sum into out
    tc_wg_wait<0>();
    tc_fence_regs(acc);
    tc_fence_regs(crs);
#pragma unroll
    for (int i = 0; i < N / 2; ++i) out[i] = KS == 3 ? acc[i] : __fadd_rn(out[i], acc[i]);
    r.release(r.prev);
    r.release(sl);
  } else if constexpr ((KS & 3) != 0) {                 // the previous stage's products are done
    tc_wg_wait<1>();
    r.release(r.prev);
  }
  r.prev = sl;
  if (++r.slot == r.nstage) { r.slot = 0; r.parity ^= 1u; }
}
template <int N, int... KS>
__device__ __forceinline__ void tc_gemm_stages(float (&out)[N / 2], float (&acc)[N / 2], float (&crs)[N / 2], uint64_t dA0, uint64_t dB, TcRing& r,
                                               PollGuard& pg, std::integer_sequence<int, KS...>) {
  (tc_gemm_stage<N, KS>(out, acc, crs, dA0, dB, r, pg), ...);
}
// One GEMM of this warpgroup's 64 rows: out[N/2] = A (the vector image streamed through the stage ring) . W (image at w_saddr),
// K = 512, as ((c0 + c1) + c2) + c3 + cross / 2048 with c_k the hi.hi products of k-steps 8k ... 8k+7.  `s` counts the stages
// consumed by this CTA.
template <int N>
__device__ __forceinline__ void tc_gemm(float (&out)[N / 2], uint32_t st0, uint32_t w_saddr, unsigned nstage, unsigned& s, unsigned long long* bar_full,
                                        unsigned long long* bar_empty, int wg, int lane, PollGuard& pg) {
  float acc[N / 2], crs[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) { acc[i] = 0.f; crs[i] = 0.f; }
  const uint64_t dB = tc_desc(w_saddr, (uint32_t)(N / 8) * 128u, 128u);
  const uint64_t dA0 = tc_desc(st0 + (uint32_t)wg * 1024u, 2048u, 128u);      // this warpgroup's 8 row groups
  TcRing r{bar_full, bar_empty, nstage, s % nstage, (s / nstage) & 1u, 0u, lane};
  tc_gemm_stages<N>(out, acc, crs, dA0, dB, r, pg, std::make_integer_sequence<int, kTcStagesPerVec>{});
  s += kTcStagesPerVec;
#pragma unroll
  for (int i = 0; i < N / 2; ++i) out[i] = __fadd_rn(out[i], crs[i] * (1.0f / 2048.0f));
  // every column counts as used: when a caller ignores some (GRU-2's zero columns), ptxas otherwise frees their accumulator
  // registers inside the MMA chain and serializes every wgmma of the kernel (C7511)
  tc_fence_regs(out);
}

__global__ void __launch_bounds__(kTcThreads, 1) wavernn_tc_kernel(TcArgs A) {
  extern __shared__ __align__(1024) uint8_t tsm[];
  __shared__ __align__(8) unsigned long long bar_full[kTcStages], bar_empty[kTcStages], bar_condfull[2], bar_condempty[2], bar_w;
  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);     // provably warp-uniform: the role branches hold wgmma
  const TcRoleInfo R = tc_role(blockIdx.x);
  const int ng = A.ng;
  uint8_t* Wsm = tsm;
  uint8_t* stages = tsm + R.wbytes;
  float* prm = reinterpret_cast<float*>(stages + (size_t)R.nstage * kTcStageBytes);
  float* fir_s = prm + kTcPrm;                         // GRU-1 CTAs only: [hop][NT]
  float* noise_s = prm + kTcPrm;                       // fc3 CTAs only: [32][256 consumer threads] log q

  if (tid == 0) {
    for (int i = 0; i < kTcStages; ++i) { mbar_init(&bar_full[i], 1); mbar_init(&bar_empty[i], kTcConsumerWarps); }
    for (int i = 0; i < 2; ++i) { mbar_init(&bar_condfull[i], kTcCondWarps); mbar_init(&bar_condempty[i], kTcConsumerWarps); }
    mbar_init(&bar_w, 1);
  }
  for (int i = tid; i < kTcPrm; i += kTcThreads) prm[i] = A.prm[(size_t)blockIdx.x * kTcPrm + i];
  if (R.role == TC_ROLE_G1)
    for (int i = tid; i < A.hop * A.NT; i += kTcThreads) fir_s[i] = A.fir[i];
  __syncthreads();
  if (tid == 0) {
    mbar_expect_tx(&bar_w, (unsigned)R.wbytes);
    const uint8_t* src = A.wimg + (size_t)blockIdx.x * kTcWimgBytes;
    for (int off = 0; off < R.wbytes; off += 32768) tma_bulk_g2s(Wsm + off, src + off, 32768u, &bar_w);
  }
  mbar_wait(&bar_w, 0);
  __syncthreads();
  PollGuard pg{A.error, 0, 0, false};
  auto vec_img = [&](int v, int g, int par) { return A.vec + (((size_t)v * ng + g) * 2 + par) * (size_t)kTcVecBytes; };
  auto counter = [&](int g, int which) { return A.cnt + ((size_t)g * TCN_COUNT + which) * 32; };

  // registers: the consumer warpgroups hold the accumulators of asynchronous MMAs, warpgroup 2 (loader + conditioning) little.
  // setmaxnreg is executed by all warps of a warpgroup, and ptxas budgets each branch by the value it starts with.
  if (warp < kTcConsumerWarps) {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kTcConsumerRegs));
    // ================= consumers: MMA + gate math; rows ra, rb = ra + 8 of the group, column pairs 8i + 2c ================
    const int wg = warp >> 2, c = lane & 3;
    const int ra = 64 * wg + 16 * (warp & 3) + (lane >> 2);
    const int rows[2] = {ra, ra + 8};
    const float ncls_m1 = (float)(A.NC - 1);
    const uint32_t w0 = tc_smem(Wsm), st0 = tc_smem(stages);
    const unsigned ns = (unsigned)R.nstage;
    unsigned s = 0;
    // One arrival per WARP: its rows are stored -> lane 0 releases (red.release.gpu is cumulative over what the warp barrier
    // ordered before it).  No block barrier on the critical path; the warp also agrees on giving up.
    auto publish = [&](int g, int which) {
      // (the generic -> async proxy fence of this exchange is executed by the CONSUMER's loader thread, after its acquire)
      if (__any_sync(0xffffffffu, pg.aborted)) { pg.aborted = true; return; }
      if (lane == 0) tc_red_release(counter(g, which), 1u);
    };
    // phase counters (A.prof): stamp(-1) opens a job, stamp(p) adds the cycles since the last stamp to phase p.  Every consumer
    // thread reads the clock, so no branch depends on the thread; all stamps sit between GEMMs, none inside a wgmma span.
    long long pf[3] = {0, 0, 0}, pt = 0;
    auto stamp = [&](int p) {
      if (A.prof) {
        const long long now = clock64();
        if (p >= 0) pf[p] += now - pt;
        pt = now;
      }
    };
    auto stamp_first_full = [&]() {                   // end of the exchange wait: the job's first stage is full
      if (A.prof) {
        tc_mbar_wait(&bar_full[s % ns], (s / ns) & 1u, pg);
        stamp(0);
      }
    };

    if (R.role == TC_ROLE_G1) {
      // units of this thread: q = 0..3 -> 2c, 2c+1, 2c+8, 2c+9; gate `gate` of unit q sits at fragment 4 (2 gate + q/2) + 2 h + q%2
      int uq[4] = {2 * c, 2 * c + 1, 2 * c + 8, 2 * c + 9};
      float h1own[kTcMaxGroups][8], ghs[kTcMaxGroups][24];     // ghs: W_hh1 . h1(t-1) in fragment order (0 at t = 0)
#pragma unroll
      for (int g = 0; g < kTcMaxGroups; ++g) {
#pragma unroll
        for (int i = 0; i < 8; ++i) h1own[g][i] = 0.f;
#pragma unroll
        for (int i = 0; i < 24; ++i) ghs[g][i] = 0.f;
      }
      const float* Ax = prm;                               // [4 kinds][16]
      const float* bhh = prm + 64;                         // [3 gates][16]
      int blk_t0 = 0, blk_t1 = 0, blk_i = -1;               // current conditioning block: steps [blk_t0, blk_t1) of all groups
      const float* cring = A.condg + (size_t)R.ci * 2 * ng * kTcCondBlk * kTcCondSlot;
      for (int t = 0; t <= A.steps; ++t) {
        if (t < A.steps && t == blk_t1) {
          blk_t0 = t;
          blk_t1 = min(min(t + kTcCondBlk, (t / A.hop + 1) * A.hop), A.steps);
          ++blk_i;
          tc_mbar_wait(&bar_condfull[blk_i & 1], (unsigned)(blk_i >> 1) & 1u, pg);
        }
#pragma unroll
        for (int g = 0; g < kTcMaxGroups; ++g) {
          if (g >= ng) continue;
          // this thread's conditioned values of (t, g) (4 kinds x 4 units x 2 rows): issued before the winner wait
          float cd[2][4][4];
          if (t < A.steps) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const float* cp = cring + ((size_t)((blk_i & 1) * ng + g) * kTcCondBlk + (t - blk_t0)) * kTcCondSlot + (size_t)rows[h] * 64 + 2 * c;
#pragma unroll
              for (int kind = 0; kind < 4; ++kind) {
                const float2 v0 = __ldcg(reinterpret_cast<const float2*>(cp + kind * 16));
                const float2 v1 = __ldcg(reinterpret_cast<const float2*>(cp + kind * 16 + 8));
                cd[h][kind][0] = v0.x; cd[h][kind][1] = v0.y; cd[h][kind][2] = v1.x; cd[h][kind][3] = v1.y;
              }
            }
          }
          float x[2] = {0.f, 0.f};
          if (t > 0) {
            tc_cnt_wait_warp(counter(g, TCN_W), (unsigned)(16 * kTcConsumerWarps) * (unsigned)t, pg, lane);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int row = rows[h], grow = g * kTcRows + row;
              const unsigned long long* wp = A.winners + ((((size_t)g * 2 + ((t - 1) & 1)) * kTcWinCopies + (R.ci & (kTcWinCopies - 1))) * kTcRows + row) * 16;
              unsigned long long best = 0ull;
#pragma unroll
              for (int i = 0; i < 16; i += 2) {
                const ulonglong2 w2 = __ldcg(reinterpret_cast<const ulonglong2*>(wp + i));
                best = w2.x > best ? w2.x : best;
                best = w2.y > best ? w2.y : best;
              }
              const int label = (int)push_cls(best);
              if (grow < A.B) {
                if (R.ci == 0 && c == 0) A.labels[(size_t)grow * A.S + (t - 1)] = (int16_t)label;
                const int fb = A.teacher ? (int)A.teacher[(size_t)grow * A.S + (t - 1)] : label;
                x[h] = label_to_float(fb, ncls_m1);
              }
            }
          }
          if (t == A.steps) continue;                      // the extra trip only collects the last winner
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float hnew[4], x1[4];
#pragma unroll
            for (int qi = 0; qi < 4; ++qi) {
              const int u = uq[qi], f = 4 * (qi >> 1) + 2 * h + (qi & 1);
              const float iout = fmaf(Ax[u], x[h], cd[h][0][qi]);
              const float gir = fmaf(Ax[16 + u], x[h], cd[h][1][qi]);
              const float giz = fmaf(Ax[32 + u], x[h], cd[h][2][qi]);
              const float gin = fmaf(Ax[48 + u], x[h], cd[h][3][qi]);
              const float hv = gru_update(gir, giz, gin, ghs[g][f] + bhh[u], ghs[g][8 + f] + bhh[16 + u], ghs[g][16 + f] + bhh[32 + u],
                                          h1own[g][4 * h + qi]);
              h1own[g][4 * h + qi] = hv;
              hnew[qi] = hv;
              x1[qi] = iout + hv;
            }
            const int row = rows[h];
            tc_store2(vec_img(TV_H1, g, t & 1), 16 * R.ci + 2 * c, row, hnew[0], hnew[1]);
            tc_store2(vec_img(TV_H1, g, t & 1), 16 * R.ci + 2 * c + 8, row, hnew[2], hnew[3]);
            tc_store2(vec_img(TV_X1, g, t & 1), 16 * R.ci + 2 * c, row, x1[0], x1[1]);
            tc_store2(vec_img(TV_X1, g, t & 1), 16 * R.ci + 2 * c + 8, row, x1[2], x1[3]);
            float* xf = A.x1f + (((size_t)g * 2 + (t & 1)) * kTcRows + row) * 512 + 16 * R.ci + 2 * c;
            *reinterpret_cast<float2*>(xf) = make_float2(x1[0], x1[1]);
            *reinterpret_cast<float2*>(xf + 8) = make_float2(x1[2], x1[3]);
          }
          publish(g, TCN_C1);
          // W_hh1 . h1(t) (the GEMM all GRU-1 CTAs start once h1(t) is complete) waits in registers for the gate math of step t+1
          tc_gemm<48>(ghs[g], st0, w0, ns, s, bar_full, bar_empty, wg, lane, pg);
        }
        if (tc_consumers_any(pg.aborted)) break;
        if (t < A.steps && t == blk_t1 - 1) {                // the block's values are all in registers / used: one arrival per warp
          __syncwarp();
          if (lane == 0) tc_mbar_arrive(&bar_condempty[blk_i & 1]);
        }
      }
    } else if (R.role == TC_ROLE_G2) {
      // units of this thread: 2c, 2c+1; gate `gate` at fragment 4 gate + 2 h + e
      float h2own[kTcMaxGroups][4], ghs[kTcMaxGroups][16];
#pragma unroll
      for (int g = 0; g < kTcMaxGroups; ++g) {
#pragma unroll
        for (int i = 0; i < 4; ++i) h2own[g][i] = 0.f;
#pragma unroll
        for (int i = 0; i < 16; ++i) ghs[g][i] = 0.f;
      }
      const float* bhh = prm;                              // [3 gates][8]
      for (int t = 0; t < A.steps; ++t) {
        const int fr = t / A.hop;
#pragma unroll
        for (int g = 0; g < kTcMaxGroups; ++g) {
          if (g >= ng) continue;
          // conditioning (aux projection + bias of the three gates, constant within a frame): table rows 32 + gate*4 + unit%4
          float cd[2][3][2];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int src = min(g * kTcRows + rows[h], A.B - 1);
            const float* tb = A.tab + (((size_t)src * (A.T + 1) + fr) * 128 + 2 * R.ci + (c >> 1)) * kPushCondRows + 32 + 2 * (c & 1);
#pragma unroll
            for (int gate = 0; gate < 3; ++gate) {
              const float2 v = __ldg(reinterpret_cast<const float2*>(tb + gate * 4));
              cd[h][gate][0] = v.x; cd[h][gate][1] = v.y;
            }
          }
          stamp(-1);
          // own units of x1 (fp32), loaded while the GEMM runs.  The counter is the one this CTA's loader waits for before the
          // GEMM's first stage; the warp's own acquire of it orders the loads.
          tc_cnt_wait_warp(counter(g, TCN_C1), (unsigned)(32 * kTcConsumerWarps) * (unsigned)(t + 1), pg, lane);
          float2 x1v[2];
#pragma unroll
          for (int h = 0; h < 2; ++h)
            x1v[h] = __ldcg(reinterpret_cast<const float2*>(A.x1f + (((size_t)g * 2 + (t & 1)) * kTcRows + rows[h]) * 512 + 8 * R.ci + 2 * c));
          float gi[16];
          stamp_first_full();
          tc_gemm<32>(gi, st0, w0, ns, s, bar_full, bar_empty, wg, lane, pg);      // W_ih2 . x1(t)
          stamp(1);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = rows[h];
            const float x1[2] = {x1v[h].x, x1v[h].y};
            float hnew[2], x2[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int u = 2 * c + e, f = 2 * h + e;
              const float hv = gru_update(gi[f] + cd[h][0][e], gi[4 + f] + cd[h][1][e], gi[8 + f] + cd[h][2][e], ghs[g][f] + bhh[u],
                                          ghs[g][4 + f] + bhh[8 + u], ghs[g][8 + f] + bhh[16 + u], h2own[g][2 * h + e]);
              h2own[g][2 * h + e] = hv;
              hnew[e] = hv;
              x2[e] = x1[e] + hv;
            }
            tc_store2(vec_img(TV_H2, g, t & 1), 8 * R.ci + 2 * c, row, hnew[0], hnew[1]);
            tc_store2(vec_img(TV_X2, g, t & 1), 8 * R.ci + 2 * c, row, x2[0], x2[1]);
          }
          publish(g, TCN_C2);
          stamp(2);
          // W_hh2 . h2(t) for step t+1
          tc_gemm<32>(ghs[g], st0, w0 + 65536u, ns, s, bar_full, bar_empty, wg, lane, pg);
        }
        if (tc_consumers_any(pg.aborted)) break;
      }
    } else if (R.role == TC_ROLE_F1 || R.role == TC_ROLE_F2) {
      // units of this thread: 8i + 2c + e, i = 0..7
      const int trow = R.role == TC_ROLE_F1 ? 44 : 48;     // table rows of the aux projection + bias: fc1 44-47, fc2 48-51
      const int vout = R.role == TC_ROLE_F1 ? TV_F1 : TV_F2, cout = R.role == TC_ROLE_F1 ? TCN_F1 : TCN_F2;
      for (int t = 0; t < A.steps; ++t) {
        const int fr = t / A.hop;
        for (int g = 0; g < ng; ++g) {
          stamp(-1);
          // aux projection + bias of this thread's units, loaded while the GEMM runs (the first step of a frame misses L2)
          float2 cd[2][8];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int src = min(g * kTcRows + rows[h], A.B - 1);
            const float* tb = A.tab + (((size_t)src * (A.T + 1) + fr) * 128 + 16 * R.ci + (c >> 1)) * kPushCondRows + trow + 2 * (c & 1);
#pragma unroll
            for (int i = 0; i < 8; ++i) cd[h][i] = __ldg(reinterpret_cast<const float2*>(tb + (size_t)(2 * i) * kPushCondRows));
          }
          float a[32];
          stamp_first_full();
          tc_gemm<64>(a, st0, w0, ns, s, bar_full, bar_empty, wg, lane, pg);
          stamp(1);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int i = 0; i < 8; ++i)
              tc_store2(vec_img(vout, g, t & 1), 64 * R.ci + 8 * i + 2 * c, rows[h], fmaxf(a[4 * i + 2 * h] + cd[h][i].x, 0.f),
                        fmaxf(a[4 * i + 2 * h + 1] + cd[h][i].y, 0.f));
          }
          publish(g, cout);
          stamp(2);
          if (tc_consumers_any(pg.aborted)) { pg.aborted = true; break; }
        }
        if (pg.aborted) break;
      }
    } else {
      // ---- fc3 + Gumbel-max: 16 of this CTA's 64 classes per row and thread, the 4 threads of a row meet by shuffles ----
      const float* b3 = prm;
      for (int t = 0; t < A.steps; ++t) {
        for (int g = 0; g < ng; ++g) {
          // noise first: it does not depend on the accumulators (log q of class 64 ci + 8i + 2c + e, fragment order); it waits
          // for the GEMM in this thread's own shared-memory slot, the registers go to the accumulators
          float* nl = noise_s + tid;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int grow = g * kTcRows + rows[h];
            const bool live = grow < A.B;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int cls = 64 * R.ci + 8 * i + 2 * c;
              float n0 = 0.f, n1 = 0.f;
              if (live && A.rng_mode == 0) {
                const unsigned long long uid = A.utt_ids ? A.utt_ids[grow] : A.utt_offset + (unsigned long long)grow;
                float q4[4];
                philox_exp4(A.seed, uid, (uint32_t)t, (uint32_t)(cls >> 2), q4);
                n0 = logf((c & 1) ? q4[2] : q4[0]);          // this thread's two of the four classes
                n1 = logf((c & 1) ? q4[3] : q4[1]);
              } else if (live) {
                const float2 v = __ldg(reinterpret_cast<const float2*>(A.q + ((size_t)t * A.B + grow) * A.NC + cls));
                n0 = logf(v.x); n1 = logf(v.y);
              }
              nl[(4 * i + 2 * h) * 256] = n0;
              nl[(4 * i + 2 * h + 1) * 256] = n1;
            }
          }
          float l[32];
          stamp(-1);
          stamp_first_full();
          tc_gemm<64>(l, st0, w0, ns, s, bar_full, bar_empty, wg, lane, pg);
          stamp(1);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = rows[h], grow = g * kTcRows + row;
            const bool live = grow < A.B;
            unsigned long long best = 0ull;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int cls = 64 * R.ci + 8 * i + 2 * c;
              const float l0 = l[4 * i + 2 * h] + b3[8 * i + 2 * c], l1 = l[4 * i + 2 * h + 1] + b3[8 * i + 2 * c + 1];
              if (live && A.logits_out) *reinterpret_cast<float2*>(A.logits_out + ((size_t)t * A.B + grow) * A.NC + cls) = make_float2(l0, l1);
              const unsigned long long p0 = push_pack(l0 - nl[(4 * i + 2 * h) * 256], (uint32_t)cls, (uint32_t)(t + 1));
              const unsigned long long p1 = push_pack(l1 - nl[(4 * i + 2 * h + 1) * 256], (uint32_t)(cls + 1), (uint32_t)(t + 1));
              best = p0 > best ? p0 : best;
              best = p1 > best ? p1 : best;
            }
#pragma unroll
            for (int o = 1; o <= 2; o <<= 1) {
              const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
              best = other > best ? other : best;
            }
            if (c == 0) {
#pragma unroll
              for (int cp = 0; cp < kTcWinCopies; ++cp)
                A.winners[((((size_t)g * 2 + (t & 1)) * kTcWinCopies + cp) * kTcRows + row) * 16 + R.ci] = best;
            }
          }
          publish(g, TCN_W);
          stamp(2);
          if (tc_consumers_any(pg.aborted)) { pg.aborted = true; break; }
        }
        if (pg.aborted) break;
      }
    }
    if (A.prof && tid == 0 && R.role != TC_ROLE_G1)
      for (int i = 0; i < 3; ++i) A.prof[(size_t)blockIdx.x * 12 + 3 * (R.role - 1) + i] = pf[i];
  } else {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kTcOtherRegs));
    if (warp == kTcLoaderWarp) {
      // ================= loader: counter -> bulk copies into the stage ring =================
      if (lane == 0) {
        unsigned s = 0;
        for (int t = 0; t < A.steps && !pg.aborted; ++t)
          for (int g = 0; g < ng && !pg.aborted; ++g)
            for (int j = 0; j < R.njobs; ++j) {
              int v, cw, nprod;
              tc_job(R.role, j, v, cw, nprod);
              if (!tc_cnt_wait(counter(g, cw), (unsigned)nprod * (unsigned)(t + 1), pg)) break;
              asm volatile("fence.proxy.async;" ::: "memory");      // generic-proxy stores of the producers -> this thread's async-proxy reads
              const uint8_t* src = vec_img(v, g, t & 1);
              for (int ks = 0; ks < kTcStagesPerVec; ++ks, ++s) {
                const unsigned slot = s % (unsigned)R.nstage, use = s / (unsigned)R.nstage;
                if (!tc_mbar_wait(&bar_empty[slot], (use & 1u) ^ 1u, pg)) break;
                mbar_expect_tx(&bar_full[slot], kTcStageBytes);
                tma_bulk_g2s(stages + (size_t)slot * kTcStageBytes, src + (size_t)ks * kTcStageBytes, kTcStageBytes, &bar_full[slot]);
              }
              if (pg.aborted) break;
            }
      }
      __syncwarp();
    } else if (R.role == TC_ROLE_G1) {
      // ================= conditioning warps (GRU-1 CTAs): the 64 conditioned values of every row, a BLOCK of <= 8 steps at a time ========
      // Within a frame the <= 7 table rows an output combines do not change, only the FIR phase does: they are loaded once per block
      // and combined for every step of it (8x fewer table loads than step by step).  The results go to a small ring in global
      // memory (two block buffers per CTA, L2 resident) that the gate threads read back one step at a time.
      // lane = value: lanes 0-15 / 16-31 take the 16 table entries (kind*4 + unit%4) of two adjacent 4-unit table blocks.
      const int cwarp = warp - kTcCondWarp0;
      const int half = lane >> 4, i16 = lane & 15;
      const size_t fstride = (size_t)128 * kPushCondRows;
      float* cring = A.condg + (size_t)R.ci * 2 * ng * kTcCondBlk * kTcCondSlot;
      int b = 0;
      for (int t0 = 0; t0 < A.steps && !pg.aborted; ++b) {
        const int fr = t0 / A.hop, ph0 = t0 - fr * A.hop;
        const int t1 = min(min(t0 + kTcCondBlk, (fr + 1) * A.hop), A.steps), n = t1 - t0;
        if (!tc_mbar_wait(&bar_condempty[b & 1], ((unsigned)(b >> 1) & 1u) ^ 1u, pg)) break;
        for (int g = 0; g < ng; ++g) {
          float* dst = cring + (size_t)((b & 1) * ng + g) * kTcCondBlk * kTcCondSlot;
#pragma unroll 2
          for (int row = cwarp; row < kTcRows; row += kTcCondWarps) {   // 2 rows x 2 blocks x 7 table loads in flight per lane
            const int src = min(g * kTcRows + row, A.B - 1);
#pragma unroll
            for (int p = 0; p < 2; ++p) {
              const int c4l = 2 * p + half;                                        // 4-unit block inside this CTA's 16 units
              const float* base = A.tab + (((size_t)src * (A.T + 1) + fr) * 128 + 4 * R.ci + c4l) * kPushCondRows;
              const float v0 = __ldg(base + 16 + i16);
              float pm[kMaxTaps];
#pragma unroll
              for (int j = 0; j < kMaxTaps; ++j) {
                const int f = fr + j - A.NT / 2;
                pm[j] = (j < A.NT && f >= 0 && f < A.T) ? __ldg(base + (ptrdiff_t)(f - fr) * (ptrdiff_t)fstride + i16) : 0.f;
              }
              float* o = dst + (size_t)row * 64 + (i16 >> 2) * 16 + c4l * 4 + (i16 & 3);
              for (int sidx = 0; sidx < n; ++sidx) {
                const float* fc = fir_s + (ph0 + sidx) * A.NT;
                float v = v0;
#pragma unroll
                for (int j = 0; j < kMaxTaps; ++j)
                  if (j < A.NT) v = fmaf(fc[j], pm[j], v);      // an absent frame contributes fir * 0 = 0 exactly (same order as push_cond16)
                o[(size_t)sidx * kTcCondSlot] = v;
              }
            }
          }
        }
        __syncwarp();
        if (lane == 0) tc_mbar_arrive(&bar_condfull[b & 1]);
        t0 = t1;
      }
    }
  }
  __syncthreads();
}

// ---- host: the per-CTA B-operand images [kTcCtas][kTcWimgBytes] and parameters [kTcCtas][kTcPrm], cut from the push kernel's
//      blobs `pb` (pack_push_model).  Every weight is split into two fp16 planes (hi, lo' = (w - hi) * 2048) in the wgmma
//      K-major no-swizzle layout [plane][k-step 32][k half 2][N/8][8 cols][8 halves].  False, with nothing packed, when the
//      model or device cannot run this kernel: it needs the push kernel's model, 1024 classes, kTcCtas SMs and a FIR table of
//      `fir_floats` that fits its shared-memory slot. ---------------------------------------------------------------------------
inline bool pack_tc_images(const PushModel& pm, const std::vector<float>& pb, int sm_count, int fir_floats,
                           std::vector<uint16_t>& img, std::vector<float>& prm) {
  img.clear();
  prm.clear();
  if (!(pm.ok && pm.NC == 1024 && sm_count >= kTcCtas && (size_t)fir_floats * sizeof(float) <= (size_t)kTcFirMaxBytes))
    return false;
  const int R = pm.R, F = pm.F;
  img.assign((size_t)kTcCtas * kTcWimgBytes / 2, 0);
  prm.assign((size_t)kTcCtas * kTcPrm, 0.f);
  auto put = [&](uint16_t* base, int N, int col, const float* wrow) {     // one weight row (K = 512) -> column `col` of an image
    for (int k = 0; k < 512; ++k) {
      const float w = wrow[k];
      const __half hi = __float2half_rn(w);
      const __half lo = __float2half_rn((w - __half2float(hi)) * 2048.0f);
      const size_t off = ((size_t)(k >> 4) * 2 + ((k >> 3) & 1)) * ((size_t)N * 8) + (size_t)(col >> 3) * 64 + (size_t)(col & 7) * 8 + (k & 7);
      base[off] = __half_as_ushort(hi);
      base[(size_t)32 * N * 16 + off] = __half_as_ushort(lo);
    }
  };
  auto unit_blob = [&](int unit) { return &pb[(size_t)(unit >> 2) * pm.blob]; };
  for (int cta = 0; cta < kTcCtas; ++cta) {
    uint16_t* wi = &img[(size_t)cta * kTcWimgBytes / 2];
    float* pr = &prm[(size_t)cta * kTcPrm];
    if (cta < 32) {                                   // GRU-1: 16 units, columns gate*16 + i
      for (int i = 0; i < 16; ++i) {
        const int unit = 16 * cta + i, j = unit & 3;
        const float* b = unit_blob(unit);
        for (int gate = 0; gate < 3; ++gate) {
          put(wi, 48, gate * 16 + i, b + pm.ohh1 + (size_t)(gate * 4 + j) * R);
          pr[64 + gate * 16 + i] = b[pm.obhh1 + gate * 4 + j];
        }
        for (int kind = 0; kind < 4; ++kind) pr[kind * 16 + i] = b[pm.oAx + kind * 4 + j];
      }
    } else if (cta < 96) {                            // GRU-2: 8 units, W_ih2 image then W_hh2 image, columns gate*8 + i (24-31 zero)
      const int ci = cta - 32;
      for (int i = 0; i < 8; ++i) {
        const int unit = 8 * ci + i, j = unit & 3;
        const float* b = unit_blob(unit);
        for (int gate = 0; gate < 3; ++gate) {
          put(wi, 32, gate * 8 + i, b + pm.oih2 + (size_t)(gate * 4 + j) * R);
          put(wi + 32768, 32, gate * 8 + i, b + pm.ohh2 + (size_t)(gate * 4 + j) * R);
          pr[gate * 8 + i] = b[pm.obhh2 + gate * 4 + j];
        }
      }
    } else if (cta < 112) {                           // fc1 / fc2: 64 units
      const bool first = cta < 104;
      const int ci = first ? cta - 96 : cta - 104;
      for (int i = 0; i < 64; ++i) {
        const int unit = 64 * ci + i, j = unit & 3;
        const float* b = unit_blob(unit);
        put(wi, 64, i, b + (first ? pm.ofc1 : pm.ofc2) + (size_t)j * R);
      }
    } else {                                          // fc3: 64 classes
      const int ci = cta - 112;
      for (int i = 0; i < 64; ++i) {
        const int cls = 64 * ci + i;
        const float* b = &pb[(size_t)(cls >> 3) * pm.blob];
        put(wi, 64, i, b + pm.ofc3 + (size_t)(cls & 7) * F);
        pr[i] = b[pm.obfc3 + (cls & 7)];
      }
    }
  }
  return true;
}

}  // namespace b200tts
