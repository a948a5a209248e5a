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

// GENERATION SESSIONS on the tensor cores (b200tts_wavernn_session_* with kernel = TC, wavernn_tc_session_kernel): row u of a
// launch resumes session u (SessRow, wavernn_push.cuh) at its position pos and runs n steps, lock-steps 0 ... n-1 being steps
// pos + t of its utterance; then it idles to the end of the run (no labels stored, its table reads clamped to its frame T).
// Every position is a multiple of hop (the run's step count is), so lock-step t has the same FIR phase in every row, the GRU-1
// conditioning blocks keep their shape, and the frame of row u is pos / hop + t / hop.  At the last lock-step a row that ran the
// whole run saves what makes its next step the one-shot step: h1 and h2 from the gate threads, W_hh1.h1 and W_hh2.h2 as the
// accumulators the run's last GEMMs left (they run one step ahead, so no extra GEMM) and the last label (the next x).  The
// state thus differs from a push session's (same size), and a session stays on the kernel it was opened for.
constexpr int kTcSessRows = kTcRows * kTcMaxGroups;
constexpr int kTcSessH1 = 0, kTcSessH2 = 512, kTcSessGh1 = 1024, kTcSessGh2 = kTcSessGh1 + 3 * 512, kTcSessLabel = kTcSessGh2 + 3 * 512;
static_assert(kTcSessLabel + 1 <= kSessStateFloats, "a tensor-core session's state fits a push session's");
struct TcSessIO {                   // passed by value (a 12 KB kernel parameter), next to TcArgs
  SessRow row[kTcSessRows];
  int16_t* labels;                  // [rows][ld]: the label of step pos + i of row u at labels[u * ld + i]
  int ld;
};
// table frame of lock-step t of session row r: clamped to its zero-conditioning frame T once the row has finished
__device__ __forceinline__ int tc_sess_frame(const SessRow& r, int t, int hop) { return min(r.pos / hop + t / hop, r.T); }
// state index of GRU-1 accumulator fragment f of thread column c in CTA ci: column 8 (f / 4) + 2c + f % 2 = gate * 16 + unit
__device__ __forceinline__ int tc_sess_gh1(int f, int c, int ci) {
  const int col = 8 * (f >> 2) + 2 * c + (f & 1);
  return kTcSessGh1 + (col >> 4) * 512 + 16 * ci + (col & 15);
}

__global__ void __launch_bounds__(kTcThreads, 1) wavernn_tc_kernel(TcArgs A) {
  constexpr bool SESS = false;
  [[maybe_unused]] const TcSessIO sio{};
#include "wavernn_tc_step.cuh"
}

// RAW generation sessions: row u resumes session u of `sio`; A carries the shared buffers, B = sessions and steps = lock-steps.
__global__ void __launch_bounds__(kTcThreads, 1) wavernn_tc_session_kernel(TcArgs A, TcSessIO sio) {
  constexpr bool SESS = true;
#include "wavernn_tc_step.cuh"
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
