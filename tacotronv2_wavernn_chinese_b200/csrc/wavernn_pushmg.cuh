// WaveRNN per-sample recurrence, MULTI-GROUP push kernel: the large-batch (33 ... 256 rows per GPU) form of wavernn_push.cuh.
//
// Same per-group data flow as wavernn_push_kernel<32> (flag-in-data exchange through L2, hoisted conditioning, recurrent
// projections one step ahead, Gumbel-max winners as tagged 64-bit words), but the batch is cut into `ng` <= 8 independent
// groups of 32 rows and every phase of a step is run for all groups in turn:
//
//     for g: P01(g)     for g: P2(g) + W_hh1      for g: P3(g) + W_hh2      for g: P4(g) + rearm + cond      for g: P5(g)
//
// so between a group's publish (say x1 in P01(g)) and its consumption (P2(g)) the block is busy with the other groups:
// with >= 2 groups the polls find their data already there and the exchange LATENCY that dominates a single group
// (tools/exchange_bench.cu: ~4 000 cycles per exchange at 32 rows) disappears behind compute; what remains is FMA issue and
// the L2 -> SM broadcast bandwidth of the activations.  Compared with the round-1 wide mapping (wavernn_grid.cuh) every
// activation word is loaded ONCE per block straight into the register of the thread that multiplies it (there: once per
// row-slice warp through L1), there are no grid barriers and no k-slice partial sums of the conditioning columns.
//
// STATUS: parity-green against the oracle on the shipped checkpoint at 64 / 100 / 128 / 256 rows, but NOT the default: on the
// previous GPU it was slower than the wide mapping of wavernn_grid.cuh at 64 / 128 / 256 rows (twice as slow at 256; not
// re-measured on the H100).  A group's L2 loads, FMAs, cross-warp reduction and gate math are serialised by its block
// barriers (a fixed cost per group and step, flat in the number of groups): latency is hidden, issue slots are not filled.  It runs
// only with B200TTS_PUSH_MAX_ROWS=256 in the environment; its one advantage is the batch-size-invariant arithmetic.
//
// Shared memory (ng = 8): weights 104 KB, two partial-sum buffers 48 KB, per group gh1/gh2 3 KB + conditioning rows 16-35
// 2.5 KB + the gate threads' own h1/h2/x1 1.5 KB, small double-buffered scratch: 222 KB.
#pragma once
#include "wavernn_push.cuh"

namespace b200tts {

constexpr int kMgG = 32;          // rows per group
constexpr int kMgMaxGroups = 8;

struct MgLayout {                 // floats after the weight blob
  int oPartX, oPartY, oC0, oCond, oGh1, oGh2, oOwn, oSmax, oKeys, total;
  __host__ __device__ explicit MgLayout(int ng) {
    constexpr int G = kMgG;
    int o = 0;
    oPartX = o; o += kPushWarps * 12 * G;
    oPartY = o; o += kPushWarps * 12 * G;
    oC0 = o; o += 2 * 16 * G;                 // P01 conditioning rows 0-15, double-buffered by group parity
    oCond = o; o += ng * 20 * G;              // rows 16-35 (aux projections + bias): GRU-2 12, fc1 4, fc2 4
    oGh1 = o; o += ng * 12 * G;
    oGh2 = o; o += ng * 12 * G;
    oOwn = o; o += ng * 3 * 4 * G;            // gate threads: h1, h2, x1 of (row, unit)
    oSmax = o; o += 2 * 2 * kPushWarps * G;   // u64 [2][16][G]
    oKeys = o; o += 2 * 8 * G;                // u64 [8][G]
    total = o;
  }
};

// conditioning rows 16-35 of step t for group g -> dst[20][G]   (aux projections + bias; constant within a frame)
__device__ __forceinline__ void mg_cond20(const PushArgs& A, float* dst, int c, int ncta, int g, int t, int tid) {
  constexpr int G = kMgG;
  const int fr0 = t / A.hop;
  for (int it = tid; it < 20 * G; it += kPushThreads) {
    const int u = it / 20, r = it - u * 20, row = g * G + u;
    int src = row, fr = fr0;
    if (A.row_stride) {
      const long long n = (long long)row * A.row_stride + t;
      src = 0;
      fr = n >= A.S_src ? A.T : (int)(n / A.hop);
    }
    dst[r * G + u] = __ldg(A.tab + (((size_t)src * (A.T + 1) + fr) * ncta + c) * kPushCondRows + 32 + r);
  }
}

__global__ void __launch_bounds__(kPushThreads, 1) wavernn_pushmg_kernel(PushModel M, PushArgs A) {
  constexpr int G = kMgG;
  using PT = PushTraits<G>;
  constexpr int NU = PT::NU;
  extern __shared__ __align__(16) float smem[];
  const int ng = A.ng;
  const MgLayout L(ng);
  float* Wb = smem;
  float* sc = smem + M.blob;
  float* partX = sc + L.oPartX;
  float* partY = sc + L.oPartY;
  float* c0 = sc + L.oC0;
  float* cond = sc + L.oCond;
  float* gh1 = sc + L.oGh1;
  float* gh2 = sc + L.oGh2;
  float* own = sc + L.oOwn;
  unsigned long long* smax = reinterpret_cast<unsigned long long*>(sc + L.oSmax);
  unsigned long long* skeys = reinterpret_cast<unsigned long long*>(sc + L.oKeys);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int c = blockIdx.x, ncta = gridDim.x;
  const int ul = tid % NU, kq = tid / NU;                 // GEMM mapping
  const int gu = tid % G, gj = tid / G;                   // gate mapping: row gu, unit gj (threads < 4G)
  const bool gate = tid < 4 * G;
  const float ncls_m1 = (float)(M.NC - 1);
  const size_t vstride = (size_t)ncta * G * 4;            // floats per parity copy of one vector of one group
  auto vecp = [&](int g, int which, int parity) { return A.vec + (((size_t)g * kPushVecs + which) * 2 + parity) * vstride; };

  {   // one-time load of this CTA's weight blob: TMA bulk copies signalled through an mbarrier
    __shared__ __align__(8) unsigned long long wbar;
    const char* src = reinterpret_cast<const char*>(A.wblob + (size_t)c * M.blob);
    const unsigned total = (unsigned)M.blob * 4u;
    if (tid == 0) mbar_init(&wbar, 1);
    __syncthreads();
    if (tid == 0) {
      mbar_expect_tx(&wbar, total);
      for (unsigned off = 0; off < total; off += 32768u)
        tma_bulk_g2s(reinterpret_cast<char*>(Wb) + off, src + off, min(32768u, total - off), &wbar);
    }
    mbar_wait(&wbar, 0);
  }
  for (int i = tid; i < ng * 12 * G; i += kPushThreads) { gh1[i] = 0.f; gh2[i] = 0.f; }   // W_hh . 0  (h1 = h2 = 0, :194-195)
  for (int i = tid; i < ng * 3 * 4 * G; i += kPushThreads) own[i] = 0.f;
  __syncthreads();
  for (int g = 0; g < ng; ++g) mg_cond20(A, cond + g * 20 * G, c, ncta, g, 0, tid);
  __syncthreads();

  PollGuard pg{A.error, 0, 0, false};
  __shared__ long long s_pf[12];
  __shared__ long long s_tmark;
  if (tid == 0) {
    for (int i = 0; i < 12; ++i) s_pf[i] = 0;
    s_tmark = clock64();
  }
#define MG_MARK(slot)                            \
  do {                                           \
    if (A.prof && tid == 0) {                    \
      const long long now_ = clock64();          \
      s_pf[slot] += now_ - s_tmark;              \
      s_tmark = now_;                            \
    }                                            \
  } while (0)

  constexpr int NCQ = kPushThreads / G, NREC = 128 / NCQ;   // 16 producer queues, 8 winner records per thread
  const int cq = tid / G;
  const size_t fstride = (size_t)ncta * kPushCondRows;
  for (int t = 0; t <= A.steps; ++t) {
    const int par = t & 1;
    const bool last = (t == A.steps);                       // the extra trip only collects the last winners
    // ================= P01: winners of step t-1 -> label -> GRU 1 =================
    for (int g = 0; g < ng; ++g) {
      const int bp = g & 1;
      // conditioning rows 0-15 of (g, t): one (row, cond row) item per thread; the table loads fly during the winner poll
      float cpa = 0.f, cpm[kMaxTaps];
      int cph = 0;
      {
        const int u = tid >> 4, r = tid & 15, row = g * G + u;
        int src = row, fr = t / A.hop;
        cph = t - fr * A.hop;
        bool beyond = false;
        if (A.row_stride) {
          const long long n = (long long)row * A.row_stride + t;
          src = 0;
          beyond = n >= A.S_src;
          fr = beyond ? A.T : (int)(n / A.hop);
          cph = beyond ? 0 : (int)(n - (long long)fr * A.hop);
        }
        if (!last) {
          const float* rowp = A.tab + (((size_t)src * (A.T + 1) + fr) * ncta + c) * kPushCondRows;
          cpa = __ldg(rowp + 16 + r);
#pragma unroll
          for (int j = 0; j < kMaxTaps; ++j) {
            const int f = fr + j - A.NT / 2;
            cpm[j] = (!beyond && j < A.NT && f >= 0 && f < A.T) ? __ldg(rowp + ((ptrdiff_t)(f - fr)) * (ptrdiff_t)fstride + r) : 0.f;
          }
        } else {
#pragma unroll
          for (int j = 0; j < kMaxTaps; ++j) cpm[j] = 0.f;
        }
      }
      if (t > 0) {
        const unsigned long long* bestg = A.best + (size_t)g * ncta * G;
        const unsigned long long want = (unsigned long long)((uint32_t)t & 0x3FFFFFu);
        unsigned long long rec[NREC];
#pragma unroll
        for (int i = 0; i < NREC; ++i) rec[i] = ld_relaxed_u64(bestg + (size_t)(cq + NCQ * i) * G + gu);
        unsigned long long bestp = 0ull;
#pragma unroll
        for (int i = 0; i < NREC; ++i) {
          unsigned long long v = rec[i];
          if ((v & 0x3FFFFFull) != want) {
            const unsigned long long* p = bestg + (size_t)(cq + NCQ * i) * G + gu;
            pg.begin();
            while (true) {
              v = ld_relaxed_u64(p);
              if ((v & 0x3FFFFFull) == want || pg.expired()) break;
            }
          }
          bestp = v > bestp ? v : bestp;
        }
        smax[(bp * kPushWarps + warp) * G + lane] = bestp;     // G == 32: lane == row, warp == producer queue
      }
      if (!last) {
        float v = cpa;
#pragma unroll
        for (int j = 0; j < kMaxTaps; ++j)
          if (j < A.NT) v = fmaf(__ldg(A.fir + cph * A.NT + j), cpm[j], v);
        c0[bp * 16 * G + (tid & 15) * G + (tid >> 4)] = v;
      }
      if (__syncthreads_or(pg.aborted ? 1 : 0)) return;
      if (gate) {
        float x = 0.f;
        const int row = g * G + gu;
        if (t > 0) {
          unsigned long long b = 0ull;
#pragma unroll
          for (int w = 0; w < kPushWarps; ++w) { const unsigned long long v = smax[(bp * kPushWarps + w) * G + gu]; b = v > b ? v : b; }
          const int label = (int)push_cls(b);
          if (row < A.B) {
            if (c == 0 && gj == 0) A.labels[(size_t)row * A.S + (t - 1)] = (int16_t)label;
            const int fb = A.teacher ? (int)A.teacher[(size_t)row * A.S + (t - 1)] : label;
            x = label_to_float(fb, ncls_m1);
          }
        }
        if (!last) {
          const float* cd = c0 + bp * 16 * G;
          const float* g1 = gh1 + g * 12 * G;
          float* ow = own + g * 3 * 4 * G;
          const float* wAx = Wb + M.oAx;
          const float* bhh = Wb + M.obhh1;
          const float iout = fmaf(wAx[gj], x, cd[gj * G + gu]);
          const float gir = fmaf(wAx[4 + gj], x, cd[(4 + gj) * G + gu]);
          const float giz = fmaf(wAx[8 + gj], x, cd[(8 + gj) * G + gu]);
          const float gin = fmaf(wAx[12 + gj], x, cd[(12 + gj) * G + gu]);
          const float h = gru_update(gir, giz, gin, g1[gj * G + gu] + bhh[gj], g1[(4 + gj) * G + gu] + bhh[4 + gj],
                                     g1[(8 + gj) * G + gu] + bhh[8 + gj], ow[tid]);
          ow[tid] = h;
          ow[2 * 4 * G + tid] = iout + h;
          const size_t e = ((size_t)c * G + gu) * 4 + gj;
          st_relaxed_f32(vecp(g, PV_H1, par) + e, h);
          st_relaxed_f32(vecp(g, PV_X1, par) + e, iout + h);
        }
      }
    }
    if (last) break;
    MG_MARK(0);

    // ================= P2: GRU 2 input projection on x1(t);  then W_hh1 . h1(t) for step t+1 =================
    for (int g = 0; g < ng; ++g) {
      push_gemm<G, 12>(Wb + M.oih2, vecp(g, PV_X1, par), partX, ul, kq, warp, lane, pg);
      if (__syncthreads_or(pg.aborted ? 1 : 0)) return;
      if (gate) {
        const float* cd = cond + g * 20 * G;
        const float* g2 = gh2 + g * 12 * G;
        float* ow = own + g * 3 * 4 * G;
        const float* bhh = Wb + M.obhh2;
        const float h = gru_update(push_part_sum<G, 12>(partX, gj, gu) + cd[gj * G + gu],
                                   push_part_sum<G, 12>(partX, 4 + gj, gu) + cd[(4 + gj) * G + gu],
                                   push_part_sum<G, 12>(partX, 8 + gj, gu) + cd[(8 + gj) * G + gu], g2[gj * G + gu] + bhh[gj],
                                   g2[(4 + gj) * G + gu] + bhh[4 + gj], g2[(8 + gj) * G + gu] + bhh[8 + gj], ow[4 * G + tid]);
        ow[4 * G + tid] = h;
        const size_t e = ((size_t)c * G + gu) * 4 + gj;
        st_relaxed_f32(vecp(g, PV_H2, par) + e, h);
        st_relaxed_f32(vecp(g, PV_X2, par) + e, ow[2 * 4 * G + tid] + h);
      }
      push_gemm<G, 12>(Wb + M.ohh1, vecp(g, PV_H1, par), partY, ul, kq, warp, lane, pg);
      if (__syncthreads_or(pg.aborted ? 1 : 0)) return;
      for (int i = tid; i < 12 * G; i += kPushThreads) gh1[g * 12 * G + i] = push_part_sum<G, 12>(partY, i / G, i % G);
    }
    MG_MARK(1);

    // ================= P3: fc1 + relu on x2(t);  then W_hh2 . h2(t) for step t+1 =================
    for (int g = 0; g < ng; ++g) {
      push_gemm<G, 4>(Wb + M.ofc1, vecp(g, PV_X2, par), partX, ul, kq, warp, lane, pg);
      if (__syncthreads_or(pg.aborted ? 1 : 0)) return;
      if (gate) {
        const float v = push_part_sum<G, 4>(partX, gj, gu) + cond[g * 20 * G + (12 + gj) * G + gu];
        st_relaxed_f32(vecp(g, PV_F1, par) + ((size_t)c * G + gu) * 4 + gj, fmaxf(v, 0.f));
      }
      push_gemm<G, 12>(Wb + M.ohh2, vecp(g, PV_H2, par), partY, ul, kq, warp, lane, pg);
      if (__syncthreads_or(pg.aborted ? 1 : 0)) return;
      for (int i = tid; i < 12 * G; i += kPushThreads) gh2[g * 12 * G + i] = push_part_sum<G, 12>(partY, i / G, i % G);
    }
    MG_MARK(2);

    // ================= P4: fc2 + relu on f1(t);  rearm;  conditioning rows 16-35 of step t+1 =================
    for (int g = 0; g < ng; ++g) {
      float* pbuf = (g & 1) ? partY : partX;                 // no barrier between a group's gate reads and the next group's partials
      push_gemm<G, 4>(Wb + M.ofc2, vecp(g, PV_F1, par), pbuf, ul, kq, warp, lane, pg);
      // the fc2 conditioning value is taken BEFORE the barrier: after it the other threads overwrite cond[g] for step t+1
      const float cv = gate ? cond[g * 20 * G + (16 + gj) * G + gu] : 0.f;
      if (__syncthreads_or(pg.aborted ? 1 : 0)) return;
      if (gate) {
        const float v = push_part_sum<G, 4>(pbuf, gj, gu) + cv;
        const size_t e = ((size_t)c * G + gu) * 4 + gj;
        st_relaxed_f32(vecp(g, PV_F2, par) + e, fmaxf(v, 0.f));
        // REARM the other parity copy of this group's vectors (proof as in wavernn_push.cuh: every CTA's winner of (g, t-1)
        // was seen in P01(g, t), and a CTA publishes a group's winner after its last read of that group's step vectors;
        // the sentinels are fenced before this CTA's winner of (g, t) is stored in the P5 loop below)
#pragma unroll
        for (int v6 = 0; v6 < kPushVecs; ++v6) st_relaxed_u32(vecp(g, v6, par ^ 1) + e, kPushSentinel);
        asm volatile("fence.acq_rel.gpu;" ::: "memory");
      }
      if (t + 1 < A.steps) mg_cond20(A, cond + g * 20 * G, c, ncta, g, t + 1, tid);
    }
    __syncthreads();                                         // P4 gate reads of partY (odd groups) vs the P5 partials
    MG_MARK(3);

    // ================= P5: fc3 on f2(t) + Gumbel-max over this CTA's 8 classes =================
    for (int g = 0; g < ng; ++g) {
      push_gemm<G, 8>(Wb + M.ofc3, vecp(g, PV_F2, par), partY, ul, kq, warp, lane, pg);
      if (__syncthreads_or(pg.aborted ? 1 : 0)) return;
      if (tid < 8 * G) {
        const int r = tid / G, u = tid % G, row = g * G + u;
        const int cls = c * kCPC + r;
        const float l = push_part_sum<G, 8>(partY, r, u) + Wb[M.obfc3 + r];
        float qv = 1.0f;
        if (row < A.B) {
          if (A.rng_mode == 0) {
            float q4[4];
            philox_exp4(A.seed, A.utt_ids ? A.utt_ids[row] : A.utt_offset + (unsigned long long)row, (uint32_t)t, (uint32_t)(cls >> 2), q4);
            qv = q4[cls & 3];
          } else {
            qv = __ldg(A.q + ((size_t)t * A.B + row) * M.NC + cls);
          }
          if (A.logits_out) A.logits_out[((size_t)t * A.B + row) * M.NC + cls] = l;
        }
        skeys[r * G + u] = push_pack(l - logf(qv), (uint32_t)cls, (uint32_t)(t + 1));
      }
      __syncthreads();
      if (tid < G) {
        unsigned long long b = skeys[tid];
#pragma unroll
        for (int r = 1; r < 8; ++r) { const unsigned long long v = skeys[r * G + tid]; b = v > b ? v : b; }
        st_relaxed_u64(A.best + ((size_t)g * ncta + c) * G + tid, b);
      }
    }
    MG_MARK(4);
  }
  if (A.prof && tid == 0)
    for (int i = 0; i < 12; ++i) A.prof[(size_t)c * 12 + i] = s_pf[i];
#undef MG_MARK
}

}  // namespace b200tts
