// The body of wavernn_grid_kernel<U, UW, GROUPS> and wavernn_grid_mol_kernel<U, UW, GROUPS> (wavernn_grid.cuh): included inside
// both kernels, with `MOL` (constexpr bool) and
// `io` (MolIO) declared by the includer.  Each kernel is thus compiled from its own copy of the text, so the RAW kernel's code
// is exactly what it was before MOL existed; `if constexpr (MOL)` selects the sampler.  Not a standalone header.
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
  [[maybe_unused]] const float ncls_m1 = (float)(M.NC - 1);
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
          if constexpr (MOL) {
            x = grid_mol_sample(A, io, u, t - 1, c == 0);
          } else {
          unsigned long long pk = __ldcg(A.best + (size_t)((t - 1) & 1) * Bp + u);
          int label = (int)unpack_idx(pk);
          if (c == 0) A.labels[(size_t)u * A.S + (t - 1)] = (int16_t)label;
          int fb = A.teacher ? (int)A.teacher[(size_t)u * A.S + (t - 1)] : label;
          x = label_to_float(fb, ncls_m1);
          }
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
      if constexpr (MOL) {
        if (c < kMolParams)
          for (int ul = tid; ul < BT; ul += NT) {
            const int u = tb + ul;
            if (u < A.B) {
              const float l = part_sum<KS1, kCPC, BT>(res, 0, 0, ul) + b[0];
              io.par[((size_t)(t & 1) * Bp + u) * 32 + c] = l;
              if (A.logits_out) A.logits_out[((size_t)t * A.B + u) * kMolParams + c] = l;
            }
          }
      } else
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
      if constexpr (MOL) {
        grid_mol_sample(A, io, u, t - 1, true);
      } else {
      unsigned long long pk = __ldcg(A.best + (size_t)((t - 1) & 1) * Bp + u);
      A.labels[(size_t)u * A.S + (t - 1)] = (int16_t)unpack_idx(pk);
      }
    }
  }
