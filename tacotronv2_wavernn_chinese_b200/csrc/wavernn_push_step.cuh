// The body of wavernn_push_kernel<G>, wavernn_push_mol_kernel<G> and wavernn_push_session_kernel<G> (wavernn_push.cuh): included
// inside each kernel, with `MOL`, `SESS` (constexpr bool), `io` (MolIO) and `sio` (SessIO) declared by the includer.  Each kernel
// is thus compiled from its own copy of the text, so the RAW kernel's code is exactly what it was before MOL and sessions
// existed; `if constexpr (MOL)` selects the sampler, `SESS` the per-session rows, state and addressing.  Not a standalone header.
  using PT = PushTraits<G>;
  constexpr int NU = PT::NU;
  extern __shared__ __align__(16) float smem[];
  float* Wb = smem;
  float* sc = smem + M.blob;
  float* partX = sc + PT::oPartX;
  float* partY = sc + PT::oPartY;
  float* cond = sc + PT::oCond;
  float* gh1 = sc + PT::oGh1;
  float* gh2 = sc + PT::oGh2;
  unsigned long long* smax = reinterpret_cast<unsigned long long*>(sc + PT::oSmax);
  unsigned long long* skeys = reinterpret_cast<unsigned long long*>(sc + PT::oKeys);
  float* xs = sc + PT::oXs;
  float* fir_s = sc + PT::oFir;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int c = blockIdx.x, ncta = gridDim.x;
  const int ul = tid % NU, kq = tid / NU;                 // GEMM mapping
  const int gu = tid % G, gj = tid / G;                   // gate mapping: row gu, unit gj (threads < 4G)
  const bool gate = tid < 4 * G;
  [[maybe_unused]] const float ncls_m1 = (float)(M.NC - 1);
  const size_t vstride = (size_t)ncta * G * 4;            // floats per parity copy of one vector
  auto vecp = [&](int which, int parity) { return A.vec + ((size_t)which * 2 + parity) * vstride; };

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
  for (int i = tid; i < A.hop * A.NT; i += kPushThreads) fir_s[i] = A.fir[i];
  for (int i = tid; i < 12 * G; i += kPushThreads) { gh1[i] = 0.f; gh2[i] = 0.f; }     // W_hh . 0  (h1 = h2 = 0, :194-195)
  __shared__ PushRowState R;
  if (tid < G) {
    // state "before step 0": an empty segment ending at step 0, so that push_row_next(..., t = 0) finds segment 0
    R.k[tid] = -1; R.utt[tid] = -1; R.t0[tid] = 0; R.end[tid] = 0; R.putt[tid] = -1; R.pn[tid] = 0; R.rst[tid] = 1;
    if (!A.pack_utt) {                                     // plain batch / folds: row u is utterance u from step 0 to the end
      R.k[tid] = 0; R.utt[tid] = tid < A.B ? tid : -1; R.end[tid] = 0x7fffffff;
    }
    if constexpr (SESS) {                                  // row u: session u from step pos (t0 = -pos) for n lock-steps
      const bool live = tid < A.B && sio.row[tid].n > 0;
      R.utt[tid] = live ? tid : -1;
      R.t0[tid] = live ? -sio.row[tid].pos : 0;
      R.end[tid] = live ? sio.row[tid].n : 0x7fffffff;
      R.rst[tid] = (!live || sio.row[tid].pos == 0) ? 1 : 0;  // position 0 starts from the zero state, as a one-shot run
    }
  }
  __syncthreads();
  if constexpr (SESS) {                                    // a resumed row: the projections its previous run saved
    for (int i = tid; i < 12 * G; i += kPushThreads) {
      const int u = i % G;
      if (R.utt[u] >= 0 && !R.rst[u]) {
        gh1[i] = sio.row[u].state[kSessGh1 + c * 12 + i / G];
        gh2[i] = sio.row[u].state[kSessGh2 + c * 12 + i / G];
      }
    }
  }
  float* cond16 = cond;                       // [2][16][G]  rows 0-15 of step t (parity buffers, written one step ahead)
  float* cond20 = cond + 2 * 16 * G;          // [20][G]     rows 16-35 of the current frame
  push_cond16<G, SESS>(A, R, sio, fir_s, cond16, c, ncta, 0, tid);
  push_cond20<G, SESS>(A, R, sio, cond20, c, ncta, 0, tid);
  __syncthreads();
  if (A.pack_utt && tid < G) {                             // enter segment 0 (kernel rows beyond the schedule stay idle)
    const bool live = tid < A.pack_rows && A.pack_segs > 0;
    R.k[tid] = 0;
    R.utt[tid] = live ? A.pack_utt[tid * A.pack_segs] : -1;
    R.t0[tid] = 0;
    R.end[tid] = live ? A.pack_start[tid * (A.pack_segs + 1) + 1] : 0x7fffffff;
  }
  __syncthreads();

  PollGuard pg{A.error, 0, 0, false};
  float h1own = 0.f, h2own = 0.f;                          // gate threads: state of unit 4c+gj, row gu
  [[maybe_unused]] float x_resume = 0.f;                   // SESS: x of a resumed row's first step (its last label)
  if constexpr (SESS) {
    if (gate && R.utt[gu] >= 0 && !R.rst[gu]) {
      const float* st = sio.row[gu].state;
      h1own = st[kSessH1 + 4 * c + gj];
      h2own = st[kSessH2 + 4 * c + gj];
      x_resume = label_to_float(reinterpret_cast<const int*>(st)[kSessLabel], ncls_m1);
    }
  }
  __shared__ long long s_pf[12];                           // optional per-phase cycle counters of thread 0 (debug)
  __shared__ long long s_tmark;
  if (tid == 0) {
    for (int i = 0; i < 12; ++i) s_pf[i] = 0;
    s_tmark = clock64();
  }
#define PUSH_MARK(slot)                          \
  do {                                           \
    if (A.prof && tid == 0) {                    \
      const long long now_ = clock64();          \
      s_pf[slot] += now_ - s_tmark;              \
      s_tmark = now_;                            \
    }                                            \
  } while (0)

  constexpr int NCQ = kPushThreads / G, NREC = 128 / NCQ;   // winner records per thread = G/4
  const int cq = tid / G;
  for (int t = 0; t <= A.steps; ++t) {
    const int par = t & 1;
    // ================= P01: winners of step t-1 -> label -> GRU 1 =================
    float x = 0.f;
    if constexpr (SESS) {
      if (t == 0) x = x_resume;
    }
    if (t > 0) {
      const unsigned long long want = (unsigned long long)((uint32_t)t & 0x3FFFFFu);
      unsigned long long rec[NREC];
#pragma unroll
      for (int i = 0; i < NREC; ++i) rec[i] = ld_relaxed_u64(A.best + (size_t)(cq + NCQ * i) * G + gu);
      [[maybe_unused]] unsigned long long bestp = 0ull;
#pragma unroll
      for (int i = 0; i < NREC; ++i) {
        unsigned long long v = rec[i];
        if ((v & 0x3FFFFFull) != want) {
          const unsigned long long* p = A.best + (size_t)(cq + NCQ * i) * G + gu;
          pg.begin();
          while (true) {
            v = ld_relaxed_u64(p);
            if ((v & 0x3FFFFFull) == want || pg.expired()) break;
          }
        }
        if constexpr (MOL) {
          const int prod = cq + NCQ * i;
          if (prod < kMolParams) reinterpret_cast<float*>(smax)[prod * G + gu] = __uint_as_float((uint32_t)(v >> 32));
        } else {
          bestp = v > bestp ? v : bestp;
        }
      }
      PUSH_MARK(0);
      if constexpr (MOL) {
        if (__syncthreads_or(pg.aborted ? 1 : 0)) return;
        const int putt = gate ? R.putt[gu] : -1, pn = gate ? R.pn[gu] : 0;
        if (putt >= 0) {                                    // sample_from_discretized_mix_logistic of step t-1
          float pm[kMolParams], uu[kMolU];
#pragma unroll
          for (int j = 0; j < kMolParams; ++j) pm[j] = reinterpret_cast<const float*>(smax)[j * G + gu];
          if (A.rng_mode == 0) {
            philox_mol_u(A.seed, A.utt_ids ? A.utt_ids[putt] : A.utt_offset + (unsigned long long)putt, (uint32_t)pn, uu);
          } else {
#pragma unroll
            for (int j = 0; j < kMolU; ++j) uu[j] = __ldg(A.q + ((size_t)pn * A.B + putt) * kMolU + j);
          }
          const float xs = mol_sample(pm, uu);
          if (c == 0 && gj == 0) io.samples[(size_t)putt * A.S + pn] = xs;
          x = io.teacher_x ? io.teacher_x[(size_t)putt * A.S + pn] : xs;
        }
      } else {
#pragma unroll
      for (int o = G; o < 32; o <<= 1) {
        const unsigned long long other = __shfl_xor_sync(0xffffffffu, bestp, o);
        bestp = other > bestp ? other : bestp;
      }
      if (lane < G) smax[warp * G + lane] = bestp;
      if (__syncthreads_or(pg.aborted ? 1 : 0)) return;
      if (gate) {                                           // every warp covered different producers: reduce the 16 warps
        unsigned long long b = 0ull;
#pragma unroll
        for (int w = 0; w < kPushWarps; ++w) { const unsigned long long v = smax[w * G + gu]; b = v > b ? v : b; }
        const int label = (int)push_cls(b);
        const int putt = R.putt[gu], pn = R.pn[gu];         // where this row was at step t-1
        if (putt >= 0) {
          if (c == 0 && gj == 0) {
            if constexpr (SESS) {
              sio.labels[(size_t)putt * sio.ld + (pn - sio.row[putt].pos)] = (int16_t)label;
              reinterpret_cast<int*>(sio.row[putt].state)[kSessLabel] = label;
            } else {
              A.labels[(size_t)putt * A.S + pn] = (int16_t)label;
            }
          }
          const int fb = A.teacher ? (int)A.teacher[(size_t)putt * A.S + pn] : label;
          x = label_to_float(fb, ncls_m1);
        }
      }
      }
    }
    if (t == A.steps) break;                                // the extra trip only collects the last winner
    const bool restart = gate && R.rst[gu] != 0;            // first step of an utterance: x = 0, h1 = h2 = 0 (:194-196)
    if (gate) {
      if (restart) { x = 0.f; h1own = 0.f; }
      const float* cd = cond16 + par * 16 * G;
      const float* wAx = Wb + M.oAx;
      const float* bhh = Wb + M.obhh1;
      const float iout = fmaf(wAx[gj], x, cd[gj * G + gu]);
      const float gir = fmaf(wAx[4 + gj], x, cd[(4 + gj) * G + gu]);
      const float giz = fmaf(wAx[8 + gj], x, cd[(8 + gj) * G + gu]);
      const float gin = fmaf(wAx[12 + gj], x, cd[(12 + gj) * G + gu]);
      const float g1r = restart ? 0.f : gh1[gj * G + gu], g1z = restart ? 0.f : gh1[(4 + gj) * G + gu],
                  g1n = restart ? 0.f : gh1[(8 + gj) * G + gu];            // W_hh1 . 0
      const float h = gru_update(gir, giz, gin, g1r + bhh[gj], g1z + bhh[4 + gj], g1n + bhh[8 + gj], h1own);
      h1own = h;
      const size_t e = ((size_t)c * G + gu) * 4 + gj;
      st_relaxed_f32(vecp(PV_H1, par) + e, h);
      st_relaxed_f32(vecp(PV_X1, par) + e, iout + h);
    }
    __syncwarp();      // (4G < 32: lanes that skip the gate block must not run ahead into a spin loop and steal its issue slots)
    PUSH_MARK(1);

    // ================= P2: W_ih2 (12 rows) AND fc1 (4 rows) on x1(t) =================
    // x2 = x1 + h2 is never exchanged: fc1 . x2 = fc1 . x1 + fc1 . h2, the first half is taken here while x1 is in registers,
    // the second in P3 from the h2 registers W_hh2 needs anyway -- one vector less through L2 per step.
    float f1x = 0.f;                                          // gate threads: (fc1 . x1)[4c + gj] of row gu
    // h1(t) was published together with x1(t): up to 16 rows (<= 4 float4 per vector and thread) its loads are issued with
    // the x1 loads, so the W_hh1 pass below starts from registers instead of paying another L2 round trip
    constexpr bool kPrefetchH1 = PT::NL <= 4;
    float4 ah1[kPrefetchH1 ? PT::NL : 1];
    {
      float4 a[PT::NL];
      push_load<G>(vecp(PV_X1, par), a, ul, kq, pg);
      if constexpr (kPrefetchH1) push_load<G>(vecp(PV_H1, par), ah1, ul, kq, pg);
      push_mma<G, 16>(Wb + M.oih2, a, partX, ul, kq, warp, lane);
    }
    PUSH_MARK(2);
    if (__syncthreads_or(pg.aborted ? 1 : 0)) return;
    if (gate) {
      const float* cd = cond20;
      const float* bhh = Wb + M.obhh2;
      if (restart) h2own = 0.f;
      const float g2r = restart ? 0.f : gh2[gj * G + gu], g2z = restart ? 0.f : gh2[(4 + gj) * G + gu],
                  g2n = restart ? 0.f : gh2[(8 + gj) * G + gu];            // W_hh2 . 0
      const float h = gru_update(push_part_sum<G, 16>(partX, gj, gu) + cd[gj * G + gu],
                                 push_part_sum<G, 16>(partX, 4 + gj, gu) + cd[(4 + gj) * G + gu],
                                 push_part_sum<G, 16>(partX, 8 + gj, gu) + cd[(8 + gj) * G + gu], g2r + bhh[gj], g2z + bhh[4 + gj],
                                 g2n + bhh[8 + gj], h2own);
      h2own = h;
      if constexpr (SESS) {
        if (R.utt[gu] >= 0 && t + 1 == R.end[gu]) {      // the row's last step of this run: save its state
          sio.row[gu].state[kSessH1 + 4 * c + gj] = h1own;
          sio.row[gu].state[kSessH2 + 4 * c + gj] = h2own;
        }
      }
      f1x = push_part_sum<G, 16>(partX, 12 + gj, gu);
      st_relaxed_f32(vecp(PV_H2, par) + ((size_t)c * G + gu) * 4 + gj, h);
    }
    __syncwarp();
    PUSH_MARK(3);
    // shadow: W_hh1 . h1(t) for step t+1
    if constexpr (kPrefetchH1) push_mma<G, 12>(Wb + M.ohh1, reinterpret_cast<const float4 (&)[PT::NL]>(ah1), partY, ul, kq, warp, lane);
    else push_gemm<G, 12>(Wb + M.ohh1, vecp(PV_H1, par), partY, ul, kq, warp, lane, pg);
    if (__syncthreads_or(pg.aborted ? 1 : 0)) return;
    for (int i = tid; i < 12 * G; i += kPushThreads) gh1[i] = push_part_sum<G, 12>(partY, i / G, i % G);
    PUSH_MARK(4);

    // ================= P3: h2(t) once: fc1 (critical), then W_hh2 . h2(t) for step t+1 from the same registers =================
    {
      float4 a[PT::NL];
      push_load<G>(vecp(PV_H2, par), a, ul, kq, pg);
      push_mma<G, 4>(Wb + M.ofc1, a, partX, ul, kq, warp, lane);
      PUSH_MARK(5);
      if (__syncthreads_or(pg.aborted ? 1 : 0)) return;
      if (gate) {
        const float v = (f1x + push_part_sum<G, 4>(partX, gj, gu)) + cond20[(12 + gj) * G + gu];
        st_relaxed_f32(vecp(PV_F1, par) + ((size_t)c * G + gu) * 4 + gj, fmaxf(v, 0.f));
      }
      __syncwarp();
      push_mma<G, 12>(Wb + M.ohh2, a, partY, ul, kq, warp, lane);
    }
    if (__syncthreads_or(pg.aborted ? 1 : 0)) return;
    for (int i = tid; i < 12 * G; i += kPushThreads) {
      gh2[i] = push_part_sum<G, 12>(partY, i / G, i % G);
      if constexpr (SESS) {                                   // this thread also wrote gh1[i] above (same mapping)
        const int u = i % G;
        if (R.utt[u] >= 0 && t + 1 == R.end[u]) {
          sio.row[u].state[kSessGh1 + c * 12 + i / G] = gh1[i];
          sio.row[u].state[kSessGh2 + c * 12 + i / G] = gh2[i];
        }
      }
    }
    PUSH_MARK(6);

    // ================= P4: fc2 + relu on f1(t) =================
    push_gemm<G, 4>(Wb + M.ofc2, vecp(PV_F1, par), partX, ul, kq, warp, lane, pg);
    // the fc2 conditioning value is taken BEFORE the barrier: after it the other threads may refresh cond20 for the next frame
    const float cv4 = gate ? cond20[(16 + gj) * G + gu] : 0.f;
    PUSH_MARK(7);
    if (__syncthreads_or(pg.aborted ? 1 : 0)) return;
    if (gate) {
      const float v = push_part_sum<G, 4>(partX, gj, gu) + cv4;
      const size_t e = ((size_t)c * G + gu) * 4 + gj;
      st_relaxed_f32(vecp(PV_F2, par) + e, fmaxf(v, 0.f));
      // REARM (shadow of the f2 exchange).  Every CTA's winner of step t-1 was seen at the top of this step, and a CTA
      // publishes its winner LAST in a step: all reads of the step t-1 vectors, which live in the other parity copy, are
      // over everywhere -- this thread's entries of that copy can take the sentinel again.  Nobody polls that copy for
      // step t+1 before it has seen THIS CTA's winner of step t, which is stored below after two block barriers that
      // follow this fence: the sentinels are performed gpu-wide by then.
#pragma unroll
      for (int v6 = 0; v6 < kPushVecs; ++v6)
        if (v6 != PV_X2) st_relaxed_u32(vecp(v6, par ^ 1) + e, kPushSentinel);      // (x2 is not exchanged by this kernel)
      asm volatile("fence.acq_rel.gpu;" ::: "memory");
    }
    __syncwarp();
    // shadow: conditioning of step t+1 (rows 0-15 into the other parity buffer; rows 16-35 only when a new frame starts)
    if (t + 1 < A.steps) {
      push_cond16<G, SESS>(A, R, sio, fir_s, cond16 + (par ^ 1) * 16 * G, c, ncta, t + 1, tid);
      if (SESS || A.row_stride || A.pack_utt || (t + 1) % A.hop == 0) push_cond20<G, SESS>(A, R, sio, cond20, c, ncta, t + 1, tid);
    }
    PUSH_MARK(8);

    // ================= P5: fc3 on f2(t) + Gumbel-max over this CTA's 8 classes =================
    push_gemm<G, 8>(Wb + M.ofc3, vecp(PV_F2, par), partY, ul, kq, warp, lane, pg);
    PUSH_MARK(9);
    if (__syncthreads_or(pg.aborted ? 1 : 0)) return;
    if constexpr (MOL) {
      if (tid < G) {                                           // parameter c of row u (none beyond the 30th CTA) + step tag
        const int u = tid;
        const float l = push_part_sum<G, 8>(partY, 0, u) + Wb[M.obfc3];
        const int utt = R.utt[u], n = t - R.t0[u];
        if (utt >= 0 && c < kMolParams && A.logits_out) A.logits_out[((size_t)n * A.B + utt) * kMolParams + c] = l;
        skeys[u] = (c < kMolParams ? (unsigned long long)__float_as_uint(l) << 32 : 0ull) | (unsigned long long)((uint32_t)(t + 1) & 0x3FFFFFu);
      }
    } else
    if (tid < 8 * G) {
      const int r = tid / G, u = tid % G;
      const int cls = c * kCPC + r;
      const float l = push_part_sum<G, 8>(partY, r, u) + Wb[M.obfc3 + r];
      float qv = 1.0f;
      const int utt = R.utt[u], n = t - R.t0[u];               // plain batch: utt == u, n == t
      if (utt >= 0) {
        if (SESS) {                                              // the session's key; n is the step within the utterance
          float q4[4];
          philox_exp4(sio.row[utt].seed, sio.row[utt].id, (uint32_t)n, (uint32_t)(cls >> 2), q4);
          qv = q4[cls & 3];
        } else if (A.rng_mode == 0) {
          float q4[4];
          philox_exp4(A.seed, A.utt_ids ? A.utt_ids[utt] : A.utt_offset + (unsigned long long)utt, (uint32_t)n, (uint32_t)(cls >> 2), q4);
          qv = q4[cls & 3];
        } else {
          qv = __ldg(A.q + ((size_t)n * A.B + utt) * M.NC + cls);
        }
        if (A.logits_out) A.logits_out[((size_t)n * A.B + utt) * M.NC + cls] = l;
      }
      skeys[r * G + u] = push_pack(l - logf(qv), (uint32_t)cls, (uint32_t)(t + 1));
    }
    __syncthreads();
    if (tid < G) {
      unsigned long long b = skeys[tid];
      if constexpr (!MOL) {
#pragma unroll
        for (int r = 1; r < 8; ++r) { const unsigned long long v = skeys[r * G + tid]; b = v > b ? v : b; }
      }
      st_relaxed_u64(A.best + (size_t)c * G + tid, b);
      // row bookkeeping for step t+1 (read by the gate threads after the barrier of the next winner poll)
      R.putt[tid] = R.utt[tid];
      R.pn[tid] = t - R.t0[tid];
      int rst = 0;
      if (t + 1 >= R.end[tid]) {                               // the row's utterance ends with this step: enter its next segment
        const int k1 = R.k[tid] + 1, e0 = R.end[tid];
        R.k[tid] = k1;
        const bool more = A.pack_utt && tid < A.pack_rows && k1 < A.pack_segs;
        R.utt[tid] = more ? A.pack_utt[tid * A.pack_segs + k1] : -1;
        R.t0[tid] = e0;
        R.end[tid] = more ? A.pack_start[tid * (A.pack_segs + 1) + k1 + 1] : 0x7fffffff;
        rst = 1;
      }
      R.rst[tid] = rst;
    }
    __syncwarp();
    PUSH_MARK(10);
  }
  if (A.prof && tid == 0)
    for (int i = 0; i < 12; ++i) A.prof[(size_t)c * 12 + i] = s_pf[i];
#undef PUSH_MARK
