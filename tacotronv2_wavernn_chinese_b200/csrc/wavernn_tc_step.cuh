// The body of wavernn_tc_kernel and wavernn_tc_session_kernel (wavernn_tc.cuh): included inside each kernel, with `SESS`
// (constexpr bool) and `sio` (TcSessIO) declared by the includer.  Each kernel is thus compiled from its own copy of the text,
// so the one-shot kernel's code is exactly what it was before sessions existed; `if constexpr (SESS)` and `SESS ? :` select the
// per-session rows, state and addressing.  Not a standalone header.
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
      if constexpr (SESS) {                                // a resumed row: the h1 and W_hh1 . h1 its previous run saved
#pragma unroll
        for (int g = 0; g < kTcMaxGroups; ++g)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int grow = g * kTcRows + rows[h];
            if (g >= ng || grow >= A.B || sio.row[grow].pos == 0) continue;
            const float* st = sio.row[grow].state;
#pragma unroll
            for (int qi = 0; qi < 4; ++qi) h1own[g][4 * h + qi] = st[kTcSessH1 + 16 * R.ci + uq[qi]];
#pragma unroll
            for (int f = 0; f < 24; ++f)
              if (((f >> 1) & 1) == h) ghs[g][f] = st[tc_sess_gh1(f, c, R.ci)];
          }
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
          if constexpr (SESS) {                            // a resumed row's first x: the last label of its previous run
            if (t == 0) {
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int grow = g * kTcRows + rows[h];
                if (grow < A.B && sio.row[grow].pos > 0)
                  x[h] = label_to_float(reinterpret_cast<const int*>(sio.row[grow].state)[kTcSessLabel], ncls_m1);
              }
            }
          }
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
                if constexpr (SESS) {                      // a row stores the labels of its own steps; the last one is the next x
                  if (R.ci == 0 && c == 0 && t - 1 < sio.row[grow].n) {
                    sio.labels[(size_t)grow * sio.ld + (t - 1)] = (int16_t)label;
                    if (t == A.steps) reinterpret_cast<int*>(sio.row[grow].state)[kTcSessLabel] = label;
                  }
                } else {
                  if (R.ci == 0 && c == 0) A.labels[(size_t)grow * A.S + (t - 1)] = (int16_t)label;
                }
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
          if constexpr (SESS) {                            // the last lock-step: a row that ran the whole run saves h1 and W_hh1 . h1
            if (t == A.steps - 1) {
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int grow = g * kTcRows + rows[h];
                if (grow >= A.B || sio.row[grow].n != A.steps) continue;
                float* st = sio.row[grow].state;
#pragma unroll
                for (int qi = 0; qi < 4; ++qi) st[kTcSessH1 + 16 * R.ci + uq[qi]] = h1own[g][4 * h + qi];
#pragma unroll
                for (int f = 0; f < 24; ++f)
                  if (((f >> 1) & 1) == h) st[tc_sess_gh1(f, c, R.ci)] = ghs[g][f];
              }
            }
          }
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
      if constexpr (SESS) {                                // a resumed row: the h2 and W_hh2 . h2 its previous run saved
#pragma unroll
        for (int g = 0; g < kTcMaxGroups; ++g)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int grow = g * kTcRows + rows[h];
            if (g >= ng || grow >= A.B || sio.row[grow].pos == 0) continue;
            const float* st = sio.row[grow].state;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int u = 8 * R.ci + 2 * c + e;
              h2own[g][2 * h + e] = st[kTcSessH2 + u];
#pragma unroll
              for (int gate = 0; gate < 3; ++gate) ghs[g][4 * gate + 2 * h + e] = st[kTcSessGh2 + gate * 512 + u];
            }
          }
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
            const float* tb = SESS ? sio.row[src].tab + ((size_t)tc_sess_frame(sio.row[src], t, A.hop) * 128 + 2 * R.ci + (c >> 1)) * kPushCondRows + 32 + 2 * (c & 1)
                                   : A.tab + (((size_t)src * (A.T + 1) + fr) * 128 + 2 * R.ci + (c >> 1)) * kPushCondRows + 32 + 2 * (c & 1);
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
          if constexpr (SESS) {                            // the last lock-step: a row that ran the whole run saves h2 and W_hh2 . h2
            if (t == A.steps - 1) {
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int grow = g * kTcRows + rows[h];
                if (grow >= A.B || sio.row[grow].n != A.steps) continue;
                float* st = sio.row[grow].state;
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  const int u = 8 * R.ci + 2 * c + e;
                  st[kTcSessH2 + u] = h2own[g][2 * h + e];
#pragma unroll
                  for (int gate = 0; gate < 3; ++gate) st[kTcSessGh2 + gate * 512 + u] = ghs[g][4 * gate + 2 * h + e];
                }
              }
            }
          }
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
            const float* tb = SESS ? sio.row[src].tab + ((size_t)tc_sess_frame(sio.row[src], t, A.hop) * 128 + 16 * R.ci + (c >> 1)) * kPushCondRows + trow + 2 * (c & 1)
                                   : A.tab + (((size_t)src * (A.T + 1) + fr) * 128 + 16 * R.ci + (c >> 1)) * kPushCondRows + trow + 2 * (c & 1);
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
                float q4[4];
                if constexpr (SESS) {                      // the session's key; the step is the step within the utterance
                  philox_exp4(sio.row[grow].seed, sio.row[grow].id, (uint32_t)(sio.row[grow].pos + t), (uint32_t)(cls >> 2), q4);
                } else {
                  const unsigned long long uid = A.utt_ids ? A.utt_ids[grow] : A.utt_offset + (unsigned long long)grow;
                  philox_exp4(A.seed, uid, (uint32_t)t, (uint32_t)(cls >> 2), q4);
                }
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
            // SESS: the row's own frame (all rows share the FIR phase ph0) and frame count
            const int frs = SESS ? tc_sess_frame(sio.row[src], t0, A.hop) : fr, Ts = SESS ? sio.row[src].T : A.T;
#pragma unroll
            for (int p = 0; p < 2; ++p) {
              const int c4l = 2 * p + half;                                        // 4-unit block inside this CTA's 16 units
              const float* base = SESS ? sio.row[src].tab + ((size_t)frs * 128 + 4 * R.ci + c4l) * kPushCondRows
                                       : A.tab + (((size_t)src * (A.T + 1) + fr) * 128 + 4 * R.ci + c4l) * kPushCondRows;
              const float v0 = __ldg(base + 16 + i16);
              float pm[kMaxTaps];
#pragma unroll
              for (int j = 0; j < kMaxTaps; ++j) {
                const int f = frs + j - A.NT / 2;
                pm[j] = (j < A.NT && f >= 0 && f < Ts) ? __ldg(base + (ptrdiff_t)(f - frs) * (ptrdiff_t)fstride + i16) : 0.f;
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
