"""Generation sessions against one-shot generate on one GPU, synthetic weights, 401-frame utterances (a 5 s sentence).

    python tools/time_session.py [--kernel auto|tc] [--frames 401] [--rows 1,8,32] [--chunks 1100,2750,11000] [--out FILE]

--kernel auto (default) times push sessions against one-shot `generate`; --kernel tc times tensor-core sessions
(open_session(kernel='tc')) against one-shot `generate(kernel='tc')`, by default at 33, 128, 129 and 256 rows and chunks of
2750 and 11000 steps (chunks must be multiples of hop there).

Prints the card name and power limit first.  Per row count N:
  * one-shot: `generate` of the N utterances in one call, host clock around the call and its synchronisation;
  * opening: the host time to open N sessions (each runs MelResNet and the conditioning tables of its utterance), synchronised;
  * per chunk size: open N sessions and advance them all by `chunk` steps per launch until done, copying every piece to the
    host as it comes (what a service hands out): time to the first piece on the host, total time, and total / one-shot;
  * the per-run overhead: runs of a few and of many steps (push: 1, 2 and 101 steps; tensor cores: 1 and 11 hops).  Step time
    = slope of the step kernel's time (CUDA events, last_kernel_ms) between the shortest and the longest run; in-kernel fixed
    cost (weight load into shared memory, set-up) = kernel time of the shortest run minus its steps; outside the kernel
    (exchange init, wave epilogue, launches, host) = host time of the shortest run minus its kernel time.
Every timed session output is checked bit for bit against the one-shot output of the same utterances.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tacotronv2_wavernn_chinese_b200 import synth                       # noqa: E402
from tacotronv2_wavernn_chinese_b200.engine import WaveRNNEngine          # noqa: E402


def _sync():
    torch.cuda.synchronize()


def one_shot(eng, mels, ids, seed, kernel):
    _sync()
    t0 = time.perf_counter()
    out = eng.generate(mels, seed=seed, utterance_ids=ids, kernel=kernel)
    wave = out['wave'].cpu().numpy()
    eng.check()
    return time.perf_counter() - t0, wave


def open_all(eng, mels, ids, seed, kernel):
    return [eng.open_session(mels[i], seed=seed, utterance_id=ids[i], kernel=kernel) for i in range(len(ids))]


def open_time(eng, mels, ids, seed, kernel):
    """Median host time (ms) to open the N sessions, synchronised."""
    t = []
    for rep in range(4):
        _sync()
        t0 = time.perf_counter()
        sessions = open_all(eng, mels, ids, seed, kernel)
        _sync()
        if rep:
            t.append(time.perf_counter() - t0)
        for s in sessions:
            s.close()
    return float(np.median(t)) * 1e3


def streamed(eng, mels, ids, seed, chunk, kernel):
    """(time to the first piece, total time, waves [N][wave_len]) of N sessions advanced together."""
    _sync()
    t0 = time.perf_counter()
    sessions = open_all(eng, mels, ids, seed, kernel)
    pieces = [[] for _ in ids]
    first = None
    while not sessions[0].done:                                  # equal lengths: all finish together
        for i, (_lab, w) in enumerate(eng.advance(sessions, chunk)):
            pieces[i].append(w.cpu().numpy())
        if first is None:
            first = time.perf_counter() - t0
        eng.check()
    total = time.perf_counter() - t0
    for s in sessions:
        s.close()
    return first, total, [np.concatenate(p) for p in pieces]


def overhead(eng, mels, ids, seed, kernel):
    """Per-run costs at N rows (see the module docstring), in microseconds."""
    runs = (1, 2, 101) if kernel == 'auto' else (eng.hop, 11 * eng.hop)
    res = {}
    for steps in runs:
        host, kern = [], []
        for rep in range(6):
            sessions = open_all(eng, mels, ids, seed, kernel)
            _sync()
            t0 = time.perf_counter()
            eng.advance(sessions, steps)
            _sync()
            h = time.perf_counter() - t0
            k = eng.last_kernel_ms() * 1e-3
            eng.check()
            for s in sessions:
                s.close()
            if rep:                                              # the first repeat warms up
                host.append(h)
                kern.append(k)
        res[steps] = (float(np.median(host)) * 1e6, float(np.median(kern)) * 1e6)
    lo, hi = runs[0], runs[-1]
    step_us = (res[hi][1] - res[lo][1]) / (hi - lo)
    return dict(step_us=step_us, kernel_fixed_us=res[lo][1] - lo * step_us, outside_kernel_us=res[lo][0] - res[lo][1],
                **{f'run_{n}_steps_host_us': res[n][0] for n in runs}, **{f'run_{n}_steps_kernel_us': res[n][1] for n in runs})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--kernel', choices=('auto', 'tc'), default='auto')
    ap.add_argument('--frames', type=int, default=401)
    ap.add_argument('--rows', default=None, help='default 1,8,32 (auto) or 33,128,129,256 (tc)')
    ap.add_argument('--chunks', default=None, help='default 1100,2750,11000 (auto) or 2750,11000 (tc)')
    ap.add_argument('--seed', type=int, default=5)
    ap.add_argument('--out', default='')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('time_session.py needs a CUDA device')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    card = q.stdout.strip() or 'unknown'
    print('card:', card)
    eng = WaveRNNEngine(synth.synth_state_dict(0), synth.DEFAULT_DIMS, device=0)
    tc = a.kernel == 'tc'
    rows_list = a.rows or ('33,128,129,256' if tc else '1,8,32')
    chunks = [int(c) for c in (a.chunks or ('2750,11000' if tc else '1100,2750,11000')).split(',')]
    if tc and any(c % eng.hop for c in chunks):
        sys.exit(f'tensor-core sessions take chunks that are multiples of hop ({eng.hop})')
    print('kernel:', a.kernel, ' max_session_rows:', eng.max_session_rows)
    report = dict(card=card, kernel=a.kernel, frames=a.frames, real_time_step_us=1e6 / synth.DEFAULT_DIMS['sample_rate'],
                  results=[])
    all_equal = True
    for rows in [int(r) for r in rows_list.split(',')]:
        mels = synth.synth_mels(rows, rows, a.frames)
        ids = [1000 + i for i in range(rows)]
        one_shot(eng, mels, ids, a.seed, a.kernel)               # warm-up
        t_one, ref = one_shot(eng, mels, ids, a.seed, a.kernel)
        t_open = open_time(eng, mels, ids, a.seed, a.kernel)
        ov = overhead(eng, mels, ids, a.seed, a.kernel)
        print(f'rows {rows}: one-shot {t_one * 1e3:.1f} ms; open {t_open:.2f} ms ({t_open / rows * 1e3:.0f} us per session); '
              f'per run: step {ov["step_us"]:.2f} us, in-kernel fixed {ov["kernel_fixed_us"]:.1f} us, outside the kernel '
              f'{ov["outside_kernel_us"]:.1f} us')
        entry = dict(rows=rows, one_shot_ms=t_one * 1e3, open_ms=t_open, overhead=ov, chunks=[])
        for chunk in chunks:
            first, total, waves = streamed(eng, mels, ids, a.seed, chunk, a.kernel)
            equal = all(np.array_equal(waves[i], ref[i]) for i in range(rows))
            all_equal &= equal
            print(f'  chunk {chunk:6d}: first piece {first * 1e3:8.1f} ms, total {total * 1e3:8.1f} ms, '
                  f'total / one-shot {total / t_one:.3f}, bit-equal {equal}')
            entry['chunks'].append(dict(chunk=chunk, first_piece_ms=first * 1e3, total_ms=total * 1e3, ratio=total / t_one,
                                        bit_equal=bool(equal)))
        report['results'].append(entry)
    report['all_bit_equal'] = bool(all_equal)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(report, f, indent=1)
    if not all_equal:
        sys.exit('a session output differs from the one-shot output')


if __name__ == '__main__':
    main()
