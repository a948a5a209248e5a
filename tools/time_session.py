"""Generation sessions against one-shot generate on one GPU, synthetic weights, 401-frame utterances (a 5 s sentence).

    python tools/time_session.py [--frames 401] [--rows 1,8,32] [--chunks 1100,2750,11000] [--out time_session.json]

Prints the card name and power limit first.  Per row count N:
  * one-shot: `generate` of the N utterances in one call, host clock around the call and its synchronisation;
  * per chunk size: open N sessions and advance them all by `chunk` steps per launch until done, copying every piece to the
    host as it comes (what a service hands out): time to the first piece on the host, total time, and total / one-shot;
  * the per-run overhead: runs of 1, 2 and 101 steps.  Step time = slope of the step kernel's time (CUDA events,
    last_kernel_ms) from 1 to 101 steps; in-kernel fixed cost (weight-blob load into shared memory, set-up) = kernel time of
    1 step minus one step; outside the kernel (exchange init, wave epilogue, launches, host) = host time of a 1-step run
    minus its kernel time.
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


def one_shot(eng, mels, ids, seed):
    _sync()
    t0 = time.perf_counter()
    out = eng.generate(mels, seed=seed, utterance_ids=ids)
    wave = out['wave'].cpu().numpy()
    eng.check()
    return time.perf_counter() - t0, wave


def streamed(eng, mels, ids, seed, chunk):
    """(time to the first piece, total time, waves [N][wave_len]) of N sessions advanced together."""
    _sync()
    t0 = time.perf_counter()
    sessions = [eng.open_session(mels[i], seed=seed, utterance_id=ids[i]) for i in range(len(ids))]
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


def overhead(eng, mels, ids, seed):
    """Per-run costs at N rows (see the module docstring), in microseconds."""
    res = {}
    for steps in (1, 2, 101):
        host, kern = [], []
        for rep in range(6):
            sessions = [eng.open_session(mels[i], seed=seed, utterance_id=ids[i]) for i in range(len(ids))]
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
    step_us = (res[101][1] - res[1][1]) / 100
    return dict(step_us=step_us, kernel_fixed_us=res[1][1] - step_us, outside_kernel_us=res[1][0] - res[1][1],
                run_1_step_host_us=res[1][0], run_2_steps_host_us=res[2][0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=401)
    ap.add_argument('--rows', default='1,8,32')
    ap.add_argument('--chunks', default='1100,2750,11000')
    ap.add_argument('--seed', type=int, default=5)
    ap.add_argument('--out', default='')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('time_session.py needs a CUDA device')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    card = q.stdout.strip() or 'unknown'
    print('card:', card)
    eng = WaveRNNEngine(synth.synth_state_dict(0), synth.DEFAULT_DIMS, device=0)
    report = dict(card=card, frames=a.frames, results=[])
    all_equal = True
    for rows in [int(r) for r in a.rows.split(',')]:
        mels = synth.synth_mels(rows, rows, a.frames)
        ids = [1000 + i for i in range(rows)]
        one_shot(eng, mels, ids, a.seed)                         # warm-up
        t_one, ref = one_shot(eng, mels, ids, a.seed)
        ov = overhead(eng, mels, ids, a.seed)
        print(f'rows {rows}: one-shot {t_one * 1e3:.1f} ms; per run: step {ov["step_us"]:.2f} us, in-kernel fixed '
              f'{ov["kernel_fixed_us"]:.1f} us, outside the kernel {ov["outside_kernel_us"]:.1f} us')
        entry = dict(rows=rows, one_shot_ms=t_one * 1e3, overhead=ov, chunks=[])
        for chunk in [int(c) for c in a.chunks.split(',')]:
            first, total, waves = streamed(eng, mels, ids, a.seed, chunk)
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
