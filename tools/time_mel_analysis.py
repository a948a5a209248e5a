#!/usr/bin/env python
"""Time mel analysis (the full `_process_utterance_v1` chain: trim, pre-emphasis, rescale, mel, training audio) on the GPU for
1, 32 and 256 five-second utterances and for 10 000 utterances of mixed length, next to the numpy float64 oracle's CPU time
for one utterance.

    python tools/time_mel_analysis.py [--reps 5] [--out timing.json]

The signals are seeded: consecutive 5 s windows of the fixture's speech (tests/golden/mel_analysis_from_reference.npz, 4.0 s,
repeated to length) scaled by a seeded gain and with seeded -60 dBFS noise added, so every row is different.  The 10 000
utterances are 2-10 s long (uniform), sorted by length and analysed in calls of --chunk rows, as a dataset tool would do.
GPU time: CUDA events around `MelAnalysisEngine.run` (inputs already on the device, outputs left there) after one warm-up call
of every shape, median of --reps.  The GPU name and power limit are printed in the same run (nvidia-smi query, read only).
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.time_griffin_lim import gpu_facts       # noqa: E402

SR = 22050


def signals(n_samples, rs):
    """Rows of the fixture's speech, repeated to length, each with its own offset, gain and noise."""
    pcm = np.load(os.path.join(ROOT, 'tests', 'golden', 'mel_analysis_from_reference.npz'))['speech_pcm'].astype(np.float32) / 32768
    out = []
    for n in n_samples:
        off = rs.randint(0, len(pcm))
        x = np.resize(np.roll(pcm, -off), n) * rs.uniform(0.3, 1.0)
        out.append((x + rs.standard_normal(n) * 1e-3).astype(np.float32))
    return out


def batch_of(wavs, torch):
    L = max(len(w) for w in wavs)
    b = np.zeros((len(wavs), L), np.float32)
    for i, w in enumerate(wavs):
        b[i, :len(w)] = w
    return torch.as_tensor(b, device='cuda'), np.array([len(w) for w in wavs])


def timed(fn, reps, torch):
    fn()                                                    # warm-up (allocations)
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return float(np.median(times)), float(min(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--n_mixed', type=int, default=10000)
    ap.add_argument('--chunk', type=int, default=1000)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    from tacotron_hparams import hparams
    from tacotronv2_wavernn_chinese_b200.tacotron.mel_analysis import MelAnalysisEngine, preprocess_flags
    from oracle import mel_analysis_oracle as mo
    flags = preprocess_flags(hparams)
    eng = MelAnalysisEngine(hparams, device=0)
    rs = np.random.RandomState(0)
    res = dict(gpu_facts(), flags=flags, reps=args.reps, gpu_ms={})
    five = signals([5 * SR] * 256, rs)
    for B in (1, 32, 256):
        x, ln = batch_of(five[:B], torch)
        ms, mn = timed(lambda: eng.run(x, ln, flags=flags, want_audio=True), args.reps, torch)
        res['gpu_ms'][f'{B} x 5 s'] = {'batch_ms': ms, 'min_batch_ms': mn, 'ms_per_utterance': ms / B,
                                        'audio_seconds_per_second': 5.0 * B / (ms / 1000.0)}
        print(f'B={B:3d} x 5 s: {ms:8.3f} ms per call, {ms / B:7.4f} ms per utterance', flush=True)
    lens = np.sort(rs.randint(2 * SR, 10 * SR + 1, size=args.n_mixed))
    mixed = signals(lens, rs)
    chunks = [batch_of(mixed[i:i + args.chunk], torch) for i in range(0, len(mixed), args.chunk)]

    def all_chunks():
        for x, ln in chunks:
            eng.run(x, ln, flags=flags, want_audio=True)
    ms, mn = timed(all_chunks, args.reps, torch)
    res['gpu_ms'][f'{args.n_mixed} x 2-10 s'] = {'total_ms': ms, 'min_total_ms': mn, 'ms_per_utterance': ms / args.n_mixed,
                                                  'audio_seconds': float(lens.sum() / SR), 'calls': len(chunks),
                                                  'audio_seconds_per_second': float(lens.sum() / SR) / (ms / 1000.0)}
    print(f'{args.n_mixed} utterances of 2-10 s ({lens.sum() / SR / 3600:.1f} h of audio) in {len(chunks)} calls: {ms:.1f} ms',
          flush=True)
    t0 = time.perf_counter()
    for w in five[:4]:
        mo.process_utterance(w)
    res['cpu_oracle_ms_per_5s_utterance'] = (time.perf_counter() - t0) * 1000.0 / 4
    res['cpu_threads'] = os.cpu_count()
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
