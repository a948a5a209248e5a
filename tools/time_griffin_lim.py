#!/usr/bin/env python
"""Time Griffin-Lim mel inversion (60 iterations) on the GPU for 1, 8 and 32 config-4-length mels, next to the numpy float64
oracle's CPU time for one sentence.

    python tools/time_griffin_lim.py [--reps 5] [--out timing.json]

The mel is the config-4 sentence of tests/golden/taco_run_from_graph.npz (405 frames = 111 100 samples, 5.04 s of audio).
GPU time: CUDA events around `GriffinLimEngine.run` after one warm-up call, median of --reps.  The GPU name and power limit
are printed in the same run (nvidia-smi query, read only).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_facts():
    import torch
    facts = {'gpu': torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        facts['power_limit_and_max_sm_clock'] = q
    except Exception as e:                               # the timing is still valid; the limit is then unknown
        facts['power_limit_and_max_sm_clock'] = f'unavailable ({e})'
    return facts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--iters', type=int, default=60)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    from tacotron_hparams import hparams
    from tacotronv2_wavernn_chinese_b200.tacotron.griffin_lim import GriffinLimEngine
    from oracle import griffin_lim_oracle as go
    mel = np.load(os.path.join(ROOT, 'tests', 'golden', 'taco_run_from_graph.npz'))['mel_graph']       # (405, 80)
    T = mel.shape[0]
    eng = GriffinLimEngine(hparams, device=0)
    res = dict(gpu_facts(), frames=T, samples=275 * (T - 1), iterations=args.iters, reps=args.reps, gpu_ms={})
    for B in (1, 8, 32):
        mels = np.repeat(mel[None], B, axis=0)
        x = torch.as_tensor(mels, device='cuda')
        eng.run(x, seed=1, n_iters=args.iters)                                              # warm-up (allocations)
        torch.cuda.synchronize()
        times = []
        for r in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            eng.run(x, seed=1, n_iters=args.iters)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        ms = float(np.median(times))
        res['gpu_ms'][B] = {'batch_ms': ms, 'ms_per_sentence': ms / B, 'min_batch_ms': float(min(times)),
                            'realtime_factor': (275 * (T - 1) / 22050.0) * B / (ms / 1000.0)}
        print(f'B={B:2d}: {ms:8.2f} ms per batch, {ms / B:7.3f} ms per sentence', flush=True)
    rs = np.random.RandomState(0)
    t0 = time.perf_counter()
    go.inv_mel_spectrogram(mel.T, rs.rand(go.N_BINS, T), n_iters=args.iters)
    res['cpu_oracle_ms_per_sentence'] = (time.perf_counter() - t0) * 1000.0
    res['cpu_threads'] = os.cpu_count()
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
