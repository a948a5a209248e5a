"""Speaking-rate control on the GPU: how long the shipped checkpoint speaks at each bias, and what the biased decoder costs.

    python tools/rate_response.py [--out DIR]

1. Length response: every sentence of tests/golden/taco_symbols.json (67) at every delta of RESPONSE_DELTAS, window off and on,
   Philox seed RESPONSE_SEED (tests/test_tacotron_rate_gpu.py length_response, the run its test 6 asserts on).  Per delta: the
   median, min and max over the sentences of (cut length at delta) / (cut length at 0), where the cut is the synthesizer's
   stop-token cut; how many stops fired before max_iters; in how many sentences the attention argmax at the stop step lies in
   the last 3 tokens.  Also the seed-to-seed spread at delta 0 (seeds RESPONSE_SEED + 1, + 2 against RESPONSE_SEED).
2. Cost: per-step decode time of the biased (taco_grid_biased_kernel / taco_decoder_biased_kernel) against the unbiased
   instantiation at B = 1 and B = 32: synthetic weights whose stop token never fires, so every run is exactly STEPS steps;
   the two alternate, CUDA events around each run, median of REPS.
Needs the shipped Tacotron checkpoint (reference checkout or its travel copy under oracle/_ref/) for part 1.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]

STEPS, REPS = 400, 9


def _gpu():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                                   # noqa: BLE001
        q = f'nvidia-smi unavailable ({e})'
    return f'{name}, power limit / max SM clock: {q}'


def response_table(eng):
    from test_tacotron_rate_gpu import RESPONSE_DELTAS, RESPONSE_SEED, length_response
    rows = []
    for window in (False, True):
        res, ln = length_response(eng, window)
        base = res[0.0][0].astype(np.float64)
        noise = np.concatenate([length_response(eng, window, deltas=(0.0,), seed=s)[0][0.0][0] / base
                                for s in (RESPONSE_SEED + 1, RESPONSE_SEED + 2)])
        print(f'window {"on" if window else "off"}: seed-to-seed length ratio at delta 0: '
              f'median {np.median(noise):.3f}, min {noise.min():.3f}, max {noise.max():.3f}')
        for d in RESPONSE_DELTAS:
            cut, ns, am = res[d]
            r = cut / base
            row = dict(window=window, delta=d, median=float(np.median(r)), min=float(r.min()), max=float(r.max()),
                       stops=int((ns < 2000).sum()), attention_at_end=int((am >= ln - 3).sum()), sentences=len(ln),
                       mean_frames=float(cut.mean()))
            rows.append(row)
            print(f'  delta {d:+.2f}: length ratio median {row["median"]:.3f} (min {row["min"]:.3f}, max {row["max"]:.3f}), '
                  f'mean {row["mean_frames"]:.1f} frames; stop fired {row["stops"]}/{len(ln)}; '
                  f'attention in the last 3 tokens at the stop {row["attention_at_end"]}/{len(ln)}', flush=True)
        rows.append(dict(window=window, noise_median=float(np.median(noise)), noise_min=float(noise.min()),
                         noise_max=float(noise.max())))
    return rows


def step_cost():
    import torch
    from taco_common import synth_taco_weights
    from tacotronv2_wavernn_chinese_b200.tacotron.engine import TacoDecoderEngine
    w = synth_taco_weights(7)
    w['decoder/stop_token_projection/projection_stop_token_projection/bias'] = np.array([-20.0], np.float32)   # never stops
    eng = TacoDecoderEngine(w)
    rows = []
    for B in (1, 32):
        mem = torch.as_tensor(np.random.RandomState(B).uniform(-1, 1, (B, 40, 512)).astype(np.float32)).cuda()
        runs = {'unbiased': lambda: eng.decode(mem, seed=1, max_steps=STEPS, want_align=False),
                'biased': lambda: eng.decode(mem, seed=1, max_steps=STEPS, want_align=False, mu_bias=0.1)}
        for f in runs.values():                              # warm-up: module load, attribute setting, buffers
            assert int(f()['nsteps'].min()) == STEPS
        times = {k: [] for k in runs}
        for _ in range(REPS):
            for k, f in runs.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                f()
                b.record()
                torch.cuda.synchronize()
                times[k].append(a.elapsed_time(b) * 1e3 / STEPS)
        row = dict(B=B, steps=STEPS, reps=REPS, **{f'{k}_us_per_step': float(np.median(v)) for k, v in times.items()},
                   **{f'{k}_spread_us': [float(min(v)), float(max(v))] for k, v in times.items()})
        rows.append(row)
        print(f'B={B:2d} ({"taco_grid" if B == 1 else "taco_decoder"} kernels): unbiased {row["unbiased_us_per_step"]:.2f} us/step '
              f'(range {row["unbiased_spread_us"][0]:.2f}-{row["unbiased_spread_us"][1]:.2f}), biased {row["biased_us_per_step"]:.2f} '
              f'(range {row["biased_spread_us"][0]:.2f}-{row["biased_spread_us"][1]:.2f}), median of {REPS} x {STEPS} steps', flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='directory for rate_response.json')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('rate_response.py measures on the GPU and has no CPU mode')
    gpu = _gpu()
    print(gpu)
    from taco_common import real_taco_weights
    from tacotronv2_wavernn_chinese_b200.tacotron.engine import TacoDecoderEngine
    w = real_taco_weights()
    if w is None:
        raise SystemExit('the length response needs the shipped Tacotron checkpoint')
    result = dict(gpu=gpu, response=response_table(TacoDecoderEngine(w)), cost=step_cost())
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'rate_response.json'), 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
