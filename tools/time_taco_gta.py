#!/usr/bin/env python
"""Time ground-truth-aligned (GTA) decoding -- the teacher-forced Tacotron decoder loop of wavernn_preprocess.py,
b200tts_taco_decode_gta, one thread block per sentence -- on the length distribution of the reference's train.txt.

    python tools/time_taco_gta.py [--reps 3] [--batch 512] [--out timing.json]

Workload: the 10 000 lines of train.txt (tests/golden/train_txt_lengths.npz: 64-624 mel frames, 2.92 M decoder steps in all;
6-71 pinyin tokens, plus the EOS symbol).  Synthetic weights with the checkpoint's shapes (tests/taco_common.py), seeded
random encoder memory and targets: the decoder's cost depends on the shapes and lengths, not on the values (no stop rule,
a fixed number of steps per sentence).  Sizes: the first 1, 32 and 132 lines in one launch, and the whole list in
consecutive --batch chunks in train.txt order, as wavernn_preprocess.py runs it.  Philox prenet dropout, no alignment output.
GPU time: CUDA events around `TacoDecoderEngine.decode_gta` (inputs already on the device), after one warm-up call of every
shape, median of --reps.  The GPU name and power limit are printed in the same run (nvidia-smi query, read only).
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from tools.time_griffin_lim import gpu_facts        # noqa: E402
from tools.time_mel_analysis import timed            # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--batch', type=int, default=512)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    from taco_common import synth_taco_weights
    from tacotronv2_wavernn_chinese_b200.tacotron.engine import TacoDecoderEngine
    z = np.load(os.path.join(ROOT, 'tests', 'golden', 'train_txt_lengths.npz'))
    ty = z['mel_frames'].astype(np.int32)
    tx = z['pinyin_tokens'].astype(np.int32) + 1                                   # + EOS (text_to_sequence)
    eng = TacoDecoderEngine(synth_taco_weights(7), device=0)
    rs = np.random.RandomState(0)

    def inputs(lo, hi):
        B, Tx, Ty = hi - lo, int(tx[lo:hi].max()), int(ty[lo:hi].max())
        mem = torch.as_tensor(rs.uniform(-1, 1, (B, Tx, 512)).astype(np.float32), device='cuda')
        tg = torch.as_tensor(rs.uniform(-4, 4, (B, Ty, 80)).astype(np.float32), device='cuda')
        return mem, torch.as_tensor(tx[lo:hi], device='cuda'), tg, torch.as_tensor(ty[lo:hi], device='cuda'), lo

    def run(chunks):
        for mem, ln, tg, tl, lo in chunks:
            eng.decode_gta(mem, ln, tg, tl, seed=1, utterance_offset=lo)

    res = dict(gpu_facts(), reps=args.reps, batch=args.batch, lines=len(ty), decoder_steps=int(ty.sum()), gpu_ms={})
    for B in (1, 32, 132):
        chunks = [inputs(0, B)]
        ms, mn = timed(lambda: run(chunks), args.reps, torch)
        steps = int(ty[:B].sum())
        res['gpu_ms'][f'{B} sentences'] = {'ms': ms, 'min_ms': mn, 'decoder_steps': steps, 'longest': int(ty[:B].max()),
                                           'us_per_step_of_longest': ms * 1000.0 / int(ty[:B].max()),
                                           'steps_per_second': steps / (ms / 1000.0)}
        print(f'{B:4d} sentences ({steps} steps, longest {int(ty[:B].max())}): {ms:9.2f} ms, '
              f'{ms * 1000.0 / int(ty[:B].max()):6.1f} us per step of the longest', flush=True)
    chunks = [inputs(i, min(i + args.batch, len(ty))) for i in range(0, len(ty), args.batch)]
    ms, mn = timed(lambda: run(chunks), args.reps, torch)
    res['gpu_ms'][f'all {len(ty)} lines'] = {'ms': ms, 'min_ms': mn, 'calls': len(chunks), 'ms_per_line': ms / len(ty),
                                             'steps_per_second': float(ty.sum()) / (ms / 1000.0)}
    print(f'all {len(ty)} lines ({int(ty.sum())} steps) in {len(chunks)} calls of {args.batch}: {ms / 1000.0:.2f} s, '
          f'{ms / len(ty):.3f} ms per line', flush=True)
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
