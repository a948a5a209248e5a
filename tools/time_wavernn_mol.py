"""RAW against MOL WaveRNN generation per lock-step, on synthetic weights, on one GPU.

    python tools/time_wavernn_mol.py [--steps 1100] [--repeats 3]

For each row count the two modes run alternately, `repeats` times each, in one process (kernel=auto: RAW takes the push,
wide-grid or tensor-core kernel, MOL the push or wide-grid kernel).  Prints the card name and power limit first, then per row count
the median microseconds per lock-step of each mode (CUDA events around the step kernel, b200tts_wavernn_last_kernel_ms).
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tacotronv2_wavernn_chinese_b200 import synth                       # noqa: E402
from tacotronv2_wavernn_chinese_b200.engine import WaveRNNEngine          # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=1100)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--rows', default='1,8,32,64,128,256')
    a = ap.parse_args()
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    print('card:', q.stdout.strip() or 'unknown')
    raw = WaveRNNEngine(synth.synth_state_dict(0), synth.DEFAULT_DIMS, device=0)
    mol = WaveRNNEngine(synth.synth_state_dict(0, mode='MOL'), dict(synth.DEFAULT_DIMS, mode='MOL'), device=0)
    T = (a.steps + 274) // 275
    print(f'{"rows":>5} {"RAW us/step":>12} {"kernel":>22} {"MOL us/step":>12} {"kernel":>22} {"MOL/RAW":>8}')
    for rows in [int(r) for r in a.rows.split(',')]:
        mels = synth.synth_mels(1, rows, T)
        t = {'RAW': [], 'MOL': []}
        names = {}
        for rep in range(a.repeats + 1):                 # the first round warms both up
            for mode, eng in (('RAW', raw), ('MOL', mol)):
                eng.generate(mels, seed=rep, max_steps=a.steps, want_wave=False)
                ms = eng.last_kernel_ms()
                names[mode] = eng.last_kernel()
                if rep:
                    t[mode].append(ms * 1e3 / a.steps)
        r, m = float(np.median(t['RAW'])), float(np.median(t['MOL']))
        print(f'{rows:>5} {r:>12.1f} {names["RAW"]:>22} {m:>12.1f} {names["MOL"]:>22} {m / r:>8.2f}', flush=True)


if __name__ == '__main__':
    main()
