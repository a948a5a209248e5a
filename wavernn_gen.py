#!/usr/bin/env python
"""Vocode a mel `.npy` with WaveRNN on an H100 -- drop-in for the reference's `wavernn_gen.py`.

Same command line (reference wavernn_gen.py:49-61), same input contract (float32 `(T, 80)` mel in [0, 1], :22-28), same
output name `./wavernn_inference_output/{stem}_gen_NOT_BATCHED_step={k}k.wav` (:35-39, :124).  Deliberate differences:
  * the model runs on the GPU through libb200tts.so (the reference pins `device = cpu`, :93); `--force_cpu` is refused
    because this build has no CPU path.
  * `.wav` input is refused: that branch of the reference uses undefined names (:19, :30) and cannot run.
  * `--batched` really selects fold-with-overlap generation (the reference parses the flag, then forces it off, :77).
  * extra flags: `--seed` (Philox stream of the sampler), `--kernel {auto,utterance,grid}`.
"""
from __future__ import annotations

import argparse
import os
import time

import numpy as np
import torch

from tacotronv2_wavernn_chinese_b200.wavernn.models.fatchord_version import WaveRNN
from tacotronv2_wavernn_chinese_b200.wavernn.utils import hparams as hp
from tacotronv2_wavernn_chinese_b200.wavernn.utils.display import simple_table
from tacotronv2_wavernn_chinese_b200.wavernn.utils.paths import Paths

OUT_DIR = './wavernn_inference_output'

# (flags, argparse keywords) -- names and types are the reference's, the wording is ours
CLI = [
    (('--batched', '-b'), dict(dest='batched', action='store_true', help='fold one utterance into a batch (fold-with-overlap)')),
    (('--unbatched', '-u'), dict(dest='batched', action='store_false', help='generate the utterance sample by sample')),
    (('--samples', '-s'), dict(type=int, help='utterances to take from the test set (unused: --file only)')),
    (('--target', '-t'), dict(type=int, help='samples per fold in --batched mode (default hp.voc_target)')),
    (('--overlap', '-o'), dict(type=int, help='cross-fade samples between folds (default hp.voc_overlap)')),
    (('--file', '-f'), dict(type=str, help='mel spectrogram .npy, float32 (T, num_mels) in [0, 1]')),
    (('--voc_weights', '-w'), dict(type=str, help='checkpoint to load instead of logs_wavernn/checkpoints/latest_weights.pyt')),
    (('--gta', '-g'), dict(dest='gta', action='store_true', help='accepted for compatibility, ignored')),
    (('--force_cpu', '-c'), dict(action='store_true', help='refused: there is no CPU path')),
    (('--hp_file',), dict(metavar='FILE', default='wavernn_hparams.py', help='hyper-parameter python file')),
    (('--seed',), dict(type=int, default=None, help='Philox seed of the sampling noise')),
    (('--kernel',), dict(choices=('auto', 'utterance', 'grid'), default='auto', help='generation kernel')),
]


def load_mel(path):
    """`.npy` -> float32 tensor [1, num_mels, T]; shape / range checks as in the reference (:22-28)."""
    path = str(path)
    if not path.endswith('.npy'):
        raise ValueError(f'Expected a .npy mel spectrogram, but got {os.path.splitext(path)[1] or path}!')
    mel = np.load(path).T
    if mel.ndim != 2 or mel.shape[0] != hp.num_mels:
        raise ValueError(f'Expected a numpy array shaped (n_hops, n_mels={hp.num_mels}), but got {mel.T.shape}!')
    lo, hi = float(mel.min()), float(mel.max())
    if hi >= 1.01 or lo <= -0.01:
        raise ValueError(f'Expected spectrogram range in [0,1] but was instead [{lo}, {hi}]')
    return torch.tensor(mel, dtype=torch.float32).unsqueeze(0)


def gen_from_file(model, load_path, save_path, batched, target, overlap, seed=None, kernel='auto'):
    k = model.get_step() // 1000
    mel = load_mel(load_path)
    stem = str(load_path).split('/')[-1].strip().split('.')[0]
    mode = f'gen_batched_target{target}_overlap{overlap}' if batched else 'gen_NOT_BATCHED'
    save_str = os.path.join(str(save_path), f'{stem}_{mode}_step={k}k.wav')
    t0 = time.time()
    wav = model.generate(mel, save_str, batched, target, overlap, hp.mu_law, seed=seed, kernel=kernel)
    dt = time.time() - t0
    print(f'\n\nstep = {k * 1000}')
    print(f'{len(wav)} samples in {dt:.2f} s  ({len(wav) / dt / 1000:.1f} kHz, RTF {dt / (len(wav) / hp.sample_rate):.3f}) -> {save_str}')
    return save_str


def build_model():
    dims = dict(rnn_dims=hp.voc_rnn_dims, fc_dims=hp.voc_fc_dims, bits=hp.bits, pad=hp.voc_pad,
                upsample_factors=hp.voc_upsample_factors, feat_dims=hp.num_mels, compute_dims=hp.voc_compute_dims,
                res_out_dims=hp.voc_res_out_dims, res_blocks=hp.voc_res_blocks, hop_length=hp.hop_length,
                sample_rate=hp.sample_rate, mode=hp.voc_mode)
    return WaveRNN(**dims)


def main(argv=None):
    parser = argparse.ArgumentParser(description='WaveRNN vocoder on H100')
    for flags, kw in CLI:
        parser.add_argument(*flags, **kw)
    parser.set_defaults(batched=None)
    args = parser.parse_args(argv)

    hp.configure(args.hp_file)
    target = args.target if args.target is not None else hp.voc_target
    overlap = args.overlap if args.overlap is not None else hp.voc_overlap
    batched = hp.voc_gen_batched if args.batched is None else args.batched
    if args.force_cpu:
        raise SystemExit('--force_cpu: this build runs the generation loop on sm_90a only; there is no CPU fallback')
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device visible; the WaveRNN path has no CPU fallback')
    print('Using device:', torch.device('cuda'))
    print('\nInitialising Model...\n')
    model = build_model()
    weights = args.voc_weights or Paths(hp.voc_model_id).voc_latest_weights
    print(weights)
    model.load(weights)
    simple_table([('Generation Mode', 'Batched' if batched else 'Unbatched'),
                  ('Target Samples', target if batched else 'N/A'),
                  ('Overlap Samples', overlap if batched else 'N/A')])
    if args.file:
        os.makedirs(OUT_DIR, exist_ok=True)
        gen_from_file(model, args.file, OUT_DIR, batched, target, overlap, seed=args.seed, kernel=args.kernel)
    print('\n\nExiting...\n')


if __name__ == '__main__':
    main()
