#!/usr/bin/env python
"""Vocode a mel `.npy` with WaveRNN on an H100 -- drop-in for the reference's `wavernn_gen.py`.

Same command line (reference wavernn_gen.py:49-61), same input contract (float32 `(T, 80)` mel in [0, 1], :22-28), same
output name `./wavernn_inference_output/{stem}_gen_NOT_BATCHED_step={k}k.wav` (:35-39, :124).  Deliberate differences:
  * the model runs on the GPU through libb200tts.so (the reference pins `device = cpu`, :93); `--force_cpu` is refused
    because this build has no CPU path.
  * `.wav` input is copy-synthesis: the file is loaded, written back as `__{stem}__{k}k_steps_target.wav` (:19, whose
    undefined `file_name` is read as the stem), analysed on the GPU and vocoded.  The reference's branch would call
    `wavernn/utils/dsp.py: melspectrogram` (fmax = sr/2, no ref_level_db, [0, 1] normalisation, reflect padding) and crashes
    before it gets there; we compute instead the features the shipped checkpoint was trained on: the Tacotron preprocessor's
    `_process_utterance_v1` (trim silence, pre-emphasis, rescale, melspectrogram with the Tacotron hparams) mapped to [0, 1]
    as wavernn_preprocess.py:155-157 does.  The file must already be at the model's sample rate (no resampling).
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
from tacotronv2_wavernn_chinese_b200.wavernn.utils.dsp import save_wav
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
    (('--file', '-f'), dict(type=str, help='mel spectrogram .npy, float32 (T, num_mels) in [0, 1], or a .wav to re-synthesise')),
    (('--voc_weights', '-w'), dict(type=str, help='checkpoint to load instead of logs_wavernn/checkpoints/latest_weights.pyt')),
    (('--gta', '-g'), dict(dest='gta', action='store_true', help='accepted for compatibility, ignored')),
    (('--force_cpu', '-c'), dict(action='store_true', help='refused: there is no CPU path')),
    (('--hp_file',), dict(metavar='FILE', default='wavernn_hparams.py', help='hyper-parameter python file')),
    (('--seed',), dict(type=int, default=None, help='Philox seed of the sampling noise')),
    (('--kernel',), dict(choices=('auto', 'utterance', 'grid'), default='auto', help='generation kernel')),
]


def tacotron_hparams():
    """The Tacotron hparams the WaveRNN features are computed with; they must agree with the WaveRNN hparams on the sample
    rate, the hop and the number of mels."""
    from tacotron_hparams import hparams as taco
    for a, b in (('sample_rate', 'sample_rate'), ('hop_size', 'hop_length'), ('num_mels', 'num_mels')):
        if getattr(taco, a) != getattr(hp, b):
            raise ValueError(f'Tacotron {a} = {getattr(taco, a)} differs from WaveRNN {b} = {getattr(hp, b)}')
    return taco


def wav_to_mel(wav):
    """Float32 samples -> the [0, 1] mel [num_mels, T] WaveRNN was trained on: `_process_utterance_v1`'s features
    (tacotron/datasets/preprocessor.py:52-121) through clip((mel + 4) / 8, 0, 1) (wavernn_preprocess.py:155-157)."""
    from tacotronv2_wavernn_chinese_b200.tacotron import audio
    taco = tacotron_hparams()
    mel = audio.preprocess_wav(wav, taco)[0]                      # [T][num_mels], symmetric scale
    m = taco.max_abs_value
    return np.clip((mel + m) / (2 * m), 0, 1).T


def load_mel(path, target_path=None):
    """`.npy` or `.wav` -> float32 tensor [1, num_mels, T]; shape / range checks as in the reference (:22-28).  A `.wav` is
    loaded at hp.sample_rate, written to `target_path` (if given) and analysed (see the module docstring)."""
    path = str(path)
    if path.endswith('.wav'):
        from tacotronv2_wavernn_chinese_b200.tacotron import audio
        wav = audio.load_wav(path, hp.sample_rate)
        if target_path is not None:
            save_wav(wav, target_path)
        mel = wav_to_mel(wav)
    elif path.endswith('.npy'):
        mel = np.load(path).T
    else:
        raise ValueError(f'Expected an extension of .wav or .npy, but got {os.path.splitext(path)[1] or path}!')
    if mel.ndim != 2 or mel.shape[0] != hp.num_mels:
        raise ValueError(f'Expected a numpy array shaped (n_hops, n_mels={hp.num_mels}), but got {mel.T.shape}!')
    lo, hi = float(mel.min()), float(mel.max())
    if hi >= 1.01 or lo <= -0.01:
        raise ValueError(f'Expected spectrogram range in [0,1] but was instead [{lo}, {hi}]')
    return torch.tensor(mel, dtype=torch.float32).unsqueeze(0)


def gen_from_file(model, load_path, save_path, batched, target, overlap, seed=None, kernel='auto'):
    k = model.get_step() // 1000
    stem = str(load_path).split('/')[-1].strip().split('.')[0]
    mel = load_mel(load_path, target_path=os.path.join(str(save_path), f'__{stem}__{k}k_steps_target.wav'))
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
