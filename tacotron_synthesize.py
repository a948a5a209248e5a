#!/usr/bin/env python
"""Text (pinyin tokens) -> mel `.npy` with Tacotron-2 on an H100 -- drop-in for the reference's `tacotron_synthesize.py`.

    python tacotron_synthesize.py --text 'm ao2 h a2 d eng3 b ei4 l ei4 。'

Same output contract: `./tacotron_inference_output/step-{step}-{md5(text)}-mel-pred.npy`, float32 (T, 80) =
clip((mel + 4) / 8, 0, 1) (reference :114-116, :187-191), which `wavernn_gen.py --file` consumes.  Differences:
  * encoder / decoder loop / postnet run on the GPU through libb200tts.so; the TF checkpoint is read without TensorFlow.
  * `--text` takes Hanzi (or Hanzi mixed with inline pinyin / digits / #1-#4 prosody marks) exactly like the reference: the
    text goes through `get_pyin` (:187; restated TF-free in tacotronv2_wavernn_chinese_b200/tacotron/pinyin.py over the same two
    public dictionaries, checked string-for-string against the reference on 300 train.txt lines).  Space separated pinyin
    tokens pass through it unchanged, so the round-1 form `--text 'm ao2 h a2 ...'` keeps working.
  * no PNG plots (the alignment is saved as `...-align.npy` instead).  The preview wav `step-{step}-{idx}-wav-from-mel.wav`
    (:110-112) is written on request, by one of two vocoders on the GPU in the same process:
      --griffin_lim         the reference's own: Griffin-Lim mel inversion (`audio.inv_mel_spectrogram`, hparams.griffin_lim_iters
                            iterations; the random initial phase is Philox(--seed)), needs only the Tacotron checkpoint;
      --voc_weights PATH    WaveRNN from that checkpoint.
    Either way it is saved through the reference's own writer chain -- DC notch, peak normalisation, int16
    (`tacotron/datasets/audio.py:17-34`, restated in tacotronv2_wavernn_chinese_b200/tacotron/audio.py).
"""
from __future__ import annotations

import argparse
import hashlib
import os
import time

from tacotron_hparams import hparams
from tacotronv2_wavernn_chinese_b200.tacotron.synthesizer import Synthesizer


def preview_wav(mel_path, voc_weights, voc_hp_file, sample_rate, seed=0):
    """mel `.npy` -> `...-wav-from-mel.wav` next to it (reference :110-112, with WaveRNN in place of Griffin-Lim)."""
    import numpy as np
    import torch
    import wavernn_gen
    from tacotronv2_wavernn_chinese_b200.tacotron import audio
    if not wavernn_gen.hp.is_configured():                              # one-shot singleton (wavernn/utils/__init__.py:60-61)
        wavernn_gen.hp.configure(voc_hp_file)
    model = wavernn_gen.build_model()
    model.load(voc_weights)
    mel = np.load(mel_path).T                                          # (80, T) in [0, 1]: the array wavernn_gen.py --file reads
    if mel.shape[1] < 21:                                              # generate() fades out over 20 hops
        mel = np.pad(mel, ((0, 0), (0, 21 - mel.shape[1])))
    wav = model.generate(torch.tensor(mel[None], dtype=torch.float32), None, False, wavernn_gen.hp.voc_target,
                         wavernn_gen.hp.voc_overlap, wavernn_gen.hp.mu_law, seed=seed)
    wav_path = mel_path[:-len('mel-pred.npy')] + 'wav-from-mel.wav'
    audio.save_wav(wav, wav_path, sr=sample_rate)
    return wav_path


def preview_wav_griffin_lim(mel_path, hp, seed=0):
    """mel `.npy` -> `...-wav-from-mel.wav` next to it by Griffin-Lim (reference :110-112).  The saved array is
    clip((mel + 4) / 8, 0, 1), so the mel is taken back as npy * 8 - 4."""
    import numpy as np
    from tacotronv2_wavernn_chinese_b200.tacotron import audio
    mel = np.load(mel_path).astype(np.float32) * (2 * hp.max_abs_value) - hp.max_abs_value     # (T, 80)
    wav = audio.inv_mel_spectrogram(mel.T, hp, seed=seed)
    wav_path = mel_path[:-len('mel-pred.npy')] + 'wav-from-mel.wav'
    audio.save_wav(wav, wav_path, sr=hp.sample_rate)
    return wav_path


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--text', required=True, help='Hanzi sentence (or space separated pinyin tokens)')
    ap.add_argument('--checkpoint', default='logs-Tacotron-2/taco_pretrained', help='TF checkpoint prefix or directory')
    ap.add_argument('--train_txt', default=hparams.tacotron_input, help='training list the symbol table is rebuilt from')
    ap.add_argument('--symbols_json', default=None, help='JSON file with a "symbols" list (instead of scanning --train_txt)')
    ap.add_argument('--hparams', default='', help='comma separated name=value overrides')
    ap.add_argument('--out_dir', default='tacotron_inference_output')
    ap.add_argument('--seed', type=int, default=0, help='Philox seed of the (always on) prenet dropout')
    ap.add_argument('--voc_weights', default=None, help='WaveRNN checkpoint: also write the preview wav step-..-wav-from-mel.wav')
    ap.add_argument('--voc_hp_file', default='wavernn_hparams.py', help='WaveRNN hyper-parameter file (with --voc_weights)')
    ap.add_argument('--griffin_lim', action='store_true', help='also write the preview wav step-..-wav-from-mel.wav by Griffin-Lim')
    ap.add_argument('--mu_bias', type=float, default=0.0,
                    help='speaking rate: the forward-attention speed bias the reference ships switched off '
                         '(tacotron/models/attention.py:163-165, delta_val), added to the transition agent mu at every decoder '
                         'step; finite in [-1, 1], positive is faster (DESIGN.md 3.13 has the measured length response)')
    args = ap.parse_args(argv)
    if args.griffin_lim and args.voc_weights:
        ap.error('--griffin_lim and --voc_weights both choose the preview vocoder; give one')
    if not (abs(args.mu_bias) <= 1.0):
        ap.error('--mu_bias must be finite and in [-1, 1]')
    hp = hparams.parse(args.hparams)
    from tacotronv2_wavernn_chinese_b200.tacotron.pinyin import get_pyin
    pyin, text = get_pyin(args.text)                    # reference :187: pinyin feeds the model, the normalised text names the files
    symbols = None
    if args.symbols_json:
        import json
        symbols = json.load(open(args.symbols_json, encoding='utf-8'))['symbols']
    synth = Synthesizer().load(args.checkpoint, hp, symbols=symbols, train_txt=args.train_txt)
    idx = hashlib.md5(text.encode('utf8')).hexdigest()
    t0 = time.time()
    mel_path, align_path = synth.synthesize(pyin, args.out_dir, idx, seed=args.seed, mu_bias=args.mu_bias)
    print(f'pred_mel_path: {mel_path}')
    if args.voc_weights:
        print(f'wav_path: {preview_wav(mel_path, args.voc_weights, args.voc_hp_file, hp.sample_rate, args.seed)}')
    elif args.griffin_lim:
        print(f'wav_path: {preview_wav_griffin_lim(mel_path, hp, args.seed)}')
    print(f'last: {time.time() - t0} seconds')
    return mel_path


if __name__ == '__main__':
    main()
