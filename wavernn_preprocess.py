#!/usr/bin/env python
"""Vocoder training pairs with ground-truth-aligned (GTA) mels on an H100 -- drop-in for the reference's
`wavernn_preprocess.py`.

    python wavernn_preprocess.py --data_dir training_data

Reads `{data_dir}/train.txt`, the Tacotron training list (`audio-*.npy|mel-*.npy|time_steps|mel_frames|hanzi|pinyin`, the
layout tacotron_preprocess.py writes).  For every line, into `--out_dir`:
  * `audio-*.npy`  the training audio through `audio.encode_mu_law` (mu = 1024; float32 levels in [0, 1023])   (:147-152)
  * `mel-*.npy`    the recorded mel mapped to [0, 1]: clip((mel + 4) / 8, 0, 1)                               (:154-159)
  * `mel-{idx}-pred.npy`  the GTA mel: Tacotron teacher-forced on the recorded mel (clipped to +-4), frame for frame,
                   then the postnet, clipped, cropped to the target length and mapped to [0, 1]                  (:72-120)
and one line `wav_path|mel_path_new|pred_mel_path|hanzi` per training line to `--index`, paths absolute   (:161-170).
The text fed to the model is the Hanzi field through `get_pyin` (:161, :85); idx is the number in the mel file name (:162).

Deliberate differences from the reference:
  * `--data_dir` is required (the reference hard-codes its author's dataset path, :139); the output directory, the index
    file, the checkpoint and the symbol table are arguments too (the symbol table as in tacotron_synthesize.py).
  * the output directory is never deleted (the reference `rmtree`s it, :134-137); files with the same names are overwritten.
  * no PNG plots of the predicted mel or the alignment (:111, :113-115).
  * the encoder, the teacher-forced decoder loop and the postnet run on the GPU through libb200tts.so, `--batch` sentences per
    launch.  Prenet dropout (on, as in the reference) is Philox keyed by (`--seed`, line index, step, unit), so a line's GTA
    mel depends only on the seed and its position in train.txt, not on `--batch`.
  * every line is parsed before the model is loaded: a malformed line fails before any GPU work.
"""
from __future__ import annotations

import argparse
import os
import time

import numpy as np

from tacotron_hparams import hparams


def parse_line(line, lineno):
    """-> (audio_name, mel_name, hanzi, idx) of one train.txt line (reference :145-162), or ValueError."""
    f = line.strip().split('|')
    if len(f) < 6:
        raise ValueError(f'train.txt line {lineno}: expected 6 "|"-separated fields '
                         '(audio|mel|time_steps|mel_frames|hanzi|pinyin), got {len(f)}')
    audio_name, mel_name, text = f[0].strip(), f[1].strip(), f[-2].strip()
    parts = mel_name.split('-')
    if not audio_name or len(parts) < 2 or not parts[1].split('.')[0].strip() or not text:
        raise ValueError(f'train.txt line {lineno}: cannot take the index from mel file name {mel_name!r} '
                         'or the text is empty')
    return audio_name, mel_name, text, parts[1].split('.')[0].strip()


def read_train_txt(path, limit=None):
    entries = []
    with open(path, encoding='utf-8') as fh:
        for lineno, line in enumerate(fh, 1):
            if not line.strip():
                continue
            entries.append(parse_line(line, lineno))
            if limit is not None and len(entries) >= limit:
                break
    return entries


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[1])
    ap.add_argument('--data_dir', required=True, help='directory holding train.txt and its audio-*.npy / mel-*.npy files')
    ap.add_argument('--out_dir', default='predicted_mel', help='output directory (created if missing, never emptied)')
    ap.add_argument('--index', default='wavernn_training_data.txt', help='the vocoder training list to write')
    ap.add_argument('--checkpoint', default='logs-Tacotron-2/taco_pretrained', help='TF checkpoint prefix or directory')
    ap.add_argument('--train_txt', default=hparams.tacotron_input, help='training list the symbol table is rebuilt from')
    ap.add_argument('--symbols_json', default=None, help='JSON file with a "symbols" list (instead of scanning --train_txt)')
    ap.add_argument('--seed', type=int, default=0, help='Philox seed of the (always on) prenet dropout')
    ap.add_argument('--batch', type=int, default=512, help='sentences per decoder launch')
    ap.add_argument('--limit', type=int, default=None, help='process only the first N lines')
    args = ap.parse_args(argv)
    if args.batch < 1:
        ap.error('--batch must be >= 1')
    if args.limit is not None and args.limit < 1:
        ap.error('--limit must be >= 1')
    list_path = os.path.join(args.data_dir, 'train.txt')
    if not os.path.isfile(list_path):
        ap.error(f'{list_path} not found')
    try:
        entries = read_train_txt(list_path, args.limit)
    except ValueError as e:
        ap.error(str(e))
    from tacotronv2_wavernn_chinese_b200.tacotron import audio
    from tacotronv2_wavernn_chinese_b200.tacotron.pinyin import get_pyin
    from tacotronv2_wavernn_chinese_b200.tacotron.synthesizer import Synthesizer
    symbols = None
    if args.symbols_json:
        import json
        symbols = json.load(open(args.symbols_json, encoding='utf-8'))['symbols']
    synth = Synthesizer().load(args.checkpoint, hparams, symbols=symbols, train_txt=args.train_txt)
    out_dir = os.path.abspath(args.out_dir)                # the reference joins os.getcwd() with its names (:125, :134)
    os.makedirs(out_dir, exist_ok=True)
    mx = hparams.max_abs_value
    t0 = time.time()
    with open(os.path.abspath(args.index), 'w', encoding='utf-8') as res:
        for i0 in range(0, len(entries), args.batch):
            chunk = entries[i0:i0 + args.batch]
            pyins, targets, rows = [], [], []
            for audio_name, mel_name, text, idx in chunk:
                wav = audio.encode_mu_law(np.load(os.path.join(args.data_dir, audio_name)))
                wav_path = os.path.join(out_dir, audio_name)
                np.save(wav_path, wav, allow_pickle=False)
                target = np.load(os.path.join(args.data_dir, mel_name))
                mel = np.clip((target + mx) / (2 * mx), 0, 1.0)
                mel_path_new = os.path.join(out_dir, mel_name)
                np.save(mel_path_new, mel, allow_pickle=False)
                pyins.append(get_pyin(text)[0])
                targets.append(target)
                rows.append((wav_path, mel_path_new, os.path.join(out_dir, f'mel-{idx}-pred.npy'), text))
            preds = synth.gta_mels(pyins, targets, seed=args.seed, utterance_offset=i0)
            for pred, row in zip(preds, rows):
                np.save(row[2], pred, allow_pickle=False)
                res.write('|'.join(row) + '\n')
            res.flush()
            print(f'{i0 + len(chunk)}/{len(entries)} lines, {time.time() - t0:.1f} s')
    return os.path.abspath(args.index)


if __name__ == '__main__':
    main()
