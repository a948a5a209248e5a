"""`Synthesizer` with the reference's surface (tacotron_synthesize.py:38-127), computed on the GPU.

    synth = Synthesizer(); synth.load('logs-Tacotron-2/taco_pretrained', symbols=...)
    mel_path = synth.synthesize('m ao2 h a2 ...', out_dir, idx, step)      # writes step-{step}-{idx}-mel-pred.npy

Encoder, decoder loop and postnet all run through libb200tts (b200tts_taco_encode / _decode / _postnet); the checkpoint is
the reference's TF bundle read without TensorFlow (tacotron/ckpt.py).  Not reproduced: the Griffin-Lim preview wav and the
matplotlib PNGs the reference also writes (:110-111, :118-125) -- feature extraction / plotting are out of scope.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from . import ckpt
from .engine import TacoDecoderEngine
from .text import Symbols, build_symbols

MAX_ABS_VALUE = 4.0          # tacotron_hparams.py:99, symmetric_mels=True -> T2_output_range = (-4, 4)


class Synthesizer:
    def __init__(self):
        self.engine = None
        self.symbols = None
        self.step = 0
        self.max_iters = 2000          # tacotron_hparams.py:158

    def load(self, checkpoint_path, hparams=None, symbols=None, train_txt='train.txt', device=None):
        """checkpoint_path: TF checkpoint prefix or the directory holding the `checkpoint` pointer file (:138-139)."""
        if str(checkpoint_path).endswith('.npz'):          # variables already extracted from the TF bundle (np.savez of ckpt.load_tacotron_weights)
            w = dict(np.load(checkpoint_path))
        else:
            w = ckpt.load_tacotron_weights(checkpoint_path)
        self.step = int(w.get('global_step', 0))
        if symbols is None:
            symbols = build_symbols(train_txt)
        self.symbols = symbols if isinstance(symbols, Symbols) else Symbols(symbols)
        if len(self.symbols) != w['inputs_embedding'].shape[0]:
            raise ValueError(f'symbol table has {len(self.symbols)} entries, the checkpoint embedding {w["inputs_embedding"].shape[0]}')
        if hparams is not None:
            self.max_iters = int(getattr(hparams, 'max_iters', self.max_iters))
        self.engine = TacoDecoderEngine(w, device=device)
        return self

    def mels(self, texts, seed=0, window=False, max_iters=None, utterance_offset=0):
        """Batch of pinyin strings -> (list of np.float32 mel [T_b, 80] scaled to [0,1] like the .npy the reference saves,
        dict with device tensors).  Each sentence decodes until its own stop token (reference graph is batch 1)."""
        seqs = [self.symbols.text_to_sequence(t) for t in texts]
        B, Tx = len(seqs), max(len(s) for s in seqs)
        ids = np.zeros((B, Tx), dtype=np.int32)
        for b, s in enumerate(seqs):
            ids[b, :len(s)] = s
        lengths = np.array([len(s) for s in seqs], dtype=np.int32)
        eng = self.engine
        mem = eng.encode(ids, lengths)
        ms = int(max_iters or self.max_iters)
        # the prenet-dropout Philox stream is keyed by the GLOBAL sentence index: a sentence's mel must not depend on
        # how the batch is sharded over ranks
        dec = eng.decode(mem, lengths, seed=seed, utterance_offset=utterance_offset, max_steps=ms, window=window, want_align=True)
        mel = eng.postnet(dec['frames'], dec['nsteps'])
        n = dec['nsteps'].cpu().numpy()
        if (n < 0).any():
            raise RuntimeError('Tacotron decoder kernel gave up waiting for a peer thread block (nsteps < 0); results are invalid')
        stop = dec['stop'].cpu().numpy()
        mel_h = mel.cpu().numpy()
        out = []
        for b in range(B):
            rounded = np.round(stop[b, :n[b]])
            target = int(np.argmax(rounded == 1)) if (rounded == 1).any() else int(n[b])       # :104-105
            m = np.clip(mel_h[b, :target], -MAX_ABS_VALUE, MAX_ABS_VALUE)                        # :107-108
            out.append(np.clip((m + MAX_ABS_VALUE) / (2 * MAX_ABS_VALUE), 0, 1).astype(np.float32))   # :115
        return out, dict(decode=dec, memory=mem, lengths=lengths)

    def synthesize(self, text, out_dir, idx, step=None, seed=0):
        step = self.step if step is None else step
        os.makedirs(out_dir, exist_ok=True)
        mels, info = self.mels([text], seed=seed)
        pred_mel_path = os.path.join(out_dir, f'step-{step}-{idx}-mel-pred.npy')
        np.save(pred_mel_path, mels[0], allow_pickle=False)
        align = info['decode']['align'][0, :mels[0].shape[0] + 1].cpu().numpy()
        alignment_path = os.path.join(out_dir, f'step-{step}-{idx}-align.npy')
        np.save(alignment_path, align, allow_pickle=False)
        return pred_mel_path, alignment_path
