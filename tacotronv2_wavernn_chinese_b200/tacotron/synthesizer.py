"""`Synthesizer` with the reference's surface (tacotron_synthesize.py:38-127), computed on the GPU.

    synth = Synthesizer(); synth.load('logs-Tacotron-2/taco_pretrained', symbols=...)
    mel_path = synth.synthesize('m ao2 h a2 ...', out_dir, idx, step)      # writes step-{step}-{idx}-mel-pred.npy

Encoder, decoder loop and postnet all run through libb200tts (b200tts_taco_encode / _decode / _postnet); the checkpoint is
the reference's TF bundle read without TensorFlow (tacotron/ckpt.py).  The Griffin-Lim preview wav (:110-112) is written by
tacotron_synthesize.py --griffin_lim from the saved mel (tacotron/audio.py inv_mel_spectrogram, on the GPU).  Not reproduced:
the matplotlib PNGs the reference also writes (:111, :118-125) -- plotting is out of scope.

Ground-truth-aligned mels for vocoder training (the reference's wavernn_preprocess.py, its own `Synthesizer`):

    mels = synth.gta_mels(['m ao2 ...'], [target_mel])                        # teacher-forced on the recorded mel
    synth.synthesize_gta(hanzi, 'mel-000001.npy', out_dir, '000001')          # writes mel-000001-pred.npy
"""
from __future__ import annotations

import os

import numpy as np
import torch

from . import ckpt
from .engine import TacoDecoderEngine, mu_bias_array
from .pinyin import get_pyin
from .text import Symbols, build_symbols

MAX_ABS_VALUE = 4.0          # tacotron_hparams.py:99, symmetric_mels=True -> T2_output_range = (-4, 4)


def unit_mel(m):
    """A postnet output [T, 80] (numpy, float32) -> the [0, 1] mel the reference saves (tacotron_synthesize.py:107-108, :115)."""
    m = np.clip(m, -MAX_ABS_VALUE, MAX_ABS_VALUE)
    return np.clip((m + MAX_ABS_VALUE) / (2 * MAX_ABS_VALUE), 0, 1).astype(np.float32)


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

    def _encode(self, texts):
        """Pinyin strings -> (encoder output [B, Tx, enc_dim] CUDA tensor, lengths [B] int32 numpy), Tx the longest."""
        seqs = [self.symbols.text_to_sequence(t) for t in texts]
        lengths = np.array([len(s) for s in seqs], dtype=np.int32)
        ids = np.zeros((len(seqs), int(lengths.max())), dtype=np.int32)
        for b, s in enumerate(seqs):
            ids[b, :len(s)] = s
        return self.engine.encode(ids, lengths), lengths

    def mels(self, texts, seed=0, window=False, max_iters=None, utterance_offset=0, mu_bias=None):
        """Batch of pinyin strings -> (list of np.float32 mel [T_b, 80] scaled to [0,1] like the .npy the reference saves,
        dict with device tensors).  Each sentence decodes until its own stop token (reference graph is batch 1).
        mu_bias: speaking-rate bias, a scalar or one per text (TacoDecoderEngine.decode; positive speaks faster)."""
        mu_bias = mu_bias_array(mu_bias, len(texts))
        mem, lengths = self._encode(texts)
        eng = self.engine
        ms = int(max_iters or self.max_iters)
        # the prenet-dropout Philox stream is keyed by the GLOBAL sentence index: a sentence's mel must not depend on
        # how the batch is sharded over ranks
        dec = eng.decode(mem, lengths, seed=seed, utterance_offset=utterance_offset, max_steps=ms, window=window, want_align=True,
                         mu_bias=mu_bias)
        mel = eng.postnet(dec['frames'], dec['nsteps'])
        n = dec['nsteps'].cpu().numpy()
        if (n < 0).any():
            raise RuntimeError('Tacotron decoder kernel gave up waiting for a peer thread block (nsteps < 0); results are invalid')
        stop = dec['stop'].cpu().numpy()
        mel_h = mel.cpu().numpy()
        out = []
        for b in range(len(texts)):
            rounded = np.round(stop[b, :n[b]])
            target = int(np.argmax(rounded == 1)) if (rounded == 1).any() else int(n[b])       # :104-105
            out.append(unit_mel(mel_h[b, :target]))
        return out, dict(decode=dec, memory=mem, lengths=lengths)

    def decode_device(self, texts, ids, seed=0, window=False, max_iters=None, mu_bias=None):
        """Batch of pinyin strings -> (postnet output [B, max_iters, 80] on the +-4 scale, target lengths [B] int32), both
        CUDA tensors: what `mels` computes before its host copy (rows past a sentence's length are unspecified).  The prenet
        dropout of sentence b is keyed by ids[b], an arbitrary global id, so a sentence's mel does not depend on which others
        share its batch.  Consecutive ids draw the PHILOX stream directly; otherwise each run of consecutive ids gets its keep
        flags from philox_masks, which by its contract equal that stream.  mu_bias: as in `mels`."""
        ids = [int(i) for i in ids]
        if len(ids) != len(texts) or not texts:
            raise ValueError('need one id per text, and at least one text')
        mu_bias = mu_bias_array(mu_bias, len(texts))
        mem, lengths = self._encode(texts)
        eng = self.engine
        ms = int(max_iters or self.max_iters)
        runs = [[ids[0], 1]]
        for i in ids[1:]:
            if i == runs[-1][0] + runs[-1][1]:
                runs[-1][1] += 1
            else:
                runs.append([i, 1])
        if len(runs) == 1:
            dec = eng.decode(mem, lengths, seed=seed, utterance_offset=ids[0], max_steps=ms, window=window, want_align=False,
                             mu_bias=mu_bias)
        else:
            masks = torch.cat([eng.philox_masks(seed, start, count, ms) for start, count in runs])
            dec = eng.decode(mem, lengths, masks=masks, max_steps=ms, window=window, want_align=False, mu_bias=mu_bias)
        mel = eng.postnet(dec['frames'], dec['nsteps'])
        return mel, eng.target_lengths(dec['stop'], dec['nsteps'])

    def open_decodes(self, texts, ids, seed=0, window=False, max_iters=None, mu_bias=None):
        """Encodes 1..128 pinyin strings in one batch and opens their decoder sessions (TacoDecoderEngine.open_decode_sessions),
        to be advanced in slices with `engine.advance_decodes` and finished with `finish_decodes`.  Text b's prenet dropout is keyed
        by (seed, ids[b]) and its frames are bit for bit those of the batch decoder (`taco_decoder_kernel`) on this encoder output.
        A lone text therefore differs in bits from `decode_device`, which decodes a batch of one on the single-sentence kernel."""
        if len(ids) != len(texts) or not texts:
            raise ValueError('need one id per text, and at least one text')
        mem, lengths = self._encode(texts)
        return self.engine.open_decode_sessions(mem, lengths, ids, seed=seed, max_steps=int(max_iters or self.max_iters), window=window,
                                                mu_bias=mu_bias)

    def finish_decodes(self, sessions):
        """Finished decoder sessions -> what `decode_device` returns for them: (postnet output [n, T, 80] on the +-4 scale, target
        lengths [n] int32), both CUDA tensors, T the longest decode (rows past a sentence's length are unspecified).  One postnet
        and one stop-token cut on the device for the whole set."""
        eng = self.engine
        out = eng.decode_outputs(sessions)
        mel = eng.postnet(out['frames'], out['nsteps'])
        return mel, eng.target_lengths(out['stop'], out['nsteps'])

    def synthesize(self, text, out_dir, idx, step=None, seed=0, mu_bias=None):
        step = self.step if step is None else step
        mels, info = self.mels([text], seed=seed, mu_bias=mu_bias)
        os.makedirs(out_dir, exist_ok=True)
        pred_mel_path = os.path.join(out_dir, f'step-{step}-{idx}-mel-pred.npy')
        np.save(pred_mel_path, mels[0], allow_pickle=False)
        align = info['decode']['align'][0, :mels[0].shape[0] + 1].cpu().numpy()
        alignment_path = os.path.join(out_dir, f'step-{step}-{idx}-align.npy')
        np.save(alignment_path, align, allow_pickle=False)
        return pred_mel_path, alignment_path

    def gta_mels(self, texts, targets, seed=0, utterance_offset=0):
        """Ground-truth-aligned mels (wavernn_preprocess.py:72-120): pinyin strings + their recorded mels [T_b, 80] on the +-4
        scale -> list of np.float32 [T_b, 80] in [0, 1].  Per sentence: the target is clipped to +-4 (:79; r = 1, so no
        padding, :82), the decoder runs teacher-forced for exactly T_b steps (b200tts_taco_decode_gta), then the postnet; its
        mel is clipped to +-4, cropped to T_b and mapped with clip((m + 4) / 8, 0, 1) (:101-106).  Prenet dropout is Philox
        keyed by (seed, utterance_offset + b, step, unit): a sentence's mel does not depend on the batch it is decoded in."""
        if len(texts) != len(targets) or not texts:
            raise ValueError('need one target mel per text, and at least one text')
        tg = [np.clip(np.asarray(t, dtype=np.float32), -MAX_ABS_VALUE, MAX_ABS_VALUE) for t in targets]
        for t in tg:
            if t.ndim != 2 or t.shape[1] != 80 or t.shape[0] < 1:
                raise ValueError(f'target mels must be [T >= 1, 80], got {t.shape}')
        tlen = np.array([t.shape[0] for t in tg], dtype=np.int32)
        tpad = np.zeros((len(tg), int(tlen.max()), 80), dtype=np.float32)
        for b, t in enumerate(tg):
            tpad[b, :t.shape[0]] = t
        mem, lengths = self._encode(texts)
        eng = self.engine
        dec = eng.decode_gta(mem, lengths, tpad, tlen, seed=seed, utterance_offset=utterance_offset)
        mel_h = eng.postnet(dec['frames'], dec['nsteps']).cpu().numpy()
        return [unit_mel(mel_h[b, :tlen[b]]) for b in range(len(tg))]

    def synthesize_gta(self, text, mel_path, out_dir, idx, seed=0, utterance_offset=0):
        """wavernn_preprocess.py:72-120 `Synthesizer.synthesize(text, mel, out_dir, idx)`: Hanzi text (through get_pyin, :85),
        target mel `.npy` -> out_dir/mel-{idx}-pred.npy.  Returns (pred_mel_path, None): the alignment PNG is not drawn."""
        pyin, _ = get_pyin(text)
        mel = self.gta_mels([pyin], [np.load(mel_path)], seed=seed, utterance_offset=utterance_offset)[0]
        os.makedirs(out_dir, exist_ok=True)
        pred_mel_path = os.path.join(out_dir, f'mel-{idx}-pred.npy')
        np.save(pred_mel_path, mel, allow_pickle=False)
        return pred_mel_path, None
