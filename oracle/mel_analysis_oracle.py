"""float64 numpy restatement of the reference's feature extraction, `_process_utterance_v1` without the file I/O
(tacotron/datasets/preprocessor.py:52-121) and `audio.melspectrogram` (tacotron/datasets/audio.py:95-102), for the one
configuration the reference uses (tacotron_hparams.py):
  1. trim_silence (:71-77, librosa 0.7.2 effects.trim, top_db 25, frames of 2048 samples every 512): the mean square of each
     reflect-padded frame (feature.rms, center=True, squared), a frame is non-silent when
     10 log10(max(1e-10, ms)) - 10 log10(max(1e-10, max ms)) > -25; the kept samples are [first * 512, min(n, (last + 1) * 512))
  2. preemphasis (:47-50): p[n] = x[n] - 0.97 x[n-1], x[-1] = 0, float64
  3. rescale (preprocessor.py:70-72): wav / max|wav| * 0.999 in float32, p / max|p| * 0.999 in float64
  4. melspectrogram(p): |stft(p)|^2 (librosa, n_fft 2048, hop 275, periodic Hann of 1100 centred, center=True, constant
     padding; T = 1 + n // 275 frames), Slaney filterbank (fmin 95, fmax 7600), 20 log10(max(1e-5, .)) - 20, symmetric
     normalisation to +-4 with clipping (:250-254, :273-275, :283-295); stored [T][80]
  5. out: the rescaled trimmed wav zero-padded to T * 275 samples (preprocessor.py:100-111)
(WaveRNN's input is then clip((mel + 4) / 8, 0, 1), wavernn_preprocess.py:155-157.)
The STFT and filterbank are oracle.griffin_lim_oracle's.

Test infrastructure: the GPU path (tacotronv2_wavernn_chinese_b200/csrc/mel_analysis.cuh) is checked against this module, and
this module against the reference's own functions (tests/golden/mel_analysis_from_reference.npz).
"""
from __future__ import annotations

import numpy as np

from oracle import griffin_lim_oracle as go

HOP = go.HOP
TRIM_N, TRIM_HOP, TOP_DB = 2048, 512, 25.0
PREEMPH, RESCALE_MAX = 0.97, 0.999
MIN_DB, REF_DB, MAX_ABS = -100.0, 20.0, 4.0


def trim_power(wav, n=TRIM_N, hop=TRIM_HOP):
    """Mean square of every trim frame: 1 + len // hop frames of n reflect-padded samples."""
    y = np.pad(np.asarray(wav, np.float64), n // 2, mode='reflect')
    F = 1 + (len(y) - n) // hop
    idx = np.arange(n)[None, :] + hop * np.arange(F)[:, None]
    return np.mean(y[idx] ** 2, axis=1)


def trim_db(wav, **kw):
    """power_to_db(ms, ref=np.max) per trim frame."""
    ms = trim_power(wav, **kw)
    return 10 * np.log10(np.maximum(1e-10, ms)) - 10 * np.log10(np.maximum(1e-10, ms.max()))


def trim_bounds(wav, top_db=TOP_DB, n=TRIM_N, hop=TRIM_HOP):
    """(start, end) of the samples effects.trim keeps; (0, 0) when no frame is non-silent."""
    db = trim_db(wav, n=n, hop=hop)
    nz = np.flatnonzero(db > -top_db)
    if nz.size == 0:
        return 0, 0
    return int(nz[0] * hop), int(min(len(wav), (nz[-1] + 1) * hop))


def preemphasis(x, k=PREEMPH):
    x = np.asarray(x, np.float64)
    p = x.copy()
    p[1:] = x[1:] + (-k) * x[:-1]
    return p


def melspectrogram(y):
    """float64 signal -> normalised mel [80][1 + len // HOP] (float64)."""
    S = np.abs(go.stft(y)) ** 2
    mel = go.mel_basis() @ S
    db = 20 * np.log10(np.maximum(np.exp(MIN_DB / 20 * np.log(10)), mel)) - REF_DB
    return np.clip((2 * MAX_ABS) * ((db - MIN_DB) / (-MIN_DB)) - MAX_ABS, -MAX_ABS, MAX_ABS)


def process_utterance(wav):
    """Steps 1-5 of the module docstring for float32 samples: dict(mel [T][80] float64, out [T * HOP] float32,
    bounds (start, end))."""
    wav = np.asarray(wav, np.float32)
    s, e = trim_bounds(wav)
    w = wav[s:e]
    p = preemphasis(w)
    w = w / np.abs(w).max() * np.float32(RESCALE_MAX)
    p = p / np.abs(p).max() * RESCALE_MAX
    mel = melspectrogram(p).T
    T = mel.shape[0]
    out = np.zeros(T * HOP, np.float32)
    out[:len(w)] = w
    return dict(mel=mel, out=out, bounds=(s, e))


def fixture_case(path, name):
    """One case of tests/golden/mel_analysis_from_reference.npz (oracle/make_golden_mel_analysis.py): dict(wav float32 input,
    mode ('preprocess' or 'plain'), mel [T][80], and for preprocess cases out (None unless stored), out_sha256, out_len,
    bounds, margin_db)."""
    z = np.load(path)
    src = str(z[f'{name}_input'])
    wav = z[f'{src}_pcm'].astype(np.float32) / np.float32(32768)
    c = dict(wav=wav, mode=str(z[f'{name}_mode']), mel=z[f'{name}_mel'])
    if c['mode'] == 'preprocess':
        c.update(out=z[f'{name}_out'] if f'{name}_out' in z.files else None, out_sha256=str(z[f'{name}_out_sha256']),
                 out_len=int(z[f'{name}_out_len']), bounds=tuple(int(v) for v in z[f'{name}_bounds']),
                 margin_db=float(z[f'{name}_margin_db']))
    return c


def sha256(a):
    import hashlib
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float32).tobytes()).hexdigest()
