"""Signal helpers the generation path touches, with the reference's public names
(`wavernn/utils/dsp.py`: label_2_float :8, float_2_label :12, save_wav :22, encode_mu_law :92, decode_mu_law :98).
The reference's `melspectrogram` here (:72) is not restated: the shipped checkpoint was trained on the Tacotron
preprocessor's features, whose GPU mel analysis lives in tacotronv2_wavernn_chinese_b200/tacotron/audio.py next to Griffin-Lim
mel inversion, the Tacotron side's preview vocoder.

Conventions (same as the reference): a `bits`-bit label l in [0, 2**bits - 1] maps to the float 2*l/(2**bits - 1) - 1 in
[-1, 1]; mu-law companding uses mu = n_classes - 1.
"""
from __future__ import annotations

import numpy as np

from . import hparams as hp


def _levels(bits):
    return 2 ** bits - 1.


def label_2_float(x, bits):
    """Integer label(s) -> float in [-1, 1]."""
    return 2 * x / _levels(bits) - 1.


def float_2_label(x, bits):
    """Float(s) in [-1, 1] -> (unrounded) label scale [0, 2**bits - 1]."""
    if np.abs(x).max() > 1.0:
        raise AssertionError('float_2_label expects values in [-1, 1]')
    return np.clip((x + 1.) * _levels(bits) / 2, 0, _levels(bits))


def encode_mu_law(x, mu):
    """Waveform in [-1, 1] -> mu-law label (float array of integers) for `mu` classes."""
    m = mu - 1
    companded = np.sign(x) * np.log1p(m * np.abs(x)) / np.log1p(m)
    return np.floor((companded + 1) / 2 * m + 0.5)


def decode_mu_law(y, mu, from_labels=True):
    """Inverse companding.  `from_labels=True`: y holds integer labels of a log2(mu)-bit signal; False: y already in [-1, 1]
    (what WaveRNN.generate passes, fatchord_version.py:248)."""
    if from_labels:
        y = label_2_float(y, np.log2(mu))
    m = mu - 1
    return np.sign(y) / m * (np.power(1 + m, np.abs(y)) - 1)


def save_wav(x, path, sample_rate=None):
    """float32 PCM wav at hp.sample_rate.  (The reference calls librosa.output.write_wav, which current librosa no longer
    has; scipy writes the same float32 samples.)"""
    from scipy.io import wavfile
    rate = int(sample_rate if sample_rate is not None else hp.sample_rate)
    wavfile.write(str(path), rate, np.asarray(x, dtype=np.float32))
