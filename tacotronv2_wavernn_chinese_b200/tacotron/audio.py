"""The reference's 16-bit wav writer for Tacotron-side audio (`tacotron/datasets/audio.py`: dc_notch_filter :17-23,
save_wav :25-34), the function `tacotron_synthesize.py:112` saves its preview wav with.  Host-side numpy / scipy: the file is
written once per utterance, after the samples have left the GPU.

What the chain does to a float waveform, in order:
  1. speex's DC notch: the biquad  H(z) = r (1 - z^-1)^2 / (1 - 2 r z^-1 + d z^-2),  r = 0.982,  d = r^2 + 0.7 (1 - r)^2;
  2. peak-normalise to 0.999;
  3. soften the dynamics: sign(x) |x|^0.95 (the `f1` gain of :29 cancels in step 4);
  4. scale the peak to 32767 (never by more than 32767 / 0.01) and truncate towards zero to int16.

The preview wav comes either from WaveRNN or, like the reference's, from Griffin-Lim mel inversion (`inv_mel_spectrogram`,
audio.py:122-137, on the GPU through libb200tts); the writer is the same.

Griffin-Lim (what `inv_mel_spectrogram` computes, T frames -> 275 (T - 1) samples):
  1. denormalise the symmetric mel: D = (clip(mel, -4, 4) + 4) * 100 / 8 - 100                       (_denormalize :297-309)
  2. S = max(1e-10, pinv(M) . (10 ** ((D + 20) / 20)) ** (1/2)) ** 1.5, M the Slaney mel filterbank      (_mel_to_linear :256-260)
  3. 60 Griffin-Lim iterations from a uniform random phase, librosa 0.7.2 stft / istft                  (_griffin_lim :176-186)
  4. lfilter([1], [1, -0.97])                                                                           (inv_preemphasis :52-55)
The random phase is Philox(seed) keyed by (utterance, frame, bin) instead of numpy's global generator.

Mel analysis (the reference's feature extraction, on the GPU through libb200tts; `preprocess_wav` is `_process_utterance_v1`,
tacotron/datasets/preprocessor.py:52-121, without the file I/O):
  1. load_wav: 16-bit / 32-bit / 8-bit PCM or float32, averaged to mono, at hparams.sample_rate only      (audio.py:14-15)
  2. trim silence: frames of 2048 samples every 512 more than 25 dB below the loudest are cut at both ends  (:71-77)
  3. pre-emphasis lfilter([1, -0.97], [1]) in float64, then each signal / its peak * 0.999               (:47-50, preprocessor :70-72)
  4. melspectrogram: |stft|^2, Slaney filterbank, 20 log10(max(1e-5, .)) - 20, symmetric +-4 with clipping  (:95-102)
  5. the training audio: the rescaled trimmed wav zero-padded to T * 275 samples                          (preprocessor :100-111)
`melspectrogram(wav, hparams)` is step 4 alone, as in the reference.

`encode_mu_law` is the vocoder-training quantiser wavernn_preprocess.py applies to that training audio (audio.py:8-11).
"""
from __future__ import annotations

import functools

import numpy as np

NOTCH_RADIUS = 0.982          # audio.py:19


def dc_notch_coefficients(radius=NOTCH_RADIUS):
    """(b, a) of the notch biquad (audio.py:19-22)."""
    r = float(radius)
    b = r * np.array([1.0, -2.0, 1.0])
    a = np.array([1.0, -2.0 * r, r * r + 0.7 * (1.0 - r) ** 2])
    return b, a


def dc_notch_filter(wav):
    """Remove DC / sub-sonic drift; float64 out, same length (direct-form IIR with zero initial state like lfilter, :23)."""
    from scipy import signal
    b, a = dc_notch_coefficients()
    return signal.lfilter(b, a, np.asarray(wav, dtype=np.float64))


def to_int16(wav):
    """Steps 1-4 of the module docstring -> int16 samples (what save_wav writes)."""
    y = dc_notch_filter(wav)
    peak = np.abs(y).max() if y.size else 0.0
    if not peak > 0.0:                                    # silence: the reference would divide 0 by 0; write zeros
        return np.zeros(y.shape, dtype=np.int16)
    y = y / peak * 0.999
    gain = 0.5 * 32767 / max(0.01, float(np.abs(y).max()))          # :29 (kept so the roundings match the reference's)
    y = gain * (np.sign(y) * np.power(np.abs(y), 0.95))
    y = y * (32767 / max(0.01, float(np.abs(y).max())))
    return y.astype(np.int16)


def save_wav(wav, path, sr):
    """Write `wav` (float, any scale) as a 16-bit PCM file at `sr` Hz the way the reference's `audio.save_wav` does."""
    from scipy.io import wavfile
    wavfile.write(str(path), int(sr), to_int16(wav))


# ---- Griffin-Lim mel inversion ----------------------------------------------------------------------------------------
def _hz_to_mel(f):
    """librosa 0.7.2 hz_to_mel (htk=False): linear below 1 kHz, logarithmic above (Slaney's Auditory Toolbox)."""
    f = np.asanyarray(f, dtype=np.float64)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    logstep = np.log(6.4) / 27.0
    return np.where(f >= min_log_hz, min_log_hz / f_sp + np.log(np.maximum(f, min_log_hz) / min_log_hz) / logstep, f / f_sp)


def _mel_to_hz(m):
    m = np.asanyarray(m, dtype=np.float64)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, np.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)


def mel_filterbank(sr, n_fft, n_mels, fmin, fmax):
    """[n_mels][1 + n_fft/2] float64: librosa 0.7.2 filters.mel(sr, n_fft, n_mels, fmin, fmax) (Slaney scale, each triangle
    normalised to unit area, norm=1), the `_build_mel_basis` of audio.py:268-271."""
    fftfreqs = np.linspace(0, float(sr) / 2, int(1 + n_fft // 2), endpoint=True)
    mel_f = _mel_to_hz(np.linspace(_hz_to_mel(fmin), _hz_to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    w = np.maximum(0, np.minimum(-ramps[:n_mels] / fdiff[:n_mels, None], ramps[2:] / fdiff[1:, None]))
    return w * (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None]


@functools.lru_cache(maxsize=4)
def _inv_mel_basis(sr, n_fft, n_mels, fmin, fmax):
    b = np.linalg.pinv(mel_filterbank(sr, n_fft, n_mels, fmin, fmax))
    b.flags.writeable = False
    return b


def mel_basis(hparams):
    """The filterbank rounded to float32, [num_mels][1 + n_fft/2]: what `_linear_to_mel` (audio.py:250-254) multiplies by."""
    assert hparams.fmax <= hparams.sample_rate // 2                     # audio.py:269
    return mel_filterbank(hparams.sample_rate, hparams.n_fft, hparams.num_mels, float(hparams.fmin),
                          float(hparams.fmax)).astype(np.float32)


def inv_mel_basis(hparams):
    """np.linalg.pinv of the filterbank in float64, [1 + n_fft/2][num_mels] (`_inv_mel_basis` of audio.py:256-260)."""
    assert hparams.fmax <= hparams.sample_rate // 2                     # audio.py:269
    return _inv_mel_basis(hparams.sample_rate, hparams.n_fft, hparams.num_mels, float(hparams.fmin), float(hparams.fmax))


_engines = {}


def _engine(hparams, device=None, kind='griffin_lim'):
    """The cached GPU engine of `kind` ('griffin_lim' or 'mel_analysis') for these hparams on `device`."""
    import torch
    if kind == 'griffin_lim':
        from .griffin_lim import GriffinLimEngine as cls
    elif kind == 'mel_analysis':
        from .mel_analysis import MelAnalysisEngine as cls
    else:
        raise ValueError(f'unknown engine kind {kind!r}')
    dev = torch.cuda.current_device() if device is None and torch.cuda.is_available() else device
    key = (kind, dev, tuple(sorted((k, repr(v)) for k, v in hparams.values().items())))
    if key not in _engines:
        _engines[key] = cls(hparams, device=dev)
    return _engines[key]


def griffin_lim_batch(mels, hparams, seed=0, device=None):
    """Ragged list of mels [num_mels][T_i] (the layout inv_mel_spectrogram takes) -> list of float32 waves of
    hop * (T_i - 1) samples, in one GPU launch sequence.  Utterance i draws its initial phase as utterance i of Philox(seed)."""
    import torch
    mels = [np.asarray(m, dtype=np.float32) for m in mels]
    if not mels:
        return []
    frames = np.array([m.shape[1] for m in mels], dtype=np.int32)
    T = int(frames.max())
    batch = np.zeros((len(mels), T, hparams.num_mels), dtype=np.float32)
    for i, m in enumerate(mels):
        batch[i, :m.shape[1]] = m.T
    eng = _engine(hparams, device)
    wave = eng.run(batch, frames if (frames != T).any() else None, seed=seed)['wave']
    with torch.cuda.device(eng.device):
        wave = wave.cpu().numpy()
    return [wave[i, :hparams.hop_size * (int(n) - 1)].copy() for i, n in enumerate(frames)]


def inv_mel_spectrogram(mel_spectrogram, hparams, seed=0):
    """The reference's `audio.inv_mel_spectrogram(mel.T, hparams)` (audio.py:122-137): mel [num_mels][T], T >= 2 -> float32 wave
    of hop * (T - 1) samples, Griffin-Lim with hparams.griffin_lim_iters iterations on the GPU."""
    return griffin_lim_batch([mel_spectrogram], hparams, seed=seed)[0]


# ---- mel analysis (feature extraction) ---------------------------------------------------------------------------------
def load_wav(path, sr):
    """`audio.load_wav` (audio.py:14-15, librosa.core.load(path, sr=sr)[0]) without resampling: float32 mono samples.
    PCM is scaled as soundfile does (int16 / 32768, int32 / 2^31, (uint8 - 128) / 128), float32 is read as is, channels are
    averaged.  A file at another rate, a missing or an unreadable file raise ValueError."""
    from scipy.io import wavfile
    try:
        rate, x = wavfile.read(str(path))
    except (OSError, ValueError, EOFError) as e:
        raise ValueError(f'cannot read {path}: {e}') from e
    if rate != int(sr):
        raise ValueError(f'{path} is sampled at {rate} Hz, expected {int(sr)} Hz (resampling is not implemented)')
    if x.dtype == np.int16:
        y = x.astype(np.float32) / np.float32(32768)
    elif x.dtype == np.int32:
        y = x.astype(np.float32) / np.float32(2 ** 31)
    elif x.dtype == np.uint8:
        y = (x.astype(np.float32) - np.float32(128)) / np.float32(128)
    elif x.dtype == np.float32:
        y = x
    else:
        raise ValueError(f'{path}: unsupported sample format {x.dtype}')
    if y.ndim == 2:
        y = y.mean(axis=1, dtype=np.float32)              # librosa.to_mono
    return np.ascontiguousarray(y, dtype=np.float32)


def _analyze(wavs, hparams, flags, device=None, want_audio=False):
    import torch
    wavs = [np.ascontiguousarray(w, dtype=np.float32).reshape(-1) for w in wavs]
    if any(w.size == 0 for w in wavs):
        raise ValueError('empty signal')
    lengths = np.array([w.size for w in wavs], dtype=np.int64)
    batch = np.zeros((len(wavs), int(lengths.max())), dtype=np.float32)
    for i, w in enumerate(wavs):
        batch[i, :w.size] = w
    eng = _engine(hparams, device, kind='mel_analysis')
    out = eng.run(batch, lengths, flags=flags, want_audio=want_audio)
    with torch.cuda.device(eng.device):
        return {k: (v.cpu().numpy() if v is not None else None) for k, v in out.items()}


def melspectrogram_batch(wavs, hparams, device=None):
    """Ragged list of signals -> list of float32 mels [num_mels][1 + len // hop], one GPU launch sequence."""
    if len(wavs) == 0:
        return []
    r = _analyze(wavs, hparams, 0, device)
    return [np.ascontiguousarray(r['mel'][i, :int(n)].T) for i, n in enumerate(r['frames'])]


def melspectrogram(wav, hparams):
    """The reference's `audio.melspectrogram(wav, hparams)` (audio.py:95-102): [num_mels][T] float32, T = 1 + len // hop."""
    return melspectrogram_batch([wav], hparams)[0]


def preprocess_batch(wavs, hparams, device=None):
    """`_process_utterance_v1` (preprocessor.py:52-121) without the file I/O, for a ragged list of signals as load_wav returns
    them: trim silence, pre-emphasis, rescale, melspectrogram of the pre-emphasised signal.  Returns a list of
    (mel [T][num_mels] float32, out [T * hop] float32 training audio, (start, end) of the kept samples).  A signal the trim
    empties raises ValueError (the reference cannot process it either)."""
    from .mel_analysis import preprocess_flags, TRIM
    if len(wavs) == 0:
        return []
    flags = preprocess_flags(hparams)
    if flags & TRIM:
        short = [i for i, w in enumerate(wavs) if np.size(w) < hparams.trim_fft_size]
        if short:
            raise ValueError(f'signal {short[0]} has fewer than trim_fft_size = {hparams.trim_fft_size} samples')
    r = _analyze(wavs, hparams, flags, device, want_audio=True)
    res = []
    for i, n in enumerate(r['frames']):
        n = int(n)
        if n == 0:
            raise ValueError(f'signal {i} is silent: trimming leaves no samples')
        s, e = (int(v) for v in r['bounds'][i])
        res.append((np.ascontiguousarray(r['mel'][i, :n]), r['audio'][i, :n * hparams.hop_size].copy(), (s, e)))
    return res


def preprocess_wav(wav, hparams):
    """One signal through `preprocess_batch`: (mel [T][num_mels], out [T * hop], (start, end))."""
    return preprocess_batch([wav], hparams)[0]


def encode_mu_law(x, mu=2**10):
    """The reference's `audio.encode_mu_law` (tacotron/datasets/audio.py:8-11): floor((F(x) + 1) / 2 * (mu - 1) + 0.5), F the
    mu-law companding curve with mu - 1, as float values in [0, mu - 1].  The reference ran under numpy 1.x, where
    `... / np.log(1 + mu)` divides a float32 array by a float64 scalar that value-based casting demotes to float32; so for the
    float32 training audio every operation is float32, and the result is float32.  numpy 2 would promote that statement to
    float64, which rounds some samples to the neighbouring level (tests/test_tacotron_gta_pins.py counts them), so the
    arithmetic is spelled out here in the input's own float type (float64 for anything that is not float32)."""
    x = np.asarray(x)
    f = np.float32 if x.dtype == np.float32 else np.float64
    x = x.astype(f, copy=False)
    m = mu - 1
    fx = np.sign(x) * np.log(f(1) + f(m) * np.abs(x)) / f(np.log(1 + m))
    return np.floor((fx + f(1)) / f(2) * f(m) + f(0.5))
