"""float64 numpy restatement of the reference's Griffin-Lim mel inversion, `audio.inv_mel_spectrogram(mel.T, hparams)`
(tacotron_synthesize.py:110-112 -> tacotron/datasets/audio.py:122-137 inv_mel_spectrogram, :176-186 _griffin_lim,
:203-210 _stft / _istft, :256-260 _mel_to_linear, :268-271 _build_mel_basis, :277-278 _db_to_amp,
:297-309 _denormalize, :52-55 inv_preemphasis) with
librosa 0.7.2's stft / istft / filters.mel written out for the one configuration the reference uses (n_fft 2048, hop 275,
periodic Hann of 1100 samples centred in the frame, center=True, constant padding).

The chain, for a symmetric [-4, 4] mel[80][T]:
  1. D = (clip(mel, -4, 4) + 4) * 100 / 8 - 100                                       _denormalize     :297-309
  2. S = max(1e-10, pinv(M) . (10 ** ((D + 20) / 20)) ** (1/2)) ** 1.5                 _mel_to_linear   :256-260, :134, :277-278
  3. y = istft(S e^{2 pi i u}),  u ~ U[0,1);  60 x  y = istft(S e^{i angle(stft(y))})   _griffin_lim     :176-186
  4. lfilter([1], [1, -0.97], y)                                                       inv_preemphasis  :52-55
T frames give 275 (T - 1) samples; each istft trims the 1024-sample tails, so the next stft sees zeros there.

Test infrastructure: the GPU path (tacotronv2_wavernn_chinese_b200/csrc/griffin_lim.cuh) is checked against this module, and
this module against the reference's own functions (tests/golden/griffin_lim_from_reference.npz).
"""
from __future__ import annotations

import numpy as np

N_FFT, HOP, WIN = 2048, 275, 1100
N_BINS = N_FFT // 2 + 1


# ---- librosa 0.7.2 filters.mel (norm=1 = Slaney area normalisation, Slaney mel scale) -------------------------------------
def hz_to_mel(f):
    f = np.asanyarray(f, dtype=np.float64)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, np.log(6.4) / 27.0
    return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-300) / min_log_hz) / logstep, f / f_sp)


def mel_to_hz(m):
    m = np.asanyarray(m, dtype=np.float64)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, np.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)


def mel_basis(sr=22050, n_fft=N_FFT, n_mels=80, fmin=95.0, fmax=7600.0):
    """[n_mels][1 + n_fft/2] float64 triangular filters, Slaney-normalised (librosa 0.7.2 filters.mel(sr, n_fft, n_mels, fmin, fmax))."""
    fftfreqs = np.linspace(0, float(sr) / 2, int(1 + n_fft // 2), endpoint=True)
    mel_f = mel_to_hz(np.linspace(hz_to_mel(fmin), hz_to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    lower = -ramps[:n_mels] / fdiff[:n_mels, None]
    upper = ramps[2:] / fdiff[1:, None]
    w = np.maximum(0, np.minimum(lower, upper))
    return w * (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None]


def inv_mel_basis(**kw):
    """np.linalg.pinv of the filterbank in float64: [1025][80]."""
    return np.linalg.pinv(mel_basis(**kw))


# ---- stft / istft (librosa 0.7.2 with the reference's arguments, :203-210) -----------------------------------------------
def window():
    """Periodic Hann of WIN samples (scipy get_window('hann', 1100, fftbins=True)) zero-padded to N_FFT, centred (pad_center)."""
    w = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(WIN) / WIN)
    lpad = (N_FFT - WIN) // 2
    return np.pad(w, (lpad, N_FFT - WIN - lpad))


def stft(y):
    """[1025][T] for a signal of HOP * (T - 1) samples: zero pad N_FFT/2 on both sides, frame every HOP, window, rfft."""
    w = window()
    yp = np.pad(np.asarray(y, np.float64), N_FFT // 2)
    T = 1 + (len(yp) - N_FFT) // HOP
    idx = np.arange(N_FFT)[None, :] + HOP * np.arange(T)[:, None]
    return np.fft.rfft(w[None, :] * yp[idx], axis=1).T


def envelope(T):
    """Window sum-square of T frames (librosa filters.window_sumsquare), untrimmed: N_FFT + HOP (T - 1) samples."""
    w2 = window() ** 2
    env = np.zeros(N_FFT + HOP * (T - 1))
    for t in range(T):
        env[t * HOP:t * HOP + N_FFT] += w2
    return env


def istft(X):
    """[1025][T] -> HOP (T - 1) samples: irfft, window, overlap-add, divide by the window sum-square where it exceeds
    tiny(float32), trim N_FFT/2 from both ends."""
    T = X.shape[1]
    frames = window()[None, :] * np.fft.irfft(X.T, n=N_FFT, axis=1)
    y = np.zeros(N_FFT + HOP * (T - 1))
    for t in range(T):
        y[t * HOP:t * HOP + N_FFT] += frames[t]
    env = envelope(T)
    nz = env > np.finfo(np.float32).tiny
    y[nz] /= env[nz]
    return y[N_FFT // 2:-(N_FFT // 2)]


# ---- the chain ------------------------------------------------------------------------------------------------------
def magnitude(mel, inv_basis=None, max_abs=4.0, min_level_db=-100.0, ref_level_db=20.0, magnitude_power=2.0, power=1.5):
    """mel [80][T] (symmetric, +-max_abs) -> S ** power [1025][T] (steps 1-2 of the module docstring)."""
    mel = np.asarray(mel, np.float64)
    D = (np.clip(mel, -max_abs, max_abs) + max_abs) * -min_level_db / (2 * max_abs) + min_level_db
    A = np.power(10.0, (D + ref_level_db) * 0.05) ** (1 / magnitude_power)
    B = inv_mel_basis() if inv_basis is None else inv_basis
    return np.maximum(1e-10, B @ A) ** power


def phasor(u):
    return np.exp(2j * np.pi * np.asarray(u, np.float64))


def phase_of(X):
    """angle(X) / 2 pi mod 1 -- the `u` form of a phase (np.angle(0) = 0)."""
    return np.mod(np.angle(X) / (2 * np.pi), 1.0)


def step(S, u):
    """One teacher-forced iteration: (S, u) -> (y, u_next), y = istft(S e^{2 pi i u}), u_next = phase of stft(y)."""
    y = istft(S * phasor(u))
    return y, phase_of(stft(y))


def griffin_lim(S, u, n_iters=60, trace=False):
    """_griffin_lim (:176-186) from the initial phase u [1025][T]: returns (y, u_last) where u_last is the phase the final istft
    used (u itself when n_iters = 0).  trace=True also returns the list of (y_i, u_i) for i = 0..n_iters."""
    y = istft(S * phasor(u))
    hist = [(y, np.asarray(u, np.float64))]
    for _ in range(n_iters):
        u = phase_of(stft(y))
        y = istft(S * phasor(u))
        if trace:
            hist.append((y, u))
    return (y, u, hist) if trace else (y, u)


def inv_preemphasis(y, k=0.97):
    from scipy import signal
    return signal.lfilter([1], [1, -k], y)


def inv_mel_spectrogram(mel, u, n_iters=60):
    """mel [80][T] + initial phase u [1025][T] -> float64 wave of HOP (T - 1) samples (the whole chain)."""
    y, _ = griffin_lim(magnitude(mel), u, n_iters)
    return inv_preemphasis(y)


def fixture_case(path, name):
    """One case of tests/golden/griffin_lim_from_reference.npz (oracle/make_golden_griffin_lim.py): dict(mel [80][T],
    u [1025][T] = the reference's initial phase (np.random.rand after seeding the global generator, audio.py:181),
    idx = indices of the stored samples, waves = {iterations: reference wave at idx})."""
    import os
    z = np.load(path)
    t0, t1 = (int(v) for v in z[f'{name}_frames'])
    graph = np.load(os.path.join(os.path.dirname(path), 'taco_run_from_graph.npz'))['mel_graph']
    mel = np.ascontiguousarray(graph[t0:t1].T)
    state = np.random.get_state()
    np.random.seed(int(z[f'{name}_seed']))
    u = np.random.rand(N_BINS, mel.shape[1])
    np.random.set_state(state)
    waves = {int(k.rsplit('_it', 1)[1]): z[k] for k in z.files if k.startswith(f'{name}_wave_it')}
    return dict(mel=mel, u=u, idx=z[f'{name}_idx'], waves=waves)


def spectral_convergence(S, y):
    return float(np.linalg.norm(np.abs(stft(y)) - S) / np.linalg.norm(S))
