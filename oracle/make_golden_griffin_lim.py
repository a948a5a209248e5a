#!/usr/bin/env python
"""Golden vectors for Griffin-Lim mel inversion, produced by the reference's OWN functions -- needs a checkout of the
reference (environment variable B200TTS_REFERENCE, default /root/reference).

    python oracle/make_golden_griffin_lim.py   ->  tests/golden/griffin_lim_from_reference.npz

`inv_mel_spectrogram`, `_griffin_lim`, `_stft`, `_istft`, `_mel_to_linear`, `_build_mel_basis`, `_db_to_amp`, `_denormalize`,
`inv_preemphasis` and `get_hop_size` are lifted out of tacotron/datasets/audio.py's syntax tree (as make_golden_audio.py does) and
compiled unmodified against numpy (plus the `np.complex` alias numpy 2 removed), scipy.signal and `LibrosaStandIn` below: a
restatement of librosa 0.7.2's `stft`, `istft` and `filters.mel`, dtypes included (complex64 spectra, float32 signals and
filters), so the generator needs no librosa install.  The stand-in is asserted against torch.stft / torch.istft and
torchaudio.functional.melscale_fbanks before it is used.  The hparams are the keyword values of the reference's
tacotron_hparams.py (its `HParams(...)` call, read by AST).

The reference draws its initial phase with `np.random.rand(1025, T)` (:181), so the global generator is seeded and the
fixture stores the seed; the tests regenerate u with `np.random.seed(seed); np.random.rand(1025, T)`.
Cases: `mel_graph` of tests/golden/taco_run_from_graph.npz (405 frames) and `short` = its frames 100..130, each with
griffin_lim_iters in {0, 1, 60}.  Stored per case: the frame range into that mel (the mel itself is not repeated), the seed,
the sample indices kept and the float32 wave at those indices -- every sample of `short`, and four windows of 2048 samples
of the 111 100-sample `mel_graph` wave (its first and last samples, where the trimmed frame edges are, and two interior
windows), which keeps the fixture small while every window still depends on the whole 60-iteration chain.
`oracle.griffin_lim_oracle.fixture_case` reads a case back.
Test infrastructure: nothing in the product imports this.
"""
import ast
import json
import os
import types

import numpy as np
from scipy import signal

REF = os.environ.get('B200TTS_REFERENCE', '/root/reference')
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(REF, 'tacotron', 'datasets', 'audio.py')
HP_SRC = os.path.join(REF, 'tacotron_hparams.py')
OUT = os.path.join(ROOT, 'tests', 'golden', 'griffin_lim_from_reference.npz')
LIFTED = ('inv_mel_spectrogram', '_griffin_lim', '_stft', '_istft', '_mel_to_linear', '_build_mel_basis', '_db_to_amp',
          '_denormalize', 'inv_preemphasis', 'get_hop_size')
ITERS = (0, 1, 60)
SEEDS = {'mel_graph': 1234, 'short': 77}


class LibrosaStandIn:
    """librosa 0.7.2 (core/spectrum.py stft / istft, filters.py mel / window_sumsquare), restricted to window='hann'."""

    class util:
        @staticmethod
        def tiny(x):
            return np.finfo(np.asarray(x).dtype).tiny

        @staticmethod
        def pad_center(data, size):
            lpad = int((size - len(data)) // 2)
            return np.pad(data, (lpad, int(size - len(data) - lpad)), mode='constant')

    @staticmethod
    def _hann(win_length):
        return signal.get_window('hann', win_length, fftbins=True)

    @classmethod
    def stft(cls, y, n_fft=2048, hop_length=None, win_length=None, window='hann', center=True, dtype=np.complex64,
             pad_mode='reflect'):
        assert window == 'hann' and np.issubdtype(y.dtype, np.floating) and np.isfinite(y).all()
        win_length = n_fft if win_length is None else win_length
        hop_length = int(win_length // 4) if hop_length is None else hop_length
        fft_window = cls.util.pad_center(cls._hann(win_length), n_fft).reshape((-1, 1))
        if center:
            y = np.pad(y, int(n_fft // 2), mode=pad_mode)
        n_frames = 1 + int((len(y) - n_fft) / hop_length)
        frames = np.lib.stride_tricks.as_strided(y, shape=(n_fft, n_frames), strides=(y.itemsize, hop_length * y.itemsize))
        out = np.empty((int(1 + n_fft // 2), n_frames), dtype=dtype, order='F')
        out[:] = np.fft.rfft(fft_window * frames, axis=0)
        return out

    @classmethod
    def window_sumsquare(cls, n_frames, hop_length, win_length, n_fft, dtype=np.float32):
        n = n_fft + hop_length * (n_frames - 1)
        x = np.zeros(n, dtype=dtype)
        win_sq = cls.util.pad_center(cls._hann(win_length) ** 2, n_fft)
        for i in range(n_frames):
            sample = i * hop_length
            x[sample:min(n, sample + n_fft)] += win_sq[:max(0, min(n_fft, n - sample))]
        return x

    @classmethod
    def istft(cls, stft_matrix, hop_length=None, win_length=None, window='hann', center=True, dtype=np.float32, length=None):
        assert window == 'hann' and length is None
        n_fft = 2 * (stft_matrix.shape[0] - 1)
        win_length = n_fft if win_length is None else win_length
        hop_length = int(win_length // 4) if hop_length is None else hop_length
        ifft_window = cls.util.pad_center(cls._hann(win_length), n_fft)[:, np.newaxis]
        n_frames = stft_matrix.shape[1]
        y = np.zeros(n_fft + hop_length * (n_frames - 1), dtype=dtype)
        ytmp = ifft_window * np.fft.irfft(stft_matrix, axis=0)
        for frame in range(n_frames):
            sample = frame * hop_length
            y[sample:sample + n_fft] += ytmp[:, frame]
        ifft_window_sum = cls.window_sumsquare(n_frames, hop_length, win_length, n_fft, dtype=dtype)
        nz = ifft_window_sum > cls.util.tiny(ifft_window_sum)
        y[nz] /= ifft_window_sum[nz]
        if center:
            y = y[int(n_fft // 2):-int(n_fft // 2)]
        return y

    class filters:
        @staticmethod
        def mel(sr, n_fft, n_mels=128, fmin=0.0, fmax=None, htk=False, norm=1, dtype=np.float32):
            assert not htk and norm == 1
            from oracle.griffin_lim_oracle import hz_to_mel, mel_to_hz
            fmax = float(sr) / 2 if fmax is None else fmax
            weights = np.zeros((int(n_mels), int(1 + n_fft // 2)), dtype=dtype)
            fftfreqs = np.linspace(0, float(sr) / 2, int(1 + n_fft // 2), endpoint=True)
            mel_f = mel_to_hz(np.linspace(hz_to_mel(fmin), hz_to_mel(fmax), n_mels + 2))
            fdiff = np.diff(mel_f)
            ramps = np.subtract.outer(mel_f, fftfreqs)
            for i in range(n_mels):
                lower = -ramps[i] / fdiff[i]
                upper = ramps[i + 2] / fdiff[i + 1]
                weights[i] = np.maximum(0, np.minimum(lower, upper))
            enorm = 2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels])
            weights *= enorm[:, np.newaxis]
            return weights


def check_stand_in(hp):
    """The stand-in against torch.stft / torch.istft and torchaudio's Slaney filterbank."""
    import torch
    L = LibrosaStandIn
    rs = np.random.RandomState(0)
    T = 37
    y = rs.standard_normal(hp.hop_size * (T - 1)).astype(np.float32)
    X = L.stft(y=y, n_fft=hp.n_fft, hop_length=hp.hop_size, win_length=hp.win_size, pad_mode='constant')
    w = torch.hann_window(hp.win_size, periodic=True, dtype=torch.float64)
    Xt = torch.stft(torch.from_numpy(y.astype(np.float64)), hp.n_fft, hp.hop_size, hp.win_size, w, center=True,
                    pad_mode='constant', return_complex=True).numpy()
    assert X.dtype == np.complex64 and X.shape == (hp.n_fft // 2 + 1, T)
    assert np.abs(X - Xt).max() <= 1e-5 * np.abs(Xt).max()
    Z = (rs.standard_normal(X.shape) + 1j * rs.standard_normal(X.shape))
    yi = L.istft(Z, hop_length=hp.hop_size, win_length=hp.win_size)
    yt = torch.istft(torch.from_numpy(Z), hp.n_fft, hp.hop_size, hp.win_size, w, center=True).numpy()
    assert yi.dtype == np.float32 and yi.shape == yt.shape == (hp.hop_size * (T - 1),)
    assert np.abs(yi - yt).max() <= 1e-5 * np.abs(yt).max()
    import torchaudio
    fb = torchaudio.functional.melscale_fbanks(hp.n_fft // 2 + 1, float(hp.fmin), float(hp.fmax), hp.num_mels, hp.sample_rate,
                                               norm='slaney', mel_scale='slaney').numpy().T
    M = L.filters.mel(hp.sample_rate, hp.n_fft, n_mels=hp.num_mels, fmin=hp.fmin, fmax=hp.fmax)
    assert M.dtype == np.float32 and np.abs(M - fb).max() <= 1e-5 * fb.max()


def reference_hparams():
    """Keyword values of `hparams = tf.contrib.training.HParams(...)` in the reference's tacotron_hparams.py."""
    tree = ast.parse(open(HP_SRC, encoding='utf-8').read(), HP_SRC)
    call = next(n.value for n in tree.body if isinstance(n, ast.Assign) and isinstance(n.value, ast.Call)
                and any(getattr(t, 'id', None) == 'hparams' for t in n.targets))
    out = {}
    for kw in call.keywords:
        try:
            out[kw.arg] = ast.literal_eval(kw.value)
        except ValueError:
            pass                                       # expressions that need the rest of the module (not used here)
    return types.SimpleNamespace(**out)


def reference_functions():
    tree = ast.parse(open(SRC, encoding='utf-8').read(), SRC)
    keep = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in LIFTED]
    assert sorted(n.name for n in keep) == sorted(LIFTED)
    np_shim = types.ModuleType('numpy')
    np_shim.__dict__.update(np.__dict__)
    np_shim.complex = complex                          # numpy < 1.24 alias of the builtin, used by _griffin_lim (:182)
    ns = {'np': np_shim, 'signal': signal, 'librosa': LibrosaStandIn, '_mel_basis': None, '_inv_mel_basis': None}
    exec(compile(ast.Module(body=keep, type_ignores=[]), SRC, 'exec'), ns)
    return ns


CASES = {'mel_graph': (0, 405), 'short': (100, 131)}      # frame ranges of taco_run_from_graph.npz:mel_graph
WINDOW = 2048


def sample_windows(L):
    """Indices of the stored samples of an L-sample wave: all of them for a short wave, else four windows."""
    if L <= 8 * WINDOW:
        return np.arange(L, dtype=np.int32)
    starts = [0, L // 3, (2 * L) // 3, L - WINDOW]
    return np.concatenate([np.arange(s, s + WINDOW) for s in starts]).astype(np.int32)


def main():
    hp = reference_hparams()
    assert (hp.n_fft, hp.hop_size, hp.win_size, hp.griffin_lim_iters, hp.use_lws) == (2048, 275, 1100, 60, False)
    check_stand_in(hp)
    ns = reference_functions()
    blob = {'hparams': np.array(json.dumps({k: v for k, v in sorted(vars(hp).items())
                                            if isinstance(v, (int, float, bool, str))}))}
    graph = np.load(os.path.join(ROOT, 'tests', 'golden', 'taco_run_from_graph.npz'))['mel_graph']    # [405][80] float32
    for name, (t0, t1) in CASES.items():
        mel = graph[t0:t1]
        idx = sample_windows(hp.hop_size * (mel.shape[0] - 1))
        blob[f'{name}_frames'] = np.array([t0, t1], dtype=np.int32)
        blob[f'{name}_seed'] = np.array(SEEDS[name])
        blob[f'{name}_idx'] = idx
        for it in ITERS:
            h = types.SimpleNamespace(**dict(vars(hp), griffin_lim_iters=it))
            np.random.seed(SEEDS[name])
            wav = ns['inv_mel_spectrogram'](mel.T, h)                      # mel.T [80][T], what tacotron_synthesize.py:111 passes
            assert wav.shape == (hp.hop_size * (mel.shape[0] - 1),)
            blob[f'{name}_wave_it{it}'] = wav[idx].astype(np.float32)
    np.savez_compressed(OUT, **blob)
    print(OUT, sorted(blob))


if __name__ == '__main__':
    import sys
    sys.path.insert(0, ROOT)
    main()
