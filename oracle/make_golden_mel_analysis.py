#!/usr/bin/env python
"""Golden vectors for mel analysis (feature extraction), produced by the reference's OWN functions -- needs a checkout of the
reference (environment variable B200TTS_REFERENCE, default /root/reference).

    python oracle/make_golden_mel_analysis.py   ->  tests/golden/mel_analysis_from_reference.npz

`_process_utterance_v1` is lifted out of tacotron/datasets/preprocessor.py's syntax tree, and `load_wav`, `trim_silence`,
`preemphasis`, `melspectrogram`, `_stft`, `_linear_to_mel`, `_build_mel_basis`, `_amp_to_db`, `_normalize`, `get_hop_size`
and `librosa_pad_lr` out of tacotron/datasets/audio.py's (as make_golden_griffin_lim.py does).  They are compiled unmodified
against numpy, scipy.signal and `LibrosaAnalysisStandIn` below: make_golden_griffin_lim.LibrosaStandIn (stft, filters.mel,
checked there against torch / torchaudio) extended with librosa 0.7.2's `core.load` (soundfile's scaling, no resampling),
`effects.trim` and what it calls (`feature.rms`, `util.frame`, `core.power_to_db`, `core.frames_to_samples`).  The rms framing
is checked against torch's `unfold` before use; the rest of `trim` (power_to_db with ref=np.max, the frame-to-sample
arithmetic) is a restatement of librosa 0.7.2's source that nothing here can run librosa itself against.  The hparams are the
keyword values of the reference's tacotron_hparams.py.

`_process_utterance_v1` runs into a temporary directory on a 16-bit wav written there; the generator reads back its
`audio-*.npy` and `mel-*.npy` files and checks them against the returned tuple.  Cases (every input is stored as int16):
  speech   the reference's demo/03-forward-griffin_lim.wav (88 550 samples at 22 050 Hz), through _process_utterance_v1
  padded   a 2 s slice of speech with 0.5 s of seeded -50 dBFS (rms) noise before and after, through _process_utterance_v1,
           so the trim cuts on both sides
  plain    audio.melspectrogram alone on speech's samples (no trim, pre-emphasis or rescale)
Stored per case: the input's name, the mel [T][80] float32; for the _process_utterance_v1 cases also the SHA-256 and length
of `out` (the training audio, T * 275 float32 samples; padded's `out` is stored in full as well), the trim bounds
[start, end) and the smallest distance, in dB, of any trim frame from the -25 dB threshold.  `oracle.mel_analysis_oracle.fixture_case` reads a case back.
Test infrastructure: nothing in the product imports this.
"""
import ast
import hashlib
import json
import os
import sys
import tempfile
import types

import numpy as np
from scipy import signal

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.make_golden_griffin_lim import REF, LibrosaStandIn, reference_hparams   # noqa: E402

AUDIO_SRC = os.path.join(REF, 'tacotron', 'datasets', 'audio.py')
PRE_SRC = os.path.join(REF, 'tacotron', 'datasets', 'preprocessor.py')
SPEECH = os.path.join(REF, 'demo', '03-forward-griffin_lim.wav')
OUT = os.path.join(ROOT, 'tests', 'golden', 'mel_analysis_from_reference.npz')
AUDIO_LIFTED = ('load_wav', 'trim_silence', 'preemphasis', 'melspectrogram', '_stft', '_linear_to_mel', '_build_mel_basis',
                '_amp_to_db', '_normalize', 'get_hop_size', 'librosa_pad_lr')
NOISE_SEED, NOISE_DBFS = 2024, -50.0
SLICE = (22050, 22050 + 2 * 22050)
STORE_OUT = ('padded',)        # speech's 355 KB `out` is pinned by its SHA-256 only, to keep the fixture small


class LibrosaAnalysisStandIn(LibrosaStandIn):
    """librosa 0.7.2 core.load / effects.trim / feature.rms / util.frame / core.power_to_db / core.frames_to_samples."""

    class util(LibrosaStandIn.util):
        @staticmethod
        def frame(y, frame_length=2048, hop_length=512):
            n_frames = 1 + int((len(y) - frame_length) / hop_length)
            return np.lib.stride_tricks.as_strided(y, shape=(frame_length, n_frames),
                                                   strides=(y.itemsize, hop_length * y.itemsize))

    class core:
        @staticmethod
        def to_mono(y):
            return np.mean(y, axis=0) if y.ndim > 1 else y

        @classmethod
        def load(cls, path, sr=22050, mono=True, offset=0.0, duration=None, dtype=np.float32, res_type='kaiser_best'):
            from scipy.io import wavfile
            assert offset == 0.0 and duration is None
            sr_native, x = wavfile.read(path)
            assert x.dtype == np.int16 and sr_native == sr, 'only 16-bit files at the target rate (no resampling)'
            y = (x.astype(dtype) / dtype(32768)).T                          # soundfile's int16 -> float scaling
            return (cls.to_mono(y) if mono else y), sr

        @staticmethod
        def power_to_db(S, ref=1.0, amin=1e-10, top_db=80.0):
            magnitude = np.asarray(S)
            ref_value = ref(magnitude) if callable(ref) else np.abs(ref)
            log_spec = 10.0 * np.log10(np.maximum(amin, magnitude))
            log_spec -= 10.0 * np.log10(np.maximum(amin, ref_value))
            if top_db is not None:
                log_spec = np.maximum(log_spec, log_spec.max() - top_db)
            return log_spec

        @staticmethod
        def frames_to_samples(frames, hop_length=512, n_fft=None):
            offset = int(n_fft // 2) if n_fft is not None else 0
            return (np.asanyarray(frames) * hop_length + offset).astype(int)

    class feature:
        @staticmethod
        def rms(y=None, frame_length=2048, hop_length=512, center=True, pad_mode='reflect'):
            if center:
                y = np.pad(y, int(frame_length // 2), mode=pad_mode)
            x = LibrosaAnalysisStandIn.util.frame(y, frame_length=frame_length, hop_length=hop_length)
            return np.sqrt(np.mean(np.abs(x) ** 2, axis=0, keepdims=True))

    class effects:
        @staticmethod
        def _signal_to_frame_nonsilent(y, frame_length=2048, hop_length=512, top_db=60, ref=np.max):
            L = LibrosaAnalysisStandIn
            mse = L.feature.rms(y=L.core.to_mono(y), frame_length=frame_length, hop_length=hop_length) ** 2
            return L.core.power_to_db(mse.squeeze(), ref=ref, top_db=None) > - top_db

        @classmethod
        def trim(cls, y, top_db=60, ref=np.max, frame_length=2048, hop_length=512):
            L = LibrosaAnalysisStandIn
            non_silent = cls._signal_to_frame_nonsilent(y, frame_length=frame_length, hop_length=hop_length, ref=ref, top_db=top_db)
            nonzero = np.flatnonzero(non_silent)
            if nonzero.size > 0:
                start = int(L.core.frames_to_samples(nonzero[0], hop_length))
                end = min(y.shape[-1], int(L.core.frames_to_samples(nonzero[-1] + 1, hop_length)))
            else:
                start, end = 0, 0
            full_index = [slice(None)] * y.ndim
            full_index[-1] = slice(start, end)
            return y[tuple(full_index)], np.asarray([start, end])


def check_stand_in():
    """The rms framing (reflect padding, frame count, mean square) against torch's unfold."""
    import torch
    L = LibrosaAnalysisStandIn
    rs = np.random.RandomState(1)
    for n in (2048, 2049, 5000, 88550):
        y = rs.standard_normal(n).astype(np.float32)
        r = L.feature.rms(y=y)
        assert r.dtype == np.float32 and r.shape == (1, 1 + n // 512)
        yt = torch.nn.functional.pad(torch.from_numpy(y.astype(np.float64))[None, None], (1024, 1024), mode='reflect')[0, 0]
        ms = (yt.unfold(0, 2048, 512) ** 2).mean(dim=1).numpy()
        assert ms.shape == (1 + n // 512,)
        np.testing.assert_allclose(r[0].astype(np.float64) ** 2, ms, rtol=1e-5)


def reference_functions():
    L = LibrosaAnalysisStandIn
    tree = ast.parse(open(AUDIO_SRC, encoding='utf-8').read(), AUDIO_SRC)
    keep = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in AUDIO_LIFTED]
    assert sorted(n.name for n in keep) == sorted(AUDIO_LIFTED)
    ns = {'np': np, 'signal': signal, 'librosa': L, '_mel_basis': None}
    exec(compile(ast.Module(body=keep, type_ignores=[]), AUDIO_SRC, 'exec'), ns)
    audio = types.SimpleNamespace(**{k: ns[k] for k in AUDIO_LIFTED})
    tree = ast.parse(open(PRE_SRC, encoding='utf-8').read(), PRE_SRC)
    keep = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == '_process_utterance_v1']
    assert len(keep) == 1
    pns = {'np': np, 'os': os, 'audio': audio}
    exec(compile(ast.Module(body=keep, type_ignores=[]), PRE_SRC, 'exec'), pns)
    return audio, pns['_process_utterance_v1']


def padded_pcm(speech):
    rs = np.random.RandomState(NOISE_SEED)
    amp = 32768 * 10 ** (NOISE_DBFS / 20)
    noise = [np.round(rs.standard_normal(22050 // 2) * amp).astype(np.int16) for _ in range(2)]
    return np.concatenate([noise[0], speech[SLICE[0]:SLICE[1]], noise[1]])


def main():
    from scipy.io import wavfile
    hp = reference_hparams()
    assert (hp.n_fft, hp.hop_size, hp.win_size, hp.trim_silence, hp.preemphasize, hp.rescale, hp.use_lws) == \
        (2048, 275, 1100, True, True, True, False)
    check_stand_in()
    audio, process = reference_functions()
    sr, speech = wavfile.read(SPEECH)
    assert sr == hp.sample_rate and speech.dtype == np.int16
    pcm = {'speech': speech, 'padded': padded_pcm(speech)}
    blob = {'hparams': np.array(json.dumps({k: v for k, v in sorted(vars(hp).items())
                                            if isinstance(v, (int, float, bool, str))})),
            'speech_pcm': pcm['speech'], 'padded_pcm': pcm['padded']}
    L = LibrosaAnalysisStandIn
    with tempfile.TemporaryDirectory() as tmp:
        for name in ('speech', 'padded'):
            path = os.path.join(tmp, name + '.wav')
            wavfile.write(path, hp.sample_rate, pcm[name])
            ret = process(tmp, name, path, 'text', 'pyin', hp)
            audio_file, mel_file, time_steps, mel_frames = ret[:4]
            out = np.load(os.path.join(tmp, audio_file))
            mel = np.load(os.path.join(tmp, mel_file))
            assert out.dtype == mel.dtype == np.float32 and mel.shape == (mel_frames, hp.num_mels)
            assert time_steps == len(out) == mel_frames * hp.hop_size
            wav = audio.load_wav(path, sr=hp.sample_rate)
            _, bounds = L.effects.trim(wav, top_db=hp.trim_top_db, frame_length=hp.trim_fft_size, hop_length=hp.trim_hop_size)
            db = L.core.power_to_db((L.feature.rms(y=wav, frame_length=hp.trim_fft_size, hop_length=hp.trim_hop_size) ** 2)
                                    .squeeze(), ref=np.max, top_db=None)
            blob.update({f'{name}_input': np.array(name), f'{name}_mode': np.array('preprocess'), f'{name}_mel': mel,
                         f'{name}_out_sha256': np.array(hashlib.sha256(out.tobytes()).hexdigest()),
                         f'{name}_out_len': np.array(len(out)), f'{name}_bounds': bounds.astype(np.int32),
                         f'{name}_margin_db': np.array(float(np.abs(db + hp.trim_top_db).min()))})
            if name in STORE_OUT:
                blob[f'{name}_out'] = out
            print(name, 'bounds', bounds, 'T', mel_frames, 'margin dB', float(blob[f'{name}_margin_db']))
    mel = audio.melspectrogram(pcm['speech'].astype(np.float32) / np.float32(32768), hp).astype(np.float32)
    blob.update({'plain_input': np.array('speech'), 'plain_mode': np.array('plain'), 'plain_mel': np.ascontiguousarray(mel.T)})
    np.savez_compressed(OUT, **blob)
    print(OUT, os.path.getsize(OUT), 'bytes', sorted(blob))


if __name__ == '__main__':
    main()
