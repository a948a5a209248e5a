"""Mel analysis without a GPU: the float64 oracle (oracle/mel_analysis_oracle.py) against the reference's own functions
(tests/golden/mel_analysis_from_reference.npz, oracle/make_golden_mel_analysis.py), the fixture generator's librosa stand-in,
the hparams, `load_wav`, `wavernn_gen.py`'s `.wav` checks and the ABI's argument checks.

Measured oracle-vs-reference mel differences (normalised scale, +-4; max-abs over bands within 60 dB of the frame's loudest
band / max-abs everywhere / relative L2): speech 3.9e-7 / 3.9e-7 / 2.0e-8, padded 2.9e-7 / 3.7e-7 / 2.0e-8, plain
2.8e-7 / 2.9e-7 / 2.0e-8 (the reference stores its float64 stft as complex64 and runs the rest in float32).  Bounds, T and
`out` are exact.

Calibration of the GPU bars (`GPU_BARS`): the same chain with each frame rounded to float32 and a float32 FFT
(`torch.fft.rfft`), float32 filterbank and power spectrum -- the error any fp32 FFT implementation makes -- is, against the
fixture, speech 1.1e-6 / 7.4e-6 / 7.6e-8, padded 1.0e-6 / 9.9e-6 / 9.1e-8, plain 1.5e-6 / 2.3e-5 / 1.9e-7.  The bars are
about 4x the worst of these: 6e-6 on loud bands, 1e-4 everywhere (weak bands near the -100 dB floor are dominated by FFT
rounding), 8e-7 relative L2.  `test_fp32_fft_calibration` keeps these measurements true.
"""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from oracle import griffin_lim_oracle as go
from oracle import mel_analysis_oracle as mo

FIXTURE = os.path.join(GOLDEN, 'mel_analysis_from_reference.npz')
CASES = ('speech', 'padded', 'plain')
GPU_BARS = dict(loud=6e-6, max=1e-4, rel_l2=8e-7)
LOUD_DB = 60.0


def mel_errors(a, ref):
    """(max-abs over bands within 60 dB of the frame's loudest band, max-abs, relative L2) of mels [T][80] on the +-4 scale
    (8 / 100 per dB)."""
    a, ref = np.asarray(a, np.float64), np.asarray(ref, np.float64)
    d = np.abs(a - ref)
    loud = ref >= ref.max(axis=1, keepdims=True) - LOUD_DB * 8 / 100
    return float(d[loud].max()), float(d.max()), float(np.linalg.norm(a - ref) / np.linalg.norm(ref))


def oracle_case(c):
    """The oracle's (mel [T][80], out, bounds) for a fixture case, and the float64 signal its STFT receives."""
    if c['mode'] == 'plain':
        sig = c['wav'].astype(np.float64)
        return mo.melspectrogram(sig).T, None, None, sig
    r = mo.process_utterance(c['wav'])
    s, e = r['bounds']
    p = mo.preemphasis(c['wav'][s:e])
    return r['mel'], r['out'], r['bounds'], p / np.abs(p).max() * mo.RESCALE_MAX


def fp32_fft_mel(sig):
    """The chain with float32 frames, a float32 FFT (torch.fft.rfft), float32 power spectrum and filterbank: [T][80]."""
    import torch
    y = np.pad(np.asarray(sig, np.float64), go.N_FFT // 2)
    T = 1 + (len(y) - go.N_FFT) // go.HOP
    idx = np.arange(go.N_FFT)[None, :] + go.HOP * np.arange(T)[:, None]
    fr = (go.window()[None, :] * y[idx]).astype(np.float32)
    S = (torch.fft.rfft(torch.from_numpy(fr), dim=1).abs() ** 2).numpy()
    mel = (S @ go.mel_basis().astype(np.float32).T).astype(np.float64)
    db = 20 * np.log10(np.maximum(np.exp(mo.MIN_DB / 20 * np.log(10)), mel)) - mo.REF_DB
    return np.clip((2 * mo.MAX_ABS) * ((db - mo.MIN_DB) / (-mo.MIN_DB)) - mo.MAX_ABS, -mo.MAX_ABS, mo.MAX_ABS)


@pytest.mark.parametrize('name', CASES)
def test_oracle_matches_reference_fixture(name):
    c = mo.fixture_case(FIXTURE, name)
    mel, out, bounds, _ = oracle_case(c)
    assert mel.shape == c['mel'].shape
    if c['mode'] == 'preprocess':
        assert bounds == c['bounds']
        s, e = bounds
        assert mel.shape[0] == 1 + (e - s) // 275 and len(out) == c['out_len'] == 275 * mel.shape[0]
        assert mo.sha256(out) == c['out_sha256']
        if c['out'] is not None:
            assert np.array_equal(out, c['out'])
    else:
        assert mel.shape[0] == 1 + len(c['wav']) // 275
    loud, mx, l2 = mel_errors(mel, c['mel'])
    assert loud <= 1e-6 and mx <= 1e-6 and l2 <= 1e-7, (loud, mx, l2)


@pytest.mark.parametrize('name', CASES)
def test_fp32_fft_calibration(name):
    """The GPU bars are about 4x what an fp32 FFT chain makes against the fixture."""
    pytest.importorskip('torch')
    c = mo.fixture_case(FIXTURE, name)
    errs = mel_errors(fp32_fft_mel(oracle_case(c)[3]), c['mel'])
    for e, key in zip(errs, ('loud', 'max', 'rel_l2')):
        assert e <= GPU_BARS[key] / 3, (key, e)


def test_fixture_cases():
    """speech keeps every sample (323 frames); padded is cut on both sides; every trim frame of both is at least 1e-3 dB from
    the threshold, so exact bounds are a fair demand of any implementation."""
    sp, pa = (mo.fixture_case(FIXTURE, n) for n in ('speech', 'padded'))
    assert len(sp['wav']) == 88550 and sp['bounds'] == (0, 88550) and sp['mel'].shape == (323, 80)
    s, e = pa['bounds']
    assert 0 < s and e < len(pa['wav']) and len(pa['wav']) == 3 * 22050
    for c in (sp, pa):
        assert c['margin_db'] >= 1e-3
        db = mo.trim_db(c['wav'])
        assert np.abs(db + mo.TOP_DB).min() >= 1e-3          # the float64 oracle agrees on every frame's side
    assert mo.fixture_case(FIXTURE, 'plain')['mel'].shape == (323, 80)


def test_oracle_trim_against_stand_in():
    """The oracle's trim against the generator's librosa 0.7.2 stand-in on seeded signals with quiet ends."""
    from oracle import make_golden_mel_analysis as mg
    rs = np.random.RandomState(5)
    for n in (2048, 3001, 20000, 50000):
        x = (rs.standard_normal(n) * np.exp(-((np.arange(n) - n / 2) / (n / 6)) ** 2)).astype(np.float32)
        _, b = mg.LibrosaAnalysisStandIn.effects.trim(x, top_db=25, frame_length=2048, hop_length=512)
        assert tuple(int(v) for v in b) == mo.trim_bounds(x), n


def test_fixture_generator_stand_in_against_torch():
    pytest.importorskip('torch')
    from oracle import make_golden_mel_analysis as mg
    mg.check_stand_in()


def test_hparams_match_reference():
    from tacotron_hparams import hparams as hp
    ref = json.loads(str(np.load(FIXTURE)['hparams']))
    for k in ('rescale', 'rescaling_max', 'trim_silence', 'trim_fft_size', 'trim_hop_size', 'trim_top_db', 'preemphasize',
              'preemphasis', 'n_fft', 'hop_size', 'win_size', 'num_mels', 'sample_rate', 'fmin', 'fmax', 'min_level_db',
              'ref_level_db', 'magnitude_power', 'max_abs_value', 'symmetric_mels', 'signal_normalization',
              'allow_clipping_in_normalization'):
        assert getattr(hp, k) == ref[k], k


def test_product_forward_basis():
    from tacotron_hparams import hparams as hp
    from tacotronv2_wavernn_chinese_b200.tacotron import audio
    M = audio.mel_basis(hp)
    assert M.dtype == np.float32 and M.shape == (80, 1025)
    assert np.array_equal(M, go.mel_basis().astype(np.float32))


def _write(path, rate, data):
    from scipy.io import wavfile
    wavfile.write(str(path), rate, data)
    return str(path)


def test_load_wav(tmp_path):
    from tacotronv2_wavernn_chinese_b200.tacotron import audio
    rs = np.random.RandomState(0)
    pcm = rs.randint(-32768, 32767, size=3000).astype(np.int16)
    y = audio.load_wav(_write(tmp_path / 'a.wav', 22050, pcm), 22050)
    assert y.dtype == np.float32 and np.array_equal(y, pcm.astype(np.float32) / 32768)
    f = rs.uniform(-1, 1, 1000).astype(np.float32)
    assert np.array_equal(audio.load_wav(_write(tmp_path / 'f.wav', 22050, f), 22050), f)
    st = rs.randint(-32768, 32767, size=(500, 2)).astype(np.int16)
    y = audio.load_wav(_write(tmp_path / 's.wav', 22050, st), 22050)
    assert y.shape == (500,) and np.array_equal(y, (st.astype(np.float32) / 32768).mean(axis=1, dtype=np.float32))
    i32 = (pcm.astype(np.int32) << 16)
    assert np.array_equal(audio.load_wav(_write(tmp_path / 'i.wav', 22050, i32), 22050), pcm.astype(np.float32) / 32768)
    u8 = np.array([0, 128, 255], np.uint8)
    np.testing.assert_array_equal(audio.load_wav(_write(tmp_path / 'u.wav', 22050, u8), 22050), [-1, 0, 127 / 128])
    with pytest.raises(ValueError, match='16000'):
        audio.load_wav(_write(tmp_path / 'r.wav', 16000, pcm), 22050)
    with pytest.raises(ValueError):
        audio.load_wav(tmp_path / 'missing.wav', 22050)
    (tmp_path / 'junk.wav').write_bytes(b'not a wav file')
    with pytest.raises(ValueError):
        audio.load_wav(tmp_path / 'junk.wav', 22050)


def test_wavernn_gen_wav_input_fails_before_the_model(tmp_path):
    """A .wav at another rate is refused in load_mel, before any model call or GPU work; the hparams agree."""
    code = f'''
import sys, numpy as np
sys.path.insert(0, {ROOT!r})
import wavernn_gen as g
from scipy.io import wavfile
from tacotronv2_wavernn_chinese_b200.wavernn.utils import hparams as hp
hp.configure({os.path.join(ROOT, "wavernn_hparams.py")!r})
assert g.tacotron_hparams().hop_size == hp.hop_length
wavfile.write({str(tmp_path / "r.wav")!r}, 16000, np.zeros(5000, np.int16))
class M:
    def get_step(self): return 617000
    def generate(self, *a, **k): raise SystemExit("generate reached")
try:
    g.gen_from_file(M(), {str(tmp_path / "r.wav")!r}, {str(tmp_path)!r}, False, 11000, 550)
    raise SystemExit("accepted")
except ValueError as e:
    assert "16000" in str(e)
print("OK")
'''
    r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True)
    assert r.returncode == 0 and 'OK' in r.stdout, r.stdout + r.stderr


def test_mel_error_codes_without_a_device():
    """Argument checks of the mel-analysis entry points come before any CUDA call."""
    from tacotronv2_wavernn_chinese_b200 import build, _lib as L
    build.build_lib()
    lib = L.load()
    EINVAL = -1
    h = ctypes.c_void_p()
    cfg = L.MelCfg(n_fft=2048, hop_size=275, win_size=1100, num_mels=80, max_abs_value=4, min_level_db=-100, ref_level_db=20,
                   magnitude_power=2, preemphasis=0.97, rescaling_max=0.999, trim_fft_size=2048, trim_hop_size=512,
                   trim_top_db=25)
    basis = np.zeros((80, 1025), np.float32)
    assert lib.b200tts_mel_create(ctypes.byref(h), 0, ctypes.byref(cfg), None) == EINVAL and not h.value
    assert b'null argument' in lib.b200tts_last_error()
    assert lib.b200tts_mel_create(None, 0, ctypes.byref(cfg), basis.ctypes.data) == EINVAL
    for field, value, word in (('n_fft', 1024, b'n_fft'), ('win_size', 4096, b'win_size'), ('num_mels', 200, b'num_mels'),
                               ('min_level_db', 5, b'min_level_db'), ('trim_hop_size', 0, b'trim_hop_size'),
                               ('rescaling_max', 0, b'rescaling_max')):
        bad = L.MelCfg.from_buffer_copy(cfg)
        setattr(bad, field, value)
        assert lib.b200tts_mel_create(ctypes.byref(h), 0, ctypes.byref(bad), basis.ctypes.data) == EINVAL, field
        assert word in lib.b200tts_last_error(), field
    x = ctypes.c_void_p(1)                                   # never dereferenced: every call below fails its argument checks
    fake = ctypes.c_void_p(8)
    assert lib.b200tts_mel_analyze(None, x, x, 1, 5000, 7, x, x, None, None, None) == EINVAL
    assert b'null argument' in lib.b200tts_last_error()
    assert lib.b200tts_mel_analyze(fake, x, x, 0, 5000, 7, x, x, None, None, None) == EINVAL
    assert b'B must be' in lib.b200tts_last_error()
    assert lib.b200tts_mel_analyze(fake, x, x, 1, 0, 7, x, x, None, None, None) == EINVAL
    assert b'L_max' in lib.b200tts_last_error()
    assert lib.b200tts_mel_analyze(fake, x, x, 1, 5000, 8, x, x, None, None, None) == EINVAL
    assert b'unknown flags' in lib.b200tts_last_error()
    assert lib.b200tts_mel_launch_count(None) == -1
    lib.b200tts_mel_destroy(None)                            # no-op, must not crash
    import torch
    if not torch.cuda.is_available():
        assert lib.b200tts_mel_create(ctypes.byref(h), 0, ctypes.byref(cfg), basis.ctypes.data) == -2 and not h.value
        from tacotron_hparams import hparams as hp
        from tacotronv2_wavernn_chinese_b200.tacotron.mel_analysis import MelAnalysisEngine
        with pytest.raises(RuntimeError):
            MelAnalysisEngine(hp)
