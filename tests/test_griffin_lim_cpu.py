"""Griffin-Lim mel inversion without a GPU: the float64 oracle (oracle/griffin_lim_oracle.py) against the reference's own
functions (tests/golden/griffin_lim_from_reference.npz, oracle/make_golden_griffin_lim.py), the product's filterbank / pinv and
the fixture generator's librosa stand-in against torch / torchaudio, the hparams, and the ABI's argument checks.

Measured oracle-vs-reference differences over the stored samples (relative L2 / max-abs over peak; the reference's chain is
partly float32: float32 filterbank, pinv and magnitudes, complex64 stft, float32 overlap-add):
    mel_graph (405 frames, 4 windows of 2048 samples)  0 iterations 3.5e-7 / 3.2e-7   1 iteration 4.6e-7 / 3.6e-7
                                                       60 iterations 1.2e-5 / 1.1e-5
    short (31 frames, every sample)                    0 iterations 4.3e-7 / 3.4e-7   1 iteration 5.3e-7 / 5.0e-7
                                                       60 iterations 4.4e-6 / 5.1e-6
(over the whole 405-frame wave the 60-iteration difference is 4.8e-6 / 1.1e-5: the edge windows are quiet, so a relative
measure over the windows weighs them more).  The bars below are 1e-6 up to one iteration and 3e-5 after 60: the float32 drift
grows with the iterations, as float32-vs-float64 runs of the same chain do.
"""
import ctypes
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from oracle import griffin_lim_oracle as go

FIXTURE = os.path.join(GOLDEN, 'griffin_lim_from_reference.npz')


def _rel(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b)), float(np.abs(a - b).max() / np.abs(b).max())


@pytest.mark.parametrize('name', ['short', 'mel_graph'])
def test_oracle_matches_reference_fixture(name):
    c = go.fixture_case(FIXTURE, name)
    S = go.magnitude(c['mel'])
    assert sorted(c['waves']) == [0, 1, 60]
    for it, (l2_bar, max_bar) in ((0, (1e-6, 1e-6)), (1, (1e-6, 1e-6)), (60, (3e-5, 3e-5))):
        ref = c['waves'][it]
        wav = go.inv_preemphasis(go.griffin_lim(S, c['u'], it)[0])
        assert wav.shape == (275 * (S.shape[1] - 1),) and ref.shape == c['idx'].shape
        l2, mx = _rel(wav[c['idx']], ref)
        assert l2 <= l2_bar and mx <= max_bar, (it, l2, mx)


def test_fixture_covers_the_wave_edges():
    """The long case stores windows at both ends of the signal (the trimmed frame edges) and two interior ones."""
    c = go.fixture_case(FIXTURE, 'mel_graph')
    L = 275 * (c['mel'].shape[1] - 1)
    idx = c['idx']
    assert idx[0] == 0 and idx[-1] == L - 1 and len(np.unique(idx)) == len(idx) == 4 * 2048
    assert np.array_equal(go.fixture_case(FIXTURE, 'short')['idx'], np.arange(275 * 30))


def test_oracle_step_is_one_iteration_and_converges():
    c = go.fixture_case(FIXTURE, 'short')
    S = go.magnitude(c['mel'])
    u = c['u']
    y3, u3, hist = go.griffin_lim(S, u, 3, trace=True)
    y, un = u, None
    for i in range(3):
        y, un = go.step(S, u if i == 0 else un)
        np.testing.assert_allclose(y, hist[i][0], rtol=0, atol=1e-12)
        np.testing.assert_allclose(np.exp(2j * np.pi * un), np.exp(2j * np.pi * hist[i + 1][1]), atol=1e-9)
    sc = [go.spectral_convergence(S, go.griffin_lim(S, u, n)[0]) for n in (0, 5, 30)]
    assert sc[0] > sc[1] > sc[2]
    # the signal is exactly hop (T - 1) samples and stft of it gives T frames again
    assert go.stft(y3).shape == S.shape


def test_product_filterbank_and_pinv_against_torchaudio():
    torchaudio = pytest.importorskip('torchaudio')
    from tacotron_hparams import hparams as hp
    from tacotronv2_wavernn_chinese_b200.tacotron import audio
    M = audio.mel_filterbank(hp.sample_rate, hp.n_fft, hp.num_mels, hp.fmin, hp.fmax)
    fb = torchaudio.functional.melscale_fbanks(hp.n_fft // 2 + 1, float(hp.fmin), float(hp.fmax), hp.num_mels, hp.sample_rate,
                                               norm='slaney', mel_scale='slaney').double().numpy().T
    assert M.shape == (80, 1025) and np.abs(M - fb).max() <= 1e-5 * fb.max()          # torchaudio builds it in float32
    np.testing.assert_allclose(M, go.mel_basis(), rtol=1e-12, atol=1e-15)
    P = audio.inv_mel_basis(hp)
    import torch
    np.testing.assert_allclose(P, torch.linalg.pinv(torch.from_numpy(M)).numpy(), atol=1e-10 * np.abs(P).max())
    assert P.dtype == np.float64 and P.shape == (1025, 80)
    np.testing.assert_allclose(M @ P, np.eye(80), atol=1e-9)          # full row rank: pinv is a right inverse


def test_fixture_generator_stand_in_against_torch():
    """The librosa 0.7.2 stand-in of oracle/make_golden_griffin_lim.py against torch.stft / torch.istft / torchaudio."""
    pytest.importorskip('torchaudio')
    from types import SimpleNamespace
    from oracle import make_golden_griffin_lim as mg
    mg.check_stand_in(SimpleNamespace(n_fft=2048, hop_size=275, win_size=1100, fmin=95, fmax=7600, num_mels=80, sample_rate=22050))


def test_oracle_stft_istft_against_torch():
    import torch
    rs = np.random.RandomState(3)
    T = 12
    y = rs.standard_normal(275 * (T - 1))
    w = torch.hann_window(1100, periodic=True, dtype=torch.float64)
    Xt = torch.stft(torch.from_numpy(y), 2048, 275, 1100, w, center=True, pad_mode='constant', return_complex=True).numpy()
    np.testing.assert_allclose(go.stft(y), Xt, atol=1e-10)
    np.testing.assert_allclose(go.istft(Xt), torch.istft(torch.from_numpy(Xt), 2048, 275, 1100, w, center=True).numpy(), atol=1e-10)


def test_hparams_match_reference():
    from tacotron_hparams import hparams as hp
    ref = json.loads(str(np.load(FIXTURE)['hparams']))
    for k in ('n_fft', 'hop_size', 'win_size', 'num_mels', 'sample_rate', 'fmin', 'fmax', 'min_level_db', 'ref_level_db',
              'magnitude_power', 'power', 'griffin_lim_iters', 'preemphasize', 'preemphasis', 'signal_normalization',
              'allow_clipping_in_normalization', 'symmetric_mels', 'max_abs_value'):
        assert getattr(hp, k) == ref[k], k


def test_cli_flags_are_exclusive(tmp_path):
    import subprocess
    import sys
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tacotron_synthesize.py'), '--text', 'a1', '--griffin_lim',
                        '--voc_weights', 'x.pyt'], cwd=str(tmp_path), capture_output=True, text=True,
                       env=dict(os.environ, PYTHONPATH=ROOT))
    assert r.returncode == 2 and '--griffin_lim' in r.stderr


def test_gl_error_codes_without_a_device():
    """Argument checks of the Griffin-Lim entry points come before any CUDA call."""
    from tacotronv2_wavernn_chinese_b200 import build, _lib as L
    build.build_lib()
    lib = L.load()
    EINVAL = -1
    h = ctypes.c_void_p()
    cfg = L.GlCfg(n_fft=2048, hop_size=275, win_size=1100, num_mels=80, max_abs_value=4, min_level_db=-100, ref_level_db=20,
                  magnitude_power=2, power=1.5, preemphasis=0.97)
    pinv = np.zeros((1025, 80), np.float32)
    assert lib.b200tts_gl_create(ctypes.byref(h), 0, ctypes.byref(cfg), None) == EINVAL and not h.value
    assert b'null argument' in lib.b200tts_last_error()
    assert lib.b200tts_gl_create(None, 0, ctypes.byref(cfg), pinv.ctypes.data) == EINVAL
    bad = L.GlCfg.from_buffer_copy(cfg)
    bad.n_fft = 1024
    assert lib.b200tts_gl_create(ctypes.byref(h), 0, ctypes.byref(bad), pinv.ctypes.data) == EINVAL
    assert b'n_fft' in lib.b200tts_last_error()
    bad = L.GlCfg.from_buffer_copy(cfg)
    bad.win_size = 4096
    assert lib.b200tts_gl_create(ctypes.byref(h), 0, ctypes.byref(bad), pinv.ctypes.data) == EINVAL
    assert b'win_size' in lib.b200tts_last_error()
    ph = L.GlPhase(mode=L.GL_PHASE_PHILOX)
    x = ctypes.c_void_p(1)                                   # never dereferenced: every call below fails its argument checks
    assert lib.b200tts_griffin_lim(None, x, None, 1, 10, ctypes.byref(ph), 60, x, None, None) == EINVAL
    assert b'null argument' in lib.b200tts_last_error()
    fake = ctypes.c_void_p(8)
    assert lib.b200tts_griffin_lim(fake, x, None, 1, 1, ctypes.byref(ph), 60, x, None, None) == EINVAL
    assert b'at least 2 frames' in lib.b200tts_last_error()
    assert lib.b200tts_griffin_lim(fake, x, None, 1, 10, ctypes.byref(ph), -1, x, None, None) == EINVAL
    assert b'n_iters' in lib.b200tts_last_error()
    ext = L.GlPhase(mode=L.GL_PHASE_EXT)
    assert lib.b200tts_griffin_lim(fake, x, None, 1, 10, ctypes.byref(ext), 60, x, None, None) == EINVAL
    assert b'd_u' in lib.b200tts_last_error()
    assert lib.b200tts_gl_philox_uniform(0, 1, 0, 1, 10, 1025, None, None) == EINVAL
    assert lib.b200tts_gl_launch_count(None) == -1
    lib.b200tts_gl_destroy(None)                             # no-op, must not crash
    import torch
    if not torch.cuda.is_available():
        assert lib.b200tts_gl_create(ctypes.byref(h), 0, ctypes.byref(cfg), pinv.ctypes.data) == -2 and not h.value
        from tacotron_hparams import hparams as hp
        from tacotronv2_wavernn_chinese_b200.tacotron.griffin_lim import GriffinLimEngine
        with pytest.raises(RuntimeError):
            GriffinLimEngine(hp)
