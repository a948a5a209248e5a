"""Resampling without a GPU: the restatement of resampy 0.2.2 / librosa 0.7.2 (oracle/resample_oracle.py) against the
fixture (tests/golden/resample_from_reference.npz, oracle/make_golden_resample.py) and against independent checks, the
length rules of `resample_batch`, the ABI's argument checks, the kernel's code generation and `tacotron_preprocess.py`'s
checks before any GPU work.

The fixture pins the reference's glue around resampling (load_wav -> core.load -> core.resample -> _process_utterance_v1),
run on the same restatement; it cannot pin resampy itself.  So the restatement is also checked on its own:
  * every output against an exact (math.fsum) float64 sum of the same terms, with the terms found by testing every input
    sample rather than by resampy's loop bounds, within the bound of float32 accumulation (checks wing and edge indexing);
  * the table against the Kaiser-windowed sinc evaluated without the table;
  * pass-band tones keep their amplitude and a tone above the new Nyquist is removed.
"""
import ctypes
import hashlib
import math
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from oracle import resample_oracle as ro

FIXTURE = os.path.join(GOLDEN, 'resample_from_reference.npz')
CSRC = os.path.join(ROOT, 'tacotronv2_wavernn_chinese_b200', 'csrc')
RATES = (48000, 44100, 24000, 16000, 8000)
U32 = 2.0 ** -24                      # unit roundoff of float32


def noise_input(seed, n):
    from oracle.make_golden_resample import noise_input as f
    return f(seed, n)


def test_table_checksum_and_shape():
    from tacotronv2_wavernn_chinese_b200.tacotron import resample as R
    w = R.kaiser_best_window()
    assert w.dtype == np.float64 and w.shape == (64 * 512 + 1,)
    assert hashlib.sha256(np.ascontiguousarray(w).tobytes()).hexdigest() == str(np.load(FIXTURE)['table_sha256'])


def test_table_against_analytic_window():
    """table[k] = rolloff * sinc(rolloff * k / 512) * I0(beta sqrt(1 - (k / 32768)^2)) / I0(beta), evaluated from scratch."""
    from scipy.special import i0
    from tacotronv2_wavernn_chinese_b200.tacotron import resample as R
    w = R.kaiser_best_window()
    k = np.unique(np.concatenate([np.arange(0, 600), np.arange(0, 32769, 97), np.arange(32700, 32769)]))
    x = k / 512.0
    a = R.ROLLOFF * x
    sinc = np.where(a == 0, 1.0, np.sin(np.pi * a) / np.where(a == 0, 1.0, np.pi * a))
    kaiser = i0(R.KAISER_BETA * np.sqrt(np.maximum(0.0, 1 - (k / 32768.0) ** 2))) / i0(R.KAISER_BETA)
    ref = R.ROLLOFF * sinc * kaiser
    assert np.abs(w[k] - ref).max() <= 1e-14, np.abs(w[k] - ref).max()
    assert w[0] == R.ROLLOFF and abs(w[-1]) < 1e-7


@pytest.mark.parametrize('sr', RATES)
def test_loop_against_exact_sum(sr):
    """Each output equals the exact sum of its terms within the float32 accumulation bound (K terms: each partial sum is
    rounded once to float32 and once to float64), at the start, the middle and the last outputs."""
    rs = np.random.RandomState(sr % 1000)
    for n in (3000, 37, 2 if sr < 22050 else 3):
        x = (rs.standard_normal(n) * 0.3).astype(np.float32)
        y = ro.resampy_resample(x, sr, 22050)
        ts = sorted({0, 1, 2, len(y) // 2, len(y) - 2, len(y) - 1} & set(range(len(y))))
        for t in ts:
            terms, w, m = ro.terms(x, sr, 22050, t)
            exact = ro.exact_sum(terms)
            partial = np.cumsum(np.abs(terms))
            bound = (U32 + 2.0 ** -52) * float(partial.sum()) + 1e-30
            assert abs(float(y[t]) - exact) <= bound, (sr, n, t, float(y[t]), exact, bound)
            # the terms a wing holds: never past either end of the signal, never past the table
            assert m.min() >= 0 and m.max() < n


def test_wing_sizes():
    """48 kHz -> 22 050 Hz: index_step = int(0.459375 * 512) = 235, so about 139 taps per wing."""
    x = np.ones(20000, np.float32)
    _, w, m = ro.terms(x, 48000, 22050, 5000)
    assert 275 <= len(m) <= 280
    _, w, m = ro.terms(x, 8000, 22050, 5000)           # upsampling: 512 table entries per tap, 64 taps per wing
    assert 126 <= len(m) <= 128


@pytest.mark.parametrize('sr', (48000, 44100, 24000, 16000, 8000))
def test_passband_and_stopband(sr):
    """Tones up to 0.9 x the new Nyquist keep their amplitude: within 0.1 % up to 0.45 x, within 0.5 % (0.04 dB) at 0.9 x,
    where kaiser_best's roll-off (0.9476) has begun.  A tone above the new Nyquist is removed (> 80 dB) when downsampling."""
    n = sr                                              # 1 s
    tt = np.arange(n) / sr
    lo, hi = 500, int(min(sr, 22050) / 2 * 0.9)
    for f, tol in ((lo, 1e-3), (hi // 2, 1e-3), (hi, 5e-3)):
        y = ro.resample(np.sin(2 * np.pi * f * tt).astype(np.float32), sr, 22050)
        mid = y[2000:-2000].astype(np.float64)
        amp = np.sqrt(2 * np.mean(mid ** 2))
        assert abs(amp - 1) < tol, (sr, f, amp)
    if sr / 2 > 11025 * 1.2:                              # a tone between 1.1 x the new Nyquist and the old one
        f = int(11025 * 1.1 + (sr / 2 - 11025 * 1.1) / 2)
        y = ro.resample(np.sin(2 * np.pi * f * tt).astype(np.float32), sr, 22050)
        mid = y[2000:-2000].astype(np.float64)
        assert np.sqrt(2 * np.mean(mid ** 2)) < 1e-4, (sr, f)


def test_time_register_is_a_sequential_sum():
    """t * (1 / ratio) is not resampy's register: at 48 kHz -> 22 050 Hz they differ over most of 10 s."""
    inc = 1.0 / (22050 / 48000)
    n = 220500
    seq = np.cumsum(np.concatenate([[0.0], np.full(n - 1, inc)]))
    tau = 0.0
    for t in range(0, n):                                      # spot-check the numpy accumulate against a Python loop
        if t in (0, 1, 7, 1000, n - 1):
            assert seq[t] == tau
        tau += inc
    assert (seq != np.arange(n) * inc).sum() > n // 2


def test_oracle_reproduces_fixture_noise():
    d = np.load(FIXTURE)
    for name in d['noise_cases']:
        name = str(name)
        x = noise_input(int(d[f'{name}_seed']), int(d[f'{name}_len']))
        y = ro.resample(x, int(d[f'{name}_rate']), 22050)
        assert y.dtype == np.float32 and np.array_equal(y, d[f'{name}_y']), name


@pytest.mark.parametrize('name', ('speech48k', 'speech16k'))
def test_oracle_reproduces_fixture_speech(name):
    d = np.load(FIXTURE)
    x = d[f'{name}_pcm'].astype(np.float32) / np.float32(32768)
    y = ro.resample(x, int(d[f'{name}_rate']), 22050)
    assert len(y) == int(d[f'{name}_resampled_len'])
    assert hashlib.sha256(y.tobytes()).hexdigest() == str(d[f'{name}_resampled_sha256'])
    if f'{name}_resampled' in d.files:
        assert np.array_equal(y, d[f'{name}_resampled'])


def test_oracle_through_mel_oracle_matches_fixture():
    """The resampled speech through the float64 mel-analysis oracle meets the fixture's bounds and `out` exactly."""
    from oracle import mel_analysis_oracle as mo
    d = np.load(FIXTURE)
    for name in ('speech48k', 'speech16k'):
        x = d[f'{name}_pcm'].astype(np.float32) / np.float32(32768)
        r = mo.process_utterance(ro.resample(x, int(d[f'{name}_rate']), 22050))
        assert tuple(r['bounds']) == tuple(int(v) for v in d[f'{name}_bounds'])
        assert mo.sha256(r['out']) == str(d[f'{name}_out_sha256'])
        assert np.abs(r['mel'] - d[f'{name}_mel']).max() <= 1e-6


def test_resample_lengths_and_identity():
    from tacotronv2_wavernn_chinese_b200.tacotron import audio
    from tacotronv2_wavernn_chinese_b200.tacotron.resample import resampled_length
    for sr in RATES:
        for n in (1, 2, 3, 77, 320, 999, 44100, 96001):
            r = n * (22050 / sr)
            assert resampled_length(n, sr, 22050) == (int(r), int(math.ceil(r)))
            if int(r) >= 1 and n <= 3000:
                assert len(ro.resample(np.zeros(n, np.float32), sr, 22050)) == int(math.ceil(r))
    xs = [np.arange(5, dtype=np.float32), np.ones(3, np.float64)]
    out = audio.resample_batch(xs, 22050, 22050)              # equal rates: the inputs themselves, no GPU
    assert all(a is b for a, b in zip(out, xs))
    assert audio.resample_batch([], 48000, 22050) == []
    with pytest.raises(ValueError):
        audio.resample_batch(xs, 0, 22050)
    with pytest.raises(ValueError):
        ro.resampy_resample(np.zeros(2, np.float32), 48000, 22050)   # int(2 * 0.459) = 0


def test_rs_kernel_has_no_dfma(tmp_path):
    """resampy never fuses a multiply into an add; nvcc would, unless every operation is an explicit _rn intrinsic."""
    from tacotronv2_wavernn_chinese_b200 import build
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip('nvcc not found')
    src = tmp_path / 'rs.cu'
    src.write_text('#include "resample.cuh"\n')
    cubin = tmp_path / 'rs.cubin'
    res = subprocess.run([nvcc, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '--expt-relaxed-constexpr',
                          '-I', CSRC, '-cubin', '-o', str(cubin), str(src)], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    sass = subprocess.run([os.path.join(os.path.dirname(nvcc), 'cuobjdump'), '-sass', str(cubin)],
                          capture_output=True, text=True, check=True).stdout
    body = sass.split('Function : _ZN7b200tts9rs_kernelENS_6RsArgsE', 1)[1]
    assert 'DMUL' in body and 'DADD' in body
    assert 'DFMA' not in body


def test_resample_error_codes_without_a_device():
    """Argument checks of the resampling entry points come before any CUDA call."""
    from tacotronv2_wavernn_chinese_b200 import build, _lib as L
    build.build_lib()
    lib = L.load()
    EINVAL = -1
    h = ctypes.c_void_p()
    w = np.zeros(32769, np.float64)
    assert lib.b200tts_resample_create(ctypes.byref(h), 0, 48000, 22050, None, 32769, 512) == EINVAL and not h.value
    assert b'null argument' in lib.b200tts_last_error()
    assert lib.b200tts_resample_create(None, 0, 48000, 22050, w.ctypes.data, 32769, 512) == EINVAL
    for args, word in (((0, 22050, 32769, 512), b'sample rates'), ((48000, -1, 32769, 512), b'sample rates'),
                       ((22050, 22050, 32769, 512), b'nothing to resample'), ((48000, 22050, 1, 512), b'nwin'),
                       ((48000, 22050, 32769, 0), b'num_table'), ((48000, 50, 32769, 512), b'index_step'),
                       ((48000, 100, 32769, 512), b'shared memory')):
        sr0, sr1, nwin, nt = args
        assert lib.b200tts_resample_create(ctypes.byref(h), 0, sr0, sr1, w.ctypes.data, nwin, nt) == EINVAL, args
        assert word in lib.b200tts_last_error(), (args, lib.b200tts_last_error())
        assert not h.value
    x = ctypes.c_void_p(1)                                   # never dereferenced: every call below fails its argument checks
    fake = ctypes.c_void_p(8)
    assert lib.b200tts_resample(None, x, x, 1, 5000, x, x, None) == EINVAL
    assert b'null argument' in lib.b200tts_last_error()
    assert lib.b200tts_resample(fake, None, x, 1, 5000, x, x, None) == EINVAL
    assert lib.b200tts_resample(fake, x, x, 0, 5000, x, x, None) == EINVAL
    assert b'B must be' in lib.b200tts_last_error()
    assert lib.b200tts_resample(fake, x, x, 70000, 5000, x, x, None) == EINVAL
    assert lib.b200tts_resample(fake, x, x, 1, 0, x, x, None) == EINVAL
    assert b'L_max' in lib.b200tts_last_error()
    assert lib.b200tts_resample_launch_count(None) == -1
    lib.b200tts_resample_destroy(None)                       # no-op, must not crash
    import torch
    if not torch.cuda.is_available():
        assert lib.b200tts_resample_create(ctypes.byref(h), 0, 48000, 22050, w.ctypes.data, 32769, 512) == -2
        assert not h.value
        from tacotronv2_wavernn_chinese_b200.tacotron.resample import ResampleEngine
        with pytest.raises(RuntimeError):
            ResampleEngine()


def _run_cli(args):
    code = f'''
import sys
sys.path.insert(0, {ROOT!r})
import tacotron_preprocess as tp
tp.main({args!r})
'''
    return subprocess.run([sys.executable, '-c', code], capture_output=True, text=True,
                          env=dict(os.environ, CUDA_VISIBLE_DEVICES=''))


def test_preprocess_cli_rejects_malformed_labels_before_the_gpu(tmp_path):
    lab = tmp_path / 'labels.txt'
    lab.write_text('000001\t卡尔普#2陪外孙#1玩滑梯#4。\n\tka2 er2 pu3\n000002 no tab here\n\tjia2\n', encoding='utf-8')
    r = _run_cli(['--dataset_dir', str(tmp_path), '--labels', str(lab), '--out_dir', str(tmp_path / 'out')])
    assert r.returncode == 2 and 'line 3' in r.stderr, r.stdout + r.stderr
    assert not (tmp_path / 'out').exists()
    r = _run_cli(['--dataset_dir', str(tmp_path / 'nowhere')])
    assert r.returncode == 2 and 'not found' in r.stderr


def test_preprocess_cli_skips_missing_wavs(tmp_path):
    """Missing wavs are skipped with the reference's message; with none left there is no GPU work and train.txt is empty."""
    (tmp_path / 'ProsodyLabeling').mkdir()
    (tmp_path / 'Wave').mkdir()
    (tmp_path / 'ProsodyLabeling' / '000001-010000.txt').write_text(
        '000001\t卡尔普#2陪外孙#1玩滑梯#4。\n\tka2 er2 pu3 pei2 wai4 sun1 wan2 hua2 ti1\n'
        '000002\t假语村言#2别再#1拥抱我#4。\n\tjia3 yu3 cun1 yan2 bie2 zai4 yong1 bao4 wo3\n', encoding='utf-8')
    r = _run_cli(['--dataset_dir', str(tmp_path), '--out_dir', str(tmp_path / 'out')])
    assert r.returncode == 0, r.stdout + r.stderr
    for b in ('000001', '000002'):
        assert f'file {tmp_path / "Wave" / (b + ".wav")} present in csv metadata is not present in wav folder. skipping!' \
            in r.stdout
    assert (tmp_path / 'out' / 'train.txt').read_text() == ''


def test_parse_labels_keeps_every_first_line(tmp_path):
    sys.path.insert(0, ROOT)
    import tacotron_preprocess as tp
    lab = tmp_path / 'l.txt'
    lab.write_text('000001\tA#1B\n\tx\n000002\tC\n\ty\n000003\tD\n', encoding='utf-8')
    assert tp.parse_labels(str(lab)) == [('000001', 'A#1B'), ('000002', 'C'), ('000003', 'D')]
    assert tp.parse_labels(str(lab), limit=2) == [('000001', 'A#1B'), ('000002', 'C')]
