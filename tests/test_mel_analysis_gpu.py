"""Mel analysis on the GPU (csrc/mel_analysis.cuh through tacotron/mel_analysis.py and tacotron/audio.py) against the
reference's own functions (tests/golden/mel_analysis_from_reference.npz) and the float64 oracle (oracle/mel_analysis_oracle.py).

Bars (tests/test_mel_analysis_cpu.py `GPU_BARS`, calibrated there on the CPU with a float32 FFT chain): trim bounds, T and the
training audio `out` exact; the mel within 6e-6 on bands within 60 dB of the frame's loudest band, 1e-4 everywhere and 8e-7
relative L2, against the fixture and against the oracle.  Measured against the fixture on an H100 80GB HBM3 (400 W limit):
speech 1.3e-6 / 5.7e-6 / 7.6e-8, padded 8.6e-7 / 1.4e-5 / 1.1e-7, plain 1.6e-6 / 1.8e-5 / 2.0e-7 -- what the float32 FFT
chain of the calibration makes.  The values are printed (run with -s) and recorded in DESIGN.md section 3.8.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, REF_CKPT_COPY, ROOT
from oracle import mel_analysis_oracle as mo
from test_mel_analysis_cpu import CASES, FIXTURE, GPU_BARS, mel_errors, oracle_case

pytestmark = pytest.mark.gpu

ALL = 7                                     # TRIM | PREEMPHASIS | RESCALE: _process_utterance_v1


@pytest.fixture(scope='module')
def hp():
    from tacotron_hparams import hparams
    return hparams


@pytest.fixture(scope='module')
def engine(hp):
    import torch
    assert torch.cuda.is_available()
    from tacotronv2_wavernn_chinese_b200.tacotron.mel_analysis import MelAnalysisEngine
    return MelAnalysisEngine(hp, device=0)


def _run(engine, wavs, flags):
    wavs = [np.asarray(w, np.float32) for w in wavs]
    L = max(len(w) for w in wavs)
    batch = np.zeros((len(wavs), L), np.float32)
    for i, w in enumerate(wavs):
        batch[i, :len(w)] = w
    r = engine.run(batch, [len(w) for w in wavs], flags=flags, want_audio=True)
    return {k: v.cpu().numpy() for k, v in r.items()}


def _within_bars(name, what, mel, ref):
    loud, mx, l2 = mel_errors(mel, ref)
    print(f'{name}: GPU vs {what}: loud bands {loud:.2e}, max-abs {mx:.2e}, rel L2 {l2:.2e}')
    assert loud <= GPU_BARS['loud'] and mx <= GPU_BARS['max'] and l2 <= GPU_BARS['rel_l2'], (what, loud, mx, l2)


@pytest.mark.parametrize('name', CASES)
def test_fixture_case(engine, name):
    c = mo.fixture_case(FIXTURE, name)
    flags = ALL if c['mode'] == 'preprocess' else 0
    r = _run(engine, [c['wav']], flags)
    T = int(r['frames'][0])
    assert T == c['mel'].shape[0]
    mel = r['mel'][0, :T]
    if flags:
        assert c['margin_db'] >= 1e-3                         # exact bounds are a fair demand
        assert tuple(int(v) for v in r['bounds'][0]) == c['bounds']
        out = r['audio'][0, :T * 275]
        assert mo.sha256(out) == c['out_sha256'] and len(out) == c['out_len']
        if c['out'] is not None:
            assert np.array_equal(out, c['out'])
    else:
        assert tuple(int(v) for v in r['bounds'][0]) == (0, len(c['wav']))
    assert not r['mel'][0, T:].any() and not r['audio'][0, T * 275:].any()
    _within_bars(name, 'reference', mel, c['mel'])
    _within_bars(name, 'oracle', mel, oracle_case(c)[0])


def test_public_functions(engine, hp):
    """audio.melspectrogram / preprocess_wav return what the engine computes, in the reference's layouts."""
    from tacotronv2_wavernn_chinese_b200.tacotron import audio
    sp, pa = (mo.fixture_case(FIXTURE, n) for n in ('speech', 'padded'))
    m = audio.melspectrogram(sp['wav'], hp)
    assert m.shape == (80, 323) and m.dtype == np.float32
    assert np.array_equal(m.T, _run(engine, [sp['wav']], 0)['mel'][0])
    mel, out, bounds = audio.preprocess_wav(pa['wav'], hp)
    assert bounds == pa['bounds'] and mel.shape == pa['mel'].shape and mo.sha256(out) == pa['out_sha256']
    res = audio.preprocess_batch([pa['wav'], sp['wav']], hp)
    assert np.array_equal(res[0][0], mel) and res[1][2] == sp['bounds']
    with pytest.raises(ValueError, match='silent'):
        audio.preprocess_batch([sp['wav'], np.zeros(5000, np.float32)], hp)
    with pytest.raises(ValueError, match='trim_fft_size'):
        audio.preprocess_wav(np.ones(1000, np.float32), hp)


def _seeded_signals():
    """Bursts of seeded noise between silences, 2 048 samples to 60 s."""
    rs = np.random.RandomState(17)
    sigs = []
    for n in (2048, 2049, 7777, 22050 * 5 + 3, 22050 * 60):
        env = np.zeros(n, np.float32)
        for _ in range(max(1, n // 20000)):
            a = rs.randint(0, n)
            env[a:a + rs.randint(500, 20000)] = rs.uniform(0.05, 0.8)
        sigs.append((rs.standard_normal(n).astype(np.float32) * (env + 1e-4)).astype(np.float32))
    return sigs


@pytest.mark.parametrize('flags', [ALL, 0])
def test_ragged_batch_is_bit_identical_to_standalone_runs(engine, flags):
    wavs = [mo.fixture_case(FIXTURE, n)['wav'] for n in CASES] + _seeded_signals() + [np.zeros(5000, np.float32)]
    r = _run(engine, wavs, flags)
    for i, w in enumerate(wavs):
        a = _run(engine, [w], flags)
        T = int(a['frames'][0])
        assert int(r['frames'][i]) == T and np.array_equal(r['bounds'][i], a['bounds'][0]), i
        assert np.array_equal(r['mel'][i, :T], a['mel'][0, :T]) and not r['mel'][i, T:].any(), i
        assert np.array_equal(r['audio'][i, :T * 275], a['audio'][0, :T * 275]) and not r['audio'][i, T * 275:].any(), i
        assert np.isfinite(r['mel'][i]).all()
        if flags:
            assert (T == 0) == (i == len(wavs) - 1), (i, T)        # the all-zero row, and only it, is empty
            if T:
                s, e = (int(v) for v in r['bounds'][i])
                assert (s, e) == mo.trim_bounds(w), i
                assert T == 1 + (e - s) // 275
        else:
            assert T == 1 + len(w) // 275


def test_launch_count_is_independent_of_batch(engine):
    wavs = _seeded_signals()[:4]
    counts = []
    for B in (1, 4):
        n0 = engine.launch_count
        _run(engine, wavs[:B], ALL)
        counts.append(engine.launch_count - n0)
    assert counts[0] == counts[1] == 4


def _ckpt():
    wav_ckpt = REF_CKPT_COPY if os.path.isfile(REF_CKPT_COPY) else '/root/reference/logs_wavernn/checkpoints/latest_weights.pyt'
    if not os.path.isfile(wav_ckpt):
        pytest.skip('shipped WaveRNN checkpoint not available on this box')
    return wav_ckpt


def _write_case(tmp_path, name):
    from scipy.io import wavfile
    z = np.load(FIXTURE)
    path = tmp_path / f'{name}.wav'
    wavfile.write(str(path), 22050, z[f'{name}_pcm'])
    return path


def test_cli_mel_loader_is_the_training_features(tmp_path):
    """wavernn_gen.load_mel on a .wav: exactly clip((mel + 4) / 8, 0, 1) of preprocess_wav, T = the trimmed frame count, and
    the target written is the loaded signal.  (In a subprocess: the WaveRNN hparams singleton is configured once per process.)"""
    paths = {name: str(_write_case(tmp_path, name)) for name in ('speech', 'padded')}
    frames = {name: mo.fixture_case(FIXTURE, name)['mel'].shape[0] for name in paths}
    code = f'''
import sys, numpy as np
sys.path.insert(0, {ROOT!r})
import wavernn_gen as g
from scipy.io import wavfile
from tacotron_hparams import hparams
from tacotronv2_wavernn_chinese_b200.tacotron import audio
from tacotronv2_wavernn_chinese_b200.wavernn.utils import hparams as hp
hp.configure({os.path.join(ROOT, "wavernn_hparams.py")!r})
for name, path in {paths!r}.items():
    target = path[:-4] + "_target.wav"
    mel = g.load_mel(path, target_path=target).numpy()[0]
    ref = np.clip((audio.preprocess_wav(audio.load_wav(path, 22050), hparams)[0] + 4) / 8, 0, 1).T
    assert mel.shape == ref.shape == (80, {frames!r}[name]), (name, mel.shape)
    assert np.array_equal(mel, ref), name
    sr, y = wavfile.read(target)
    assert sr == 22050 and np.array_equal(y, audio.load_wav(path, 22050)), name
print("OK")
'''
    r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and 'OK' in r.stdout, r.stdout + r.stderr


def test_cli_copy_synthesis(tmp_path):
    wav_ckpt = _ckpt()
    path = _write_case(tmp_path, 'speech')
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
    from scipy.io import wavfile
    T = mo.fixture_case(FIXTURE, 'speech')['mel'].shape[0]
    for extra, tag in (([], 'gen_NOT_BATCHED'), (['--batched', '-t', '5500', '-o', '550'], 'gen_batched_target5500_overlap550')):
        r = subprocess.run([sys.executable, os.path.join(ROOT, 'wavernn_gen.py'), '--file', str(path), '--voc_weights', wav_ckpt,
                            '--hp_file', os.path.join(ROOT, 'wavernn_hparams.py'), '--seed', '3'] + extra,
                           cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        out = tmp_path / 'wavernn_inference_output'
        sr, tgt = wavfile.read(out / '__speech__617k_steps_target.wav')
        assert sr == 22050 and tgt.dtype == np.float32 and tgt.shape == (88550,)
        sr, y = wavfile.read(out / f'speech_{tag}_step=617k.wav')
        assert sr == 22050 and y.dtype == np.float32 and y.shape == ((T - 1) * 275,) and np.abs(y).max() <= 1.0
        assert y.std() > 1e-3, tag                                    # it is audio, not silence
