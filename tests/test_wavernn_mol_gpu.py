"""Mixture-of-logistics WaveRNN generation (voc_mode = 'MOL') on the H100 against the reference's own MOL runs and the oracle.

Bars: fc3 outputs within the RAW bar 5e-6 * max|out| + 1e-4; samples within that bar carried through the sampler formula
(oracle.wavernn_mol_oracle.sample_bar); mixture indices identical except where the oracle finds a near-tie."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import wavernn_mol_oracle as mo
from tacotronv2_wavernn_chinese_b200 import synth

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
F32 = np.float32
DIMS = dict(synth.DEFAULT_DIMS, mode='MOL')


def _engine(sd):
    from tacotronv2_wavernn_chinese_b200.engine import WaveRNNEngine
    return WaveRNNEngine(sd, DIMS, device=0)


@pytest.fixture(scope='module')
def eng():
    e = _engine(synth.synth_state_dict(21, mode='MOL'))
    yield e
    e.close()


def expected_kernel(rows, kernel):
    """MOL takes the push kernel up to 32 rows and the wide grid above (auto and grid), or the utterance kernel when asked."""
    if kernel == 'utterance':
        return 'wavernn_utt_kernel'
    return 'wavernn_push_kernel' if rows <= 32 else 'wavernn_grid_kernel'


def logit_bar(ref):
    return 5e-6 * float(np.abs(ref).max()) + 1e-4


def _gumbel_gap(p, u):
    """Gap between the two best mixture keys of each row."""
    g = np.sort((p[:, :10] - np.log(-np.log(u[:, :10]))).astype(F32), axis=1)
    return g[:, -1] - g[:, -2]


def check_replay(sd, mels, u, samples, logits, fold=None, steps=None):
    """The oracle teacher-forced on the GPU's own samples: every fc3 output within the fc3 bar, every mixture index the same
    (or a near-tie), every sample within the sample bar.  Returns (mixtures, oracle output)."""
    teacher = samples.astype(F32)
    if fold is None:
        out = mo.generate(sd, mels, u, teacher=teacher, keep_logits='all', max_steps=steps)
    else:
        out = mo.generate_batched(sd, mels, fold[0], fold[1], u, teacher=teacher, keep_logits='all')
    S = samples.shape[1]
    ref = np.stack([out['logits'][i] for i in range(S)])            # [S, B, 30]
    err = logit_bar(ref)
    assert np.abs(logits[:S] - ref).max() <= err
    for i in range(S):
        k_gpu = mo.mixture_index(logits[i], u[i])
        k_or = out['mix'][:, i]
        diff = k_gpu != k_or
        if diff.any():
            assert (_gumbel_gap(ref[i], u[i])[diff] <= 4 * err).all(), i
        bar = mo.sample_bar(ref[i], u[i], k_or, err)
        d = np.abs(samples[:, i].astype(np.float64) - out['samples'][:, i])
        assert (d[~diff] <= bar[~diff]).all(), (i, d.max())
    return out


def test_reference_fixture_teacher_forced_and_free(eng):
    z = dict(np.load(os.path.join(GOLDEN, 'wavernn_mol_synth_T24.npz')))
    sd = synth.synth_state_dict(int(z['weight_seed']), mode='MOL')
    B, T = int(z['B']), int(z['T'])
    S = T * 275
    mels = synth.synth_mels(int(z['mel_seed']), B, T)
    u = synth.synth_mol_uniform(int(z['u_seed']), S, B)
    ref = z['samples']
    teacher = np.concatenate([ref, np.zeros((B, 1), F32)], axis=1)
    out = eng.generate(mels, u=u, teacher=teacher, return_logits=True)
    assert eng.last_kernel() == 'wavernn_push_kernel'
    lg = out['logits'].cpu().numpy()
    for n, s in enumerate(z['probe']):
        assert np.abs(lg[int(s)] - z['logits'][n]).max() <= logit_bar(z['logits'][n])
    got = out['samples'].cpu().numpy()
    err = logit_bar(z['logits'])
    for i in range(S - 1):
        k = mo.mixture_index(lg[i], u[i])
        assert (np.abs(got[:, i].astype(np.float64) - ref[:, i]) <= mo.sample_bar(lg[i], u[i], k, err)).all(), i
    # free-running: the oracle, fed the GPU's own samples, reproduces every one of them, and the wave is their epilogue
    free = eng.generate(mels, u=u, return_logits=True)
    fs = free['samples'].cpu().numpy()
    check_replay(sd, mels, u, fs, free['logits'].cpu().numpy())
    np.testing.assert_allclose(free['wave'].cpu().numpy(), mo.finish_wave(fs, (T - 1) * 275, 275), rtol=0, atol=1e-12)


# 265 rows: the utterance kernel runs 4 rows per CTA, and its last CTA holds one
@pytest.mark.parametrize('kernel', ['auto', 'utterance', 'grid'])
@pytest.mark.parametrize('rows', [1, 3, 7, 8, 12, 16, 20, 32, 33, 64, 100, 128, 129, 200, 256, 265, 300])
def test_rows_teacher_forced(eng, rows, kernel):
    sd = synth.synth_state_dict(21, mode='MOL')
    T, steps = 2, 300
    mels = synth.synth_mels(400 + rows, rows, T)
    u = synth.synth_mol_uniform(500 + rows, steps, rows)
    teacher = np.clip(np.random.RandomState(rows).normal(0, 0.3, (rows, T * 275)), -1, 1).astype(F32)
    out = eng.generate(mels, u=u, teacher=teacher, return_logits=True, max_steps=steps, kernel=kernel)
    assert eng.last_kernel() == expected_kernel(rows, kernel)
    ref = mo.generate(sd, mels, u, teacher=teacher, keep_logits='all', max_steps=steps)
    lg = out['logits'].cpu().numpy()
    r = np.stack([ref['logits'][i] for i in range(steps)])
    assert np.abs(lg - r).max() <= logit_bar(r)
    got = out['samples'].cpu().numpy()[:, :steps]
    for i in range(steps):
        k = mo.mixture_index(lg[i], u[i])
        ok = k == ref['mix'][:, i]
        assert (_gumbel_gap(r[i], u[i])[~ok] <= 4 * logit_bar(r)).all(), i
        d = np.abs(got[ok, i].astype(np.float64) - ref['samples'][ok, i])
        assert (d <= mo.sample_bar(r[i], u[i], k, logit_bar(r))[ok]).all(), i


@pytest.mark.parametrize('kernel', ['auto', 'utterance'])
def test_philox_free_run_every_kernel(eng, kernel):
    """2 000 free-running Philox steps on 16 and 40 rows (push / wide grid, or the utterance kernel), replayed by the oracle."""
    sd = synth.synth_state_dict(21, mode='MOL')
    for rows in (16, 40):
        steps = 2000
        mels = synth.synth_mels(30 + rows, rows, 8)
        out = eng.generate(mels, seed=78, return_logits=True, max_steps=steps, kernel=kernel)
        assert eng.last_kernel() == expected_kernel(rows, kernel)
        u = eng.philox_mol_uniform(78, 0, rows, 0, steps).cpu().numpy()
        check_replay(sd, mels, u, out['samples'].cpu().numpy()[:, :steps], out['logits'].cpu().numpy(), steps=steps)


@pytest.mark.parametrize('steps', [1, 2, 9, 274, 276, 283])
def test_step_counts_inside_a_block(eng, steps):
    sd = synth.synth_state_dict(21, mode='MOL')
    mels = synth.synth_mels(7, 2, 2)
    u = synth.synth_mol_uniform(8, steps, 2)
    out = eng.generate(mels, u=u, return_logits=True, max_steps=steps)
    assert out['wave'] is None
    check_replay(sd, mels, u, out['samples'].cpu().numpy()[:, :steps], out['logits'].cpu().numpy(), steps=steps)


def test_philox_free_run_replayed(eng):
    sd = synth.synth_state_dict(21, mode='MOL')
    rows, steps = 16, 2000
    mels = synth.synth_mels(9, rows, 8)
    out = eng.generate(mels, seed=77, utterance_offset=5, return_logits=True, max_steps=steps)
    u = eng.philox_mol_uniform(77, 5, rows, 0, steps).cpu().numpy()
    assert u.min() >= F32(1e-5) and u.max() <= F32(1 - 1e-5) and abs(float(u.mean()) - 0.5) < 0.01
    check_replay(sd, mels, u, out['samples'].cpu().numpy()[:, :steps], out['logits'].cpu().numpy(), steps=steps)


@pytest.mark.parametrize('kernel', ['auto', 'utterance'])
@pytest.mark.parametrize('folds', [1, 8, 9, 16, 17, 32, 33, 64])
def test_fold_mode(eng, folds, kernel):
    sd = synth.synth_state_dict(21, mode='MOL')
    overlap = 275
    T, target = next((t, tg) for tg in (275, 550, 1100, 2750, 5500) for t in range(21, 200)
                     if eng.fold_geometry(t, tg, overlap)[0] == folds)
    mels = synth.synth_mels(11, 1, T)
    nf, L = eng.fold_geometry(T, target, overlap)
    u = synth.synth_mol_uniform(12, L, nf)
    out = eng.generate(mels, u=u, fold=(target, overlap), return_logits=True, kernel=kernel)
    assert eng.last_kernel() == expected_kernel(nf, kernel)
    s = out['samples'].cpu().numpy()
    assert s.shape == (nf, L)
    check_replay(sd, mels, u, s, out['logits'].cpu().numpy(), fold=(target, overlap))
    np.testing.assert_allclose(out['wave'].cpu().numpy()[0], mo.unfold_wave(s, target, overlap, (T - 1) * 275, 275),
                               rtol=0, atol=1e-12)


def test_whole_utterance_production_noise(eng):
    """80 frames (22 000 steps) at B = 1 with Philox noise: the oracle teacher-forced over every step."""
    sd = synth.synth_state_dict(21, mode='MOL')
    mels = synth.synth_mels(13, 1, 80)
    out = eng.generate(mels, seed=5, return_logits=True)
    eng.check()
    assert eng.last_kernel() == 'wavernn_push_kernel'
    s = out['samples'].cpu().numpy()
    u = eng.philox_mol_uniform(5, 0, 1, 0, 80 * 275).cpu().numpy()
    check_replay(sd, mels, u, s, out['logits'].cpu().numpy())
    np.testing.assert_allclose(out['wave'].cpu().numpy(), mo.finish_wave(s, 79 * 275, 275), rtol=0, atol=1e-12)
    assert np.isfinite(s).all() and np.abs(s).max() <= 1 and s.std() > 1e-3


def test_batch_invariance(eng):
    """On the push kernel a row's samples do not depend on the batch: alone (8-row variant) and in 12- and 32-row batches."""
    mels = synth.synth_mels(14, 32, 21)
    ids = list(range(100, 132))
    batch = eng.generate(mels, seed=9, utterance_ids=ids)['samples'].cpu().numpy()
    assert eng.last_kernel() == 'wavernn_push_kernel'
    mid = eng.generate(mels[:12], seed=9, utterance_ids=ids[:12])['samples'].cpu().numpy()
    solo = eng.generate(mels[5:6], seed=9, utterance_ids=[105])['samples'].cpu().numpy()
    np.testing.assert_array_equal(batch[5], solo[0])
    np.testing.assert_array_equal(mid[5], solo[0])
    from tacotronv2_wavernn_chinese_b200 import pipeline
    frames = [21, 30, 25]
    ms = [synth.synth_mels(20 + i, 1, f)[0].T for i, f in enumerate(frames)]
    waves = pipeline.vocode_ragged(eng, ms, ids=[3, 4, 5], seed=2)
    for i, m in enumerate(ms):
        w = eng.generate(m.T[None], seed=2, utterance_ids=[3 + i])['wave'].cpu().numpy()[0]
        np.testing.assert_array_equal(waves[i], w)


def test_clamp_coverage():
    sd = synth.synth_state_dict(22, mode='MOL', mol_clamp=True)
    e = _engine(sd)
    try:
        mels = synth.synth_mels(15, 4, 2)
        steps = 400
        u = synth.synth_mol_uniform(16, steps, 4)
        out = e.generate(mels, u=u, return_logits=True, max_steps=steps)
        s = out['samples'].cpu().numpy()[:, :steps]
        lg = out['logits'].cpu().numpy()
        k = np.stack([mo.mixture_index(lg[i], u[i]) for i in range(steps)])        # [S, B]
        floor_hits = int((np.take_along_axis(lg[:, :, 20:30], k[:, :, None], 2)[..., 0] < mo.LOG_SCALE_MIN).sum())
        edge_hits = int((np.abs(s) == 1).sum())
        assert floor_hits > 0 and edge_hits > 0, (floor_hits, edge_hits)
        check_replay(sd, mels, u, s, lg, steps=steps)
    finally:
        e.close()


def test_refusals(eng):
    from tacotronv2_wavernn_chinese_b200 import _lib, dist
    mels = synth.synth_mels(1, 1, 21)
    with pytest.raises(_lib.B200TTSError, match='RAW only'):
        eng.generate(mels, kernel='tc')
    with pytest.raises(ValueError, match='packed rows'):
        eng.generate(mels, pack=dict(rows=1, utt=np.zeros((1, 1), np.int32), start=np.zeros((1, 2), np.int32), steps=1))
    with pytest.raises(_lib.B200TTSError, match='generate_mol'):
        eng.generate_host(mels.astype(np.float32))
    with pytest.raises(ValueError, match='RAW only'):
        dist.generate_sharded(eng.generate, torch.as_tensor(mels), seed=0)


def _run(args, cwd):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
    return subprocess.run([sys.executable] + args, cwd=cwd, env=env, capture_output=True, text=True, timeout=600)


def test_wavernn_gen_cli_with_mol_hparams(tmp_path):
    src = open(os.path.join(ROOT, 'wavernn_hparams.py')).read().replace("voc_mode = 'RAW'", "voc_mode = 'MOL'")
    (tmp_path / 'mol_hparams.py').write_text(src)
    torch.save({k: torch.as_tensor(v) for k, v in synth.synth_state_dict(21, mode='MOL').items()}, tmp_path / 'mol.pyt')
    T = 24
    np.save(tmp_path / 'mel.npy', synth.synth_mels(17, 1, T)[0].T.copy())
    from scipy.io import wavfile
    for extra in ([], ['--batched', '-t', '2750', '-o', '275']):
        r = _run([os.path.join(ROOT, 'wavernn_gen.py'), '--file', str(tmp_path / 'mel.npy'), '--voc_weights', str(tmp_path / 'mol.pyt'),
                  '--hp_file', str(tmp_path / 'mol_hparams.py'), '--seed', '3'] + extra, str(tmp_path))
        assert r.returncode == 0, r.stdout + r.stderr
        tag = 'mel_gen_batched' if extra else 'mel_gen_NOT_BATCHED'
        wavs = [f for f in os.listdir(tmp_path / 'wavernn_inference_output') if f.startswith(tag)]
        assert len(wavs) == 1, os.listdir(tmp_path / 'wavernn_inference_output')
        sr, y = wavfile.read(tmp_path / 'wavernn_inference_output' / wavs[0])
        assert y.shape == ((T - 1) * 275,) and np.isfinite(y).all()
