"""Griffin-Lim on the GPU (csrc/griffin_lim.cuh) against the float64 oracle at every frame count of the edge sweep
(tests/audio_edge_cases.py): T = 2 to 33 around the 16-frame magnitude tiles and the lengths where the signal is shorter than
the window (T <= 4) or the FFT (T <= 8), T = 1025 (L = 1024 * 275, every finish-scan chunk full) and T = 2000 (Tacotron's
max_iters), the floor and ceiling mels and one beyond +-4.

- n_iters = 0 with an external phase u: magnitude stage, inverse FFT, overlap-add and finish scan against
  inv_preemphasis(istft(S e^{2 pi i u})).
- Teacher forced through one iteration: the returned phase and the wave against the oracle's step.
- 60 free-running iterations from the Philox phase at T = 2, 17, 400 and 2000, with the reference-fixture bars, or 4x what a
  float32 torch chain makes from the same phase where that is more.
- A ragged batch of every mel, padding frames set to 3.0: each row against the oracle and bit-equal to its stand-alone run.
Bars (tests/audio_edge_cases.py): wave relative L2 and S-weighted phasor error <= 5e-6, and the worst error over the first and
last 2 048 samples <= 5e-6 of the wave's peak.  Run with -s to see the errors (recorded in DESIGN.md section 3.7).
"""
import numpy as np
import pytest

import audio_edge_cases as ae
from oracle import griffin_lim_oracle as go

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def engine():
    import torch
    assert torch.cuda.is_available()
    from tacotron_hparams import hparams
    from tacotronv2_wavernn_chinese_b200.tacotron.griffin_lim import GriffinLimEngine
    return GriffinLimEngine(hparams, device=0)


@pytest.fixture(scope='module')
def mels():
    return ae.gl_mels()


def _wave_ok(label, wave, ref, worst):
    l2, edge = ae.wave_errors(wave, ref)
    worst[0], worst[1] = max(worst[0], l2), max(worst[1], edge)
    return l2, edge, l2 <= ae.GL_WAVE_L2 and edge <= ae.GL_EDGE


def test_n_iters_0_every_T(engine, mels):
    worst = [0.0, 0.0]
    for name, mel in mels.items():
        T = mel.shape[1]
        u = ae.gl_phase(T)
        wave = engine.run(mel.T[None], u=u.T[None], n_iters=0)['wave'].cpu().numpy()[0]
        assert wave.shape == (ae.HOP * (T - 1),)
        ref = go.inv_preemphasis(go.istft(go.magnitude(mel) * go.phasor(u)))
        l2, edge, ok = _wave_ok(name, wave, ref, worst)
        print(f'n_iters=0 {name:10s} T={T:5d} rel L2 {l2:.2e} edge max-abs/peak {edge:.2e}')
        assert ok, (name, l2, edge)
    print(f'n_iters=0: worst rel L2 {worst[0]:.2e}, worst edge {worst[1]:.2e}')


@pytest.fixture(scope='module')
def teacher(engine, mels):
    """One iteration from the seeded phase, every mel alone: {name: (wave, u)}."""
    out = {}
    for name, mel in mels.items():
        r = engine.run(mel.T[None], u=ae.gl_phase(mel.shape[1]).T[None], n_iters=1, want_u=True)
        out[name] = (r['wave'].cpu().numpy()[0], r['u'].cpu().numpy()[0].T)
    return out


def _check_step(label, mel, wave, u, worst):
    S = go.magnitude(mel)
    _, u1 = go.step(S, ae.gl_phase(mel.shape[1]).astype(np.float64))
    pe = ae.phasor_error(u, u1, S)
    l2, edge, ok = _wave_ok(label, wave, go.inv_preemphasis(go.istft(S * go.phasor(u1))), worst)
    worst[2] = max(worst[2], pe)
    print(f'{label:22s} T={mel.shape[1]:5d} phasor {pe:.2e} rel L2 {l2:.2e} edge max-abs/peak {edge:.2e}')
    assert ok and pe <= ae.GL_PHASOR, (label, pe, l2, edge)


def test_teacher_forced_one_iteration_every_T(mels, teacher):
    worst = [0.0, 0.0, 0.0]
    for name, mel in mels.items():
        _check_step(f'one iteration {name}', mel, *teacher[name], worst)
    print(f'teacher forced: worst rel L2 {worst[0]:.2e}, edge {worst[1]:.2e}, phasor {worst[2]:.2e}')


def test_free_running_60_iterations(engine, mels):
    cases = {2: mels['slice2'], 17: mels['slice17'], 400: np.ascontiguousarray(ae.mel_graph()[:400].T), 2000: mels['tiled2000']}
    for T, mel in cases.items():
        u = engine.philox_uniform(7, 0, 1, T)
        wave = engine.run(mel.T[None], u=u, n_iters=60)['wave'].cpu().numpy()[0]
        u64 = u.cpu().numpy()[0].T.astype(np.float64)
        ref = go.inv_mel_spectrogram(mel, u64, 60)
        (bar_l2, bar_mx), fp32 = ae.free_running_bars(mel, u64, ref)
        l2 = float(np.linalg.norm(wave - ref) / np.linalg.norm(ref))
        mx = float(np.abs(wave - ref).max() / np.abs(ref).max())
        print(f'60 iterations T={T:5d}: rel L2 {l2:.2e}, max-abs/peak {mx:.2e} (float32 torch chain {fp32[0]:.2e} / '
              f'{fp32[1]:.2e}; bars {bar_l2:.1e} / {bar_mx:.1e})')
        assert l2 <= bar_l2 and mx <= bar_mx, (T, l2, mx, fp32)


def test_ragged_batch_of_every_T(engine, mels, teacher):
    names = list(mels)
    frames = [mels[k].shape[1] for k in names]
    Tm = max(frames)
    batch = np.full((len(names), Tm, 80), 3.0, np.float32)          # padding frames must not leak into a row
    u = np.full((len(names), Tm, go.N_BINS), 0.25, np.float32)
    for i, k in enumerate(names):
        batch[i, :frames[i]] = mels[k].T
        u[i, :frames[i]] = ae.gl_phase(frames[i]).T
    r = engine.run(batch, frames, u=u, n_iters=1, want_u=True)
    wave, ur = r['wave'].cpu().numpy(), r['u'].cpu().numpy()
    worst = [0.0, 0.0, 0.0]
    for i, k in enumerate(names):
        L = ae.HOP * (frames[i] - 1)
        assert np.array_equal(wave[i, :L], teacher[k][0]) and not wave[i, L:].any(), k
        assert np.array_equal(ur[i, :frames[i]].T, teacher[k][1]), k
        _check_step(f'ragged {k}', mels[k], wave[i, :L], ur[i, :frames[i]].T, worst)
    print(f'ragged: worst rel L2 {worst[0]:.2e}, edge {worst[1]:.2e}, phasor {worst[2]:.2e}')
