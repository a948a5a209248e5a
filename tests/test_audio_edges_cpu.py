"""The edge sweeps of mel analysis and Griffin-Lim without a GPU (inputs and bars: tests/audio_edge_cases.py).

- The oracle's stft / istft against float64 torch.stft / torch.istft at every Griffin-Lim frame count of the sweep.
- The sweep's signals are what their names say (trim bounds, margins, where the peaks sit).
- The bars are true: every per-signal mel bar is at least 3x the float32 FFT chain's error on that signal, and a float32
  torch stft / istft chain is at least 3x under the Griffin-Lim bars at every T.
- The bars are sharp: each perturbation of the oracle chain below fails the bar the GPU is held to on at least one input.
"""
import numpy as np
import pytest

import audio_edge_cases as ae
from oracle import griffin_lim_oracle as go
from oracle import mel_analysis_oracle as mo
from test_mel_analysis_cpu import mel_errors

torch = pytest.importorskip('torch')

GL_T = sorted({m.shape[1] for m in ae.gl_mels().values()})


@pytest.fixture(scope='module')
def plain():
    return ae.plain_signals()


@pytest.fixture(scope='module')
def pre():
    return ae.preprocess_signals()


@pytest.fixture(scope='module')
def mels():
    return ae.gl_mels()


# ---- the oracle's stft / istft ------------------------------------------------------------------------------------------
def test_oracle_stft_istft_against_torch_every_T():
    w = torch.hann_window(go.WIN, periodic=True, dtype=torch.float64)
    rs = np.random.RandomState(3)
    for T in GL_T:
        y = rs.standard_normal(go.HOP * (T - 1))
        X = torch.stft(torch.from_numpy(y), go.N_FFT, go.HOP, go.WIN, w, center=True, pad_mode='constant',
                       return_complex=True).numpy()
        assert X.shape == (go.N_BINS, T)
        assert np.abs(go.stft(y) - X).max() <= 1e-12 * np.abs(X).max(), T
        yi = torch.istft(torch.from_numpy(X), go.N_FFT, go.HOP, go.WIN, w, center=True).numpy()
        assert yi.shape == y.shape and np.abs(go.istft(X) - yi).max() <= 1e-12 * np.abs(y).max(), T


# ---- the signals --------------------------------------------------------------------------------------------------------
def test_plain_signals_cover_every_frame_count_edge(plain):
    Ls = sorted(len(x) for x in plain.values())
    assert Ls == sorted(ae.PLAIN_LENGTHS)
    frames = {1 + L // ae.HOP for L in Ls}
    assert {1, 2, 3, 4, 5, 8, 401, 402, 4811} <= frames
    for x in plain.values():
        assert x.dtype == np.float32 and np.isfinite(x).all() and np.abs(x).max() > 0


def test_preprocess_signals(pre):
    r = {k: ae.oracle_analysis(x, ae.ALL) for k, x in pre.items()}
    for k, x in pre.items():
        assert x.dtype == np.float32 and len(x) >= mo.TRIM_N, k
        assert ae.trim_margin_db(x) >= ae.MARGIN_DB, k                  # exact bounds are a fair demand
        s, e = r[k]['bounds']
        assert 0 <= s < e <= len(x) and r[k]['mel'].shape[0] == 1 + (e - s) // ae.HOP, k
    b = {k: v['bounds'] for k, v in r.items()}
    assert b['burst_at_0'][0] == 0 and b['burst_at_0'][1] < len(pre['burst_at_0'])
    assert b['burst_to_end'][1] == len(pre['burst_to_end']) and len(pre['burst_to_end']) % mo.TRIM_HOP
    assert 0 < b['burst_inside'][0] and b['burst_inside'][1] < len(pre['burst_inside'])
    s, e = b['two_bursts']
    assert mo.trim_db(pre['two_bursts'])[s // mo.TRIM_HOP:e // mo.TRIM_HOP].min() < -40      # a kept silence
    for m in (0, 1, 274):
        s, e = b[f'trim_mod{m}']
        assert (e - s) % ae.HOP == m and s > 0
    assert {len(pre[f'len{L}']) for L in (2048, 2049, 2559, 2560, 2561)} == {2048, 2049, 2559, 2560, 2561}
    # floor_then_spike: the floor frames are just under the threshold, and the first kept sample is the pre-emphasised peak
    x, (s, e) = pre['floor_then_spike'], b['floor_then_spike']
    db = mo.trim_db(x)
    assert s > 0 and -26 < db[s // mo.TRIM_HOP - 1] < -mo.TOP_DB
    assert np.argmax(np.abs(r['floor_then_spike']['sig'])) == 0 and abs(x[s - 1]) > 1e-3
    s, e = b['peak_last']
    assert e == len(pre['peak_last']) and np.argmax(np.abs(r['peak_last']['sig'])) == e - s - 1
    x, (s, e) = pre['spike_in_silence'], b['spike_in_silence']
    assert np.abs(mo.preemphasis(x)).max() > 1.5 * np.abs(mo.preemphasis(x[s:e])).max()


# ---- the bars are true ----------------------------------------------------------------------------------------------------
def _cases(plain, pre):
    """(name, flags, oracle result) of every mel the GPU sweep checks."""
    out = [(k, 0, ae.oracle_analysis(x, 0)) for k, x in plain.items()]
    out += [(k, ae.ALL, ae.oracle_analysis(x, ae.ALL)) for k, x in pre.items()]
    for k in ae.FLAG_SIGNALS:
        out += [(k, f, ae.oracle_analysis(pre[k], f)) for f in range(8) if f != ae.ALL]
    return out


def test_mel_bars_are_true(plain, pre):
    """Every per-signal bar is at least 3x the float32 FFT chain's error on that signal, and none is loose: at most 25x GPU_BARS
    (the chirp's loud-band error is the largest, 2.2e-5)."""
    from test_mel_analysis_cpu import GPU_BARS
    worst = dict.fromkeys(ae.BAR_KEYS, 0.0)
    for name, flags, r in _cases(plain, pre):
        bars, errs = ae.mel_bars(r['sig'], r['mel'])
        for k in ae.BAR_KEYS:
            assert errs[k] * 3 <= bars[k] <= 25 * GPU_BARS[k], (name, flags, k, errs[k], bars[k])
            worst[k] = max(worst[k], errs[k])
    print('fp32 chain, worst over the sweep: ' + ', '.join(f'{k} {v:.2e}' for k, v in worst.items()))


def test_griffin_lim_bars_are_true(mels):
    """A float32 stft / istft chain is at least 3x under every Griffin-Lim bar, at every T: after the magnitude stage and
    one istft (n_iters = 0), and teacher forced through one iteration."""
    worst = np.zeros(5)
    for name, mel in mels.items():
        T = mel.shape[1]
        u = ae.gl_phase(T).astype(np.float64)
        S = go.magnitude(mel)
        y0 = go.inv_preemphasis(go.istft(S * go.phasor(u)))
        _, u1 = go.step(S, u)
        w0 = ae.wave_errors(ae.fp32_griffin_lim(mel, u, 0)[0], y0)
        g1, g1u = ae.fp32_griffin_lim(mel, u, 1)
        w1 = ae.wave_errors(g1, go.inv_preemphasis(go.istft(S * go.phasor(u1))))
        e = np.array([w0[0], w0[1], w1[0], w1[1], ae.phasor_error(g1u, u1, S)])
        assert (3 * e <= [ae.GL_WAVE_L2, ae.GL_EDGE, ae.GL_WAVE_L2, ae.GL_EDGE, ae.GL_PHASOR]).all(), (name, e)
        worst = np.maximum(worst, e)
    print('fp32 Griffin-Lim, worst: n_iters=0 rel L2 %.1e edge %.1e; one iteration rel L2 %.1e edge %.1e phasor %.1e' % tuple(worst))


# ---- the bars are sharp: mel analysis -------------------------------------------------------------------------------------
def _melspec(y, window=None, shift=0, basis=None):
    """mo.melspectrogram with a replaceable window and filterbank, and the frame grid moved by `shift` samples."""
    w = go.window() if window is None else window
    yp = np.pad(np.asarray(y, np.float64), (go.N_FFT // 2 - shift, go.N_FFT // 2 + shift))
    T = 1 + len(y) // go.HOP
    idx = np.arange(go.N_FFT)[None, :] + go.HOP * np.arange(T)[:, None]
    S = np.abs(np.fft.rfft(w[None, :] * yp[idx], axis=1).T) ** 2
    mel = (go.mel_basis() if basis is None else basis) @ S
    db = 20 * np.log10(np.maximum(np.exp(mo.MIN_DB / 20 * np.log(10)), mel)) - mo.REF_DB
    return np.clip((2 * mo.MAX_ABS) * ((db - mo.MIN_DB) / (-mo.MIN_DB)) - mo.MAX_ABS, -mo.MAX_ABS, mo.MAX_ABS)


def _symmetric_hann():
    w = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(go.WIN) / (go.WIN - 1))
    lpad = (go.N_FFT - go.WIN) // 2
    return np.pad(w, (lpad, go.N_FFT - go.WIN - lpad))


def _short_band():
    """The filterbank with one band's non-zero bin range shortened by its last bin (the band where that bin weighs most)."""
    M = go.mel_basis()
    last = [np.flatnonzero(r)[-1] for r in M]
    m = int(np.argmax([M[i, last[i]] / M[i].sum() for i in range(len(M))]))
    M = M.copy()
    M[m, last[m]] = 0
    return M


MEL_PERTURBATIONS = {
    'frame grid shifted by one sample': dict(melspectrogram=lambda y: _melspec(y, shift=1)),
    'symmetric Hann': dict(melspectrogram=lambda y: _melspec(y, window=_symmetric_hann())),
    'pre-emphasis seeded with wav[s-1]': dict(seed_with_previous=True),
    'rescale peak over the untrimmed signal': dict(peak_untrimmed=True),
    "one band's bin range shortened by a bin": dict(melspectrogram=lambda y: _melspec(y, basis=_short_band())),
}


def test_mel_harness_is_the_oracle(pre):
    x = pre['burst_inside']
    assert np.array_equal(_melspec(x.astype(np.float64)), mo.melspectrogram(x.astype(np.float64)))


@pytest.mark.parametrize('what', list(MEL_PERTURBATIONS))
def test_mel_perturbation_is_rejected(plain, pre, what):
    kw = MEL_PERTURBATIONS[what]
    rejected = []
    sweep = [(k, 0, x) for k, x in plain.items()] + [(k, ae.ALL, x) for k, x in pre.items()]
    for name, flags, x in sweep:
        ref = ae.oracle_analysis(x, flags)
        bars, _ = ae.mel_bars(ref['sig'], ref['mel'])
        bad = ae.oracle_analysis(x, flags, **kw)
        if bad['mel'].shape != ref['mel'].shape or not ae.within(mel_errors(bad['mel'], ref['mel']), bars):
            rejected.append(name)
    print(f'{what}: rejected on {len(rejected)} of {len(sweep)} signals: {", ".join(rejected)}')
    assert rejected


# ---- the bars are sharp: Griffin-Lim --------------------------------------------------------------------------------------
def _istft_last_hop_short(X):
    """go.istft with the envelope of the last hop of output samples summed over T - 1 frames instead of T."""
    T = X.shape[1]
    frames = go.window()[None, :] * np.fft.irfft(X.T, n=go.N_FFT, axis=1)
    y = np.zeros(go.N_FFT + go.HOP * (T - 1))
    for t in range(T):
        y[t * go.HOP:t * go.HOP + go.N_FFT] += frames[t]
    env = go.envelope(T)
    a = go.N_FFT // 2 + go.HOP * (T - 2)                        # first untrimmed index of the last hop of output
    env[a:len(env) - go.HOP] = go.envelope(T - 1)[a:] if T > 1 else 0
    nz = env > np.finfo(np.float32).tiny
    y[nz] /= env[nz]
    return y[go.N_FFT // 2:-(go.N_FFT // 2)]


def _inv_preemphasis_restarted(y):
    """lfilter([1], [1, -0.97]) restarted from a zero state at the middle one of gl_finish_kernel's 1024 chunk boundaries."""
    chunk = -(-len(y) // 1024)
    b = chunk * max(1, (len(y) // chunk) // 2)
    if b >= len(y):
        return go.inv_preemphasis(y)
    return np.concatenate([go.inv_preemphasis(y[:b]), go.inv_preemphasis(y[b:])])


def _tile_edge_mel(mel):
    """Frame 16 of every 16-frame magnitude tile (index 15) computed from frame 15's mel (index 14)."""
    m = mel.copy()
    m[:, 15::16] = mel[:, 14::16][:, :m[:, 15::16].shape[1]]
    return m


GL_PERTURBATIONS = {
    "last hop's envelope over T - 1 frames": lambda mel, S, u: go.inv_preemphasis(_istft_last_hop_short(S * go.phasor(u))),
    'inverse pre-emphasis restarted at a chunk boundary': lambda mel, S, u: _inv_preemphasis_restarted(go.istft(S * go.phasor(u))),
    'magnitude tile frame 16 from frame 15': lambda mel, S, u: go.inv_preemphasis(go.istft(go.magnitude(_tile_edge_mel(mel))
                                                                                          * go.phasor(u))),
}


@pytest.mark.parametrize('what', list(GL_PERTURBATIONS))
def test_griffin_lim_perturbation_is_rejected(mels, what):
    """Each perturbation of the n_iters = 0 chain (magnitude, istft, inverse pre-emphasis) fails the wave bars on at least
    one mel of the sweep."""
    rejected = []
    for name, mel in mels.items():
        u = ae.gl_phase(mel.shape[1]).astype(np.float64)
        S = go.magnitude(mel)
        ref = go.inv_preemphasis(go.istft(S * go.phasor(u)))
        l2, edge = ae.wave_errors(GL_PERTURBATIONS[what](mel, S, u), ref)
        if l2 > ae.GL_WAVE_L2 or edge > ae.GL_EDGE:
            rejected.append(name)
    print(f'{what}: rejected on {len(rejected)} of {len(mels)} mels: {", ".join(rejected)}')
    assert rejected
