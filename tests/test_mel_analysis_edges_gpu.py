"""Mel analysis on the GPU (csrc/mel_analysis.cuh) against the float64 oracle at every signal of the edge sweep
(tests/audio_edge_cases.py): lengths below one hop, one window and one FFT up to 60 s, trim bounds at both ends and inside,
trimmed lengths at every remainder edge, the trimmed start and both rescale peaks, and all eight flag combinations.

Frames, bounds and the training audio `out` are exact; the mel is within the per-signal bar (6x what a float32 FFT chain makes
against the oracle on that signal); frames beyond T are zero.  A ragged call holding every signal, its padding filled with NaN,
must give each row its stand-alone result bit for bit: a kernel that read past a row's length would turn it into NaN.
Run with -s to see the errors and the GPU / float32-chain ratios (recorded in DESIGN.md section 3.8).
"""
import numpy as np
import pytest

import audio_edge_cases as ae
from test_mel_analysis_cpu import mel_errors

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def engine():
    import torch
    assert torch.cuda.is_available()
    from tacotron_hparams import hparams
    from tacotronv2_wavernn_chinese_b200.tacotron import mel_analysis
    assert (mel_analysis.TRIM, mel_analysis.PREEMPHASIS, mel_analysis.RESCALE) == (ae.TRIM, ae.PREEMPHASIS, ae.RESCALE)
    assert mel_analysis.preprocess_flags(hparams) == ae.ALL
    return mel_analysis.MelAnalysisEngine(hparams, device=0)


SIGNALS = {'plain': (ae.plain_signals, 0), 'preprocess': (ae.preprocess_signals, ae.ALL)}


def _run(engine, wavs, flags, pad=np.nan):
    L = max(len(w) for w in wavs)
    batch = np.full((len(wavs), L), pad, np.float32)
    for i, w in enumerate(wavs):
        batch[i, :len(w)] = w
    r = engine.run(batch, [len(w) for w in wavs], flags=flags, want_audio=True)
    return {k: v.cpu().numpy() for k, v in r.items()}


def _check(label, wav, flags, r, i=0):
    """Row i of a run against the oracle; returns the errors and their ratios to the float32 chain's."""
    ref = ae.oracle_analysis(wav, flags)
    T = int(r['frames'][i])
    assert T == ref['mel'].shape[0], (label, T)
    assert tuple(int(v) for v in r['bounds'][i]) == ref['bounds'], label
    out = r['audio'][i]
    assert np.array_equal(out[:T * ae.HOP], ref['out']) and not out[T * ae.HOP:].any(), label
    assert not r['mel'][i, T:].any(), label
    bars, fp32 = ae.mel_bars(ref['sig'], ref['mel'])
    errs = mel_errors(r['mel'][i, :T], ref['mel'])
    ratios = [e / max(fp32[k], 1e-30) for e, k in zip(errs, ae.BAR_KEYS)]
    print(f'{label:28s} T={T:5d} loud {errs[0]:.2e} max {errs[1]:.2e} rel L2 {errs[2]:.2e}   GPU/fp32 '
          + ' '.join(f'{x:.2f}' for x in ratios))
    assert ae.within(errs, bars), (label, errs, bars)
    return np.array(errs), np.array(ratios)


def _report(what, rows):
    errs = np.max([e for e, _ in rows], axis=0)
    ratios = np.max([q for _, q in rows], axis=0)
    print(f'{what}: worst loud {errs[0]:.2e} max {errs[1]:.2e} rel L2 {errs[2]:.2e}; worst GPU/fp32 ratio '
          + ' / '.join(f'{x:.2f}' for x in ratios))


@pytest.fixture(scope='module')
def solo(engine):
    """Stand-alone runs of every signal: {mode: {name: (signal, result)}}."""
    out = {}
    for mode, (make, flags) in SIGNALS.items():
        out[mode] = {k: (x, _run(engine, [x], flags)) for k, x in make().items()}
    return out


@pytest.mark.parametrize('mode', list(SIGNALS))
def test_every_signal_against_the_oracle(solo, mode):
    flags = SIGNALS[mode][1]
    rows = [_check(f'{mode} {k}', x, flags, r) for k, (x, r) in solo[mode].items()]
    _report(mode, rows)


def test_every_flag_combination(engine):
    """All eight combinations of TRIM, PREEMPHASIS and RESCALE on the signals where the trimmed start and the peaks matter,
    against the oracle composed in the reference's order."""
    pre = ae.preprocess_signals()
    rows = []
    for k in ae.FLAG_SIGNALS:
        for flags in range(8):
            rows.append(_check(f'{k} flags={flags}', pre[k], flags, _run(engine, [pre[k]], flags)))
    _report('flags 0-7', rows)


@pytest.mark.parametrize('mode', list(SIGNALS))
def test_ragged_nan_padded_batch(engine, solo, mode):
    """One call with every signal, padding beyond each row's length NaN: each row matches the oracle and is bit-equal to its
    stand-alone run."""
    flags = SIGNALS[mode][1]
    names = list(solo[mode])
    wavs = [solo[mode][k][0] for k in names]
    r = _run(engine, wavs, flags, pad=np.nan)
    rows = []
    for i, k in enumerate(names):
        a = solo[mode][k][1]
        T = int(a['frames'][0])
        assert int(r['frames'][i]) == T and np.array_equal(r['bounds'][i], a['bounds'][0]), k
        assert np.array_equal(r['mel'][i, :T], a['mel'][0, :T]), k
        assert np.array_equal(r['audio'][i, :T * ae.HOP], a['audio'][0, :T * ae.HOP]), k
        assert np.isfinite(r['mel'][i]).all() and np.isfinite(r['audio'][i]).all(), k
        rows.append(_check(f'ragged {mode} {k}', wavs[i], flags, r, i))
    _report(f'ragged {mode}', rows)
