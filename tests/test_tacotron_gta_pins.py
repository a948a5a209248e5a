"""Ground-truth-aligned (GTA) decoding, the teacher-forced loop of the reference's wavernn_preprocess.py (CPU suite).

Pins of oracle.tacotron_gta_oracle.decode_gta:
  * against tests/golden/taco_gta_from_graph.npz: the reference's demo recording (demo/03) teacher-forced through its own
    serialized decoder-step graph for all 323 steps, next input and step count from the reference's own TacoTrainingHelper
    (oracle/make_golden_taco_gta.py; measured difference 0.0);
  * fed the frames of the free-running graph run (tests/golden/taco_run_from_graph.npz) with the same masks, it replays
    that run exactly;
  * float32 against float64 over every step of both cases: the calibration of the GPU bar (a fed frame removes the feedback
    that makes the free-running decoder chaotic, tests/test_tacotron_oracle.py).
Also the `encode_mu_law` restatement and the argument checks of wavernn_preprocess.py.
"""
import ast
import os
import types
import warnings

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import tacotron_gta_oracle as gta
from oracle import tacotron_oracle as to
from taco_common import real_taco_weights, synth_taco_weights

REF_AUDIO = '/root/reference/tacotron/datasets/audio.py'


def _gta_fixture():
    z = np.load(os.path.join(GOLDEN, 'taco_gta_from_graph.npz'))
    n = int(z['n_steps'])
    masks = np.unpackbits(z['masks'], axis=1)[:, :512].reshape(n, 2, 256).astype(np.float32)
    src = np.load(os.path.join(GOLDEN, str(z['target_file'])))[str(z['target_key'])]
    targets = np.clip(src, -float(z['target_clip']), float(z['target_clip'])).astype(np.float32)
    return z, n, masks, targets


def _run_fixture():
    z = np.load(os.path.join(GOLDEN, 'taco_run_from_graph.npz'))
    n = int(z['n_steps'])
    masks = np.unpackbits(z['masks'], axis=1)[:, :512].reshape(n, 2, 256).astype(np.float32)
    return z, n, masks


def _weights():
    w = real_taco_weights()
    if w is None:
        pytest.skip('shipped Tacotron checkpoint not available on this box')
    return w


def _quiet(fn, *a, **k):
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', RuntimeWarning)                  # exp overflow inside the sigmoid of large logits
        return fn(*a, **k)


def test_gta_fixture_and_reference_helper_semantics():
    """What the reference's own TacoTrainingHelper did while the fixture was made: the GO frame is all zeros, the input
    after step t is targets[t] (r = 1), `finished` is first true after exactly len(targets) steps."""
    z, n, masks, targets = _gta_fixture()
    assert n == targets.shape[0] == 323 and z['frames'].shape == (n, 80) and z['mel_graph'].shape == (n, 80)
    assert z['memory_graph'].shape == (len(z['ids']), 512)
    assert str(z['text']) == '如果打穿地球，那么从一头到另一头h ui4发生什么？'
    assert np.array_equal(z['helper_go'], np.zeros(80, np.float32))
    assert np.array_equal(z['helper_finished'], np.arange(n) + 1 >= n)
    for t, nxt in zip(z['helper_probe_times'], z['helper_probe_next']):
        assert np.array_equal(nxt, targets[t]), t
    assert 0.4 < masks.mean() < 0.6
    am = z['align_argmax'].astype(int)
    assert am[0] <= 1 and am[-1] >= len(z['ids']) - 2 and (np.diff(am) >= -1).all()   # attends to the end of the text


def test_oracle_gta_semantics_synthetic_weights():
    """decode_gta = decode with the recorded frame fed back: fed a free run's own frames it replays that run; it runs exactly
    len(targets) steps whatever the stop token says; and the first step sees the GO frame, not targets[0]."""
    w = synth_taco_weights(7)
    mem = np.random.RandomState(1).uniform(-1, 1, (19, 512)).astype(np.float32)
    masks = (np.random.RandomState(2).uniform(size=(30, 2, 256)) >= 0.5).astype(np.float32)
    free = to.decode(w, mem, dropout_masks=masks, max_iters=30)
    n = free['n_steps']
    g = gta.decode_gta(w, mem, free['frames'], dropout_masks=masks)
    assert g['n_steps'] == n and np.array_equal(g['frames'], free['frames'])
    assert np.array_equal(g['alignments'], free['alignments'])
    tg = np.random.RandomState(3).uniform(-4, 4, (41, 80)).astype(np.float32)
    a = gta.decode_gta(w, mem, tg, seed=5)
    assert a['n_steps'] == 41 and a['masks'].shape == (41, 2, 256)
    b = gta.decode_gta(w, mem, np.concatenate([tg[:40], -tg[40:]]), seed=5)           # the last target is never fed
    assert np.array_equal(a['frames'], b['frames'])
    c = gta.decode_gta(w, mem, np.concatenate([-tg[:1], tg[1:]]), seed=5)             # targets[0] feeds step 1, not step 0
    assert np.array_equal(a['frames'][0], c['frames'][0]) and not np.array_equal(a['frames'][1], c['frames'][1])


def test_gta_replays_the_free_running_graph_run():
    """Fed the 405 frames of the free-running graph run (tests/golden/taco_run_from_graph.npz) with its masks, decode_gta
    reproduces those frames exactly (measured difference 0.0)."""
    w = _weights()
    z, n, masks = _run_fixture()
    d = _quiet(gta.decode_gta, w, to.encoder(w, z['ids']), z['frames'], dropout_masks=masks)
    err = np.abs(d['frames'] - z['frames']).max(axis=1)
    assert d['n_steps'] == n == 405
    assert err.max() <= 1e-6, (int(err.argmax()), float(err.max()))
    assert np.array_equal(d['alignments'].argmax(1), z['align_argmax'])


def test_gta_matches_the_teacher_forced_graph_run():
    """Demo-03 against the serialized graph driven by the reference's TacoTrainingHelper: every frame and alignment over all
    323 steps (measured 0.0), and the postnet over the whole mel (measured 1.2e-6 on the +-4 scale)."""
    w = _weights()
    z, n, masks, targets = _gta_fixture()
    d = _quiet(gta.decode_gta, w, z['memory_graph'], targets, dropout_masks=masks)
    assert d['n_steps'] == n
    err = np.abs(d['frames'] - z['frames']).max(axis=1)
    assert err.max() <= 1e-6, (int(err.argmax()), float(err.max()))
    assert np.array_equal(d['alignments'].argmax(1), z['align_argmax'])
    np.testing.assert_allclose(d['alignments'].max(1), z['align_peak'], rtol=0, atol=1e-6)
    assert np.abs(to.postnet(w, d['frames']) - z['mel_graph']).max() <= 1e-5


def _gta64(w, memory, targets, masks):
    old = to.F32
    try:
        to.F32 = np.float64
        return _quiet(gta.decode_gta, {k: v.astype(np.float64) for k, v in w.items()}, memory.astype(np.float64),
                      targets.astype(np.float64), dropout_masks=masks.astype(np.float64))
    finally:
        to.F32 = old


@pytest.mark.parametrize('case', ['run405', 'demo03'])
def test_gta_is_not_chaotic_fp32_vs_fp64(case):
    """The calibration of the GPU bar: float32 and float64 evaluations of decode_gta with the same masks stay within 2e-5 over
    EVERY step (measured 7.8e-6 over 405 steps and 4.5e-6 over 323), where free running parts ways after ~100 steps."""
    w = _weights()
    if case == 'run405':
        z, n, masks = _run_fixture()
        memory, targets = to.encoder(w, z['ids']), z['frames']
    else:
        z, n, masks, targets = _gta_fixture()
        memory = z['memory_graph']
    r32 = _quiet(gta.decode_gta, w, memory, targets, dropout_masks=masks)
    r64 = _gta64(w, memory, targets, masks)
    err = np.abs(r32['frames'] - r64['frames']).max(axis=1)
    assert len(err) == n and err.max() < 2e-5, (int(err.argmax()), float(err.max()))
    assert np.abs(r32['alignments'] - r64['alignments']).max() < 2e-6


# ---------------------------------------------------------------- encode_mu_law (tacotron/datasets/audio.py:8-11)

def _lifted_reference_mu_law(numpy_module):
    """The reference's `encode_mu_law`, lifted from its source by AST and executed with `np` bound to `numpy_module`."""
    if not os.path.isfile(REF_AUDIO):
        pytest.skip('reference checkout not present')
    tree = ast.parse(open(REF_AUDIO, encoding='utf-8').read())
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == 'encode_mu_law')
    ns = {'np': numpy_module}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), REF_AUDIO, 'exec'), ns)
    return ns['encode_mu_law']


def _numpy1_log():
    """numpy with numpy 1.x's value-based casting for the one statement where it matters: `np.log(1 + mu)` of a Python int is a
    float64 scalar, which numpy 1.x demoted to the float32 of the array it divides."""
    m = types.SimpleNamespace(**{k: getattr(np, k) for k in ('sign', 'abs', 'floor')})
    m.log = lambda v: np.log(v) if isinstance(v, np.ndarray) else np.float32(np.log(v))
    return m


def _demo_training_audio():
    from oracle import mel_analysis_oracle as mo
    c = mo.fixture_case(os.path.join(GOLDEN, 'mel_analysis_from_reference.npz'), 'speech')
    out = mo.process_utterance(c['wav'])['out']
    assert mo.sha256(out) == c['out_sha256']                        # the reference's own training audio of demo/03
    return out


def test_encode_mu_law_values():
    from tacotronv2_wavernn_chinese_b200.tacotron.audio import encode_mu_law
    x = np.array([-1.0, -0.5, 0.0, 1e-4, 0.5, 1.0], dtype=np.float32)
    y = encode_mu_law(x)
    assert y.dtype == np.float32 and y[0] == 0 and y[2] == 512 and y[-1] == 1023
    assert (np.diff(y) >= 0).all() and (y == np.floor(y)).all()
    assert encode_mu_law(x.astype(np.float64)).dtype == np.float64


def test_encode_mu_law_pinned_to_the_reference():
    """Under numpy 1.x (the reference's TF 1.14 environment) every operation on the float32 training audio is float32; the
    restatement equals the lifted reference statement evaluated that way on the demo's training audio and on a dense grid.
    Evaluated verbatim under numpy 2 (float64 from the division on), the statement rounds 0 of the demo's 88 825 samples
    and 41 of 2 000 001 grid points to the neighbouring level; in float64 the restatement is the verbatim statement."""
    from tacotronv2_wavernn_chinese_b200.tacotron.audio import encode_mu_law
    ref_np1 = _lifted_reference_mu_law(_numpy1_log())
    ref_np2 = _lifted_reference_mu_law(np)
    demo = _demo_training_audio()
    grid = np.linspace(-1, 1, 2_000_001, dtype=np.float32)
    for x in (demo, grid):
        ours = encode_mu_law(x)
        r1 = ref_np1(x)
        assert r1.dtype == np.float32 and np.array_equal(ours, r1)
        assert np.array_equal(encode_mu_law(x.astype(np.float64)), ref_np2(x.astype(np.float64)))
        r2 = ref_np2(x)
        assert r2.dtype == np.float64 and np.abs(r2 - ours).max() <= 1
    assert int((ref_np2(demo) != encode_mu_law(demo)).sum()) == 0 and len(demo) == 88825
    assert int((ref_np2(grid) != encode_mu_law(grid)).sum()) == 41


# ---------------------------------------------------------------- wavernn_preprocess.py argument checks

def _no_model(monkeypatch):
    from tacotronv2_wavernn_chinese_b200.tacotron import synthesizer

    def refuse(*a, **k):
        raise AssertionError('the model was loaded before the arguments were checked')
    monkeypatch.setattr(synthesizer.Synthesizer, 'load', refuse)


def test_cli_requires_data_dir(monkeypatch, capsys):
    import wavernn_preprocess
    _no_model(monkeypatch)
    with pytest.raises(SystemExit):
        wavernn_preprocess.main([])
    assert '--data_dir' in capsys.readouterr().err


@pytest.mark.parametrize('bad', ['audio-000002.npy|mel-000002.npy|51425|187', 'audio-000002.npy|mel.npy|51425|187|假语。|j ia3 。'])
def test_cli_rejects_a_malformed_line_before_the_model(tmp_path, monkeypatch, capsys, bad):
    import wavernn_preprocess
    _no_model(monkeypatch)
    good = 'audio-000001.npy|mel-000001.npy|46200|168|卡尔普陪外孙玩滑梯。|k a3 er3 p u3 p ei2 w ai4 s un1 w an2 h ua2 t i1 。'
    (tmp_path / 'train.txt').write_text(good + '\n' + bad + '\n', encoding='utf-8')
    with pytest.raises(SystemExit):
        wavernn_preprocess.main(['--data_dir', str(tmp_path), '--out_dir', str(tmp_path / 'out')])
    assert 'line 2' in capsys.readouterr().err
    assert not (tmp_path / 'out').exists()
    assert wavernn_preprocess.parse_line(good, 1) == ('audio-000001.npy', 'mel-000001.npy', '卡尔普陪外孙玩滑梯。', '000001')


def test_cli_missing_list_and_bad_batch(tmp_path, monkeypatch, capsys):
    import wavernn_preprocess
    _no_model(monkeypatch)
    with pytest.raises(SystemExit):
        wavernn_preprocess.main(['--data_dir', str(tmp_path)])
    assert 'train.txt' in capsys.readouterr().err
    with pytest.raises(SystemExit):
        wavernn_preprocess.main(['--data_dir', str(tmp_path), '--batch', '0'])
