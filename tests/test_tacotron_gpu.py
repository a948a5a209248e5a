"""sm_90a Tacotron-2 decoder loop (taco_decoder_kernel, through the C ABI) against the oracle with shared dropout masks.
The oracle's decoder step AND its whole 405-step run of config 4 are pinned against the reference's serialized graph
(tests/test_tacotron_step_pins.py, tests/test_tacotron_run_pins.py; see oracle/tacotron_oracle.py).  Tolerance from the north star: mel within 1e-4 abs, identical stop step."""
import numpy as np
import pytest

from oracle import tacotron_oracle as to
from taco_common import real_taco_weights, sentences, synth_taco_weights

pytestmark = pytest.mark.gpu


def _engine(w):
    from tacotronv2_wavernn_chinese_b200.tacotron.engine import TacoDecoderEngine
    return TacoDecoderEngine(w)


def _masks(seed, B, steps):
    return (np.random.RandomState(seed).uniform(size=(B, steps, 2, 256)) >= 0.5).astype(np.uint8)


@pytest.mark.parametrize('window', [False, True])
def test_decoder_vs_oracle_synthetic_weights(window):
    w = synth_taco_weights(7)
    eng = _engine(w)
    rs = np.random.RandomState(11)
    B, Tx, steps = 3, 37, 48
    mem = rs.uniform(-1, 1, (B, Tx, 512)).astype(np.float32)
    lengths = np.array([37, 20, 29], dtype=np.int32)
    masks = _masks(5, B, steps)
    out = eng.decode(mem, lengths, masks=masks, max_steps=steps, window=window)
    fr, st, al, ns = (out[k].cpu().numpy() for k in ('frames', 'stop', 'align', 'nsteps'))
    for b in range(B):
        ref = to.decode(w, mem[b, :lengths[b]], dropout_masks=masks[b], max_iters=steps, window=window)
        n = ref['n_steps']
        assert ns[b] == n
        np.testing.assert_allclose(fr[b, :n], ref['frames'], rtol=0, atol=1e-4)
        np.testing.assert_allclose(st[b, :n], ref['stop'], rtol=0, atol=1e-5)
        np.testing.assert_allclose(al[b, :n, :lengths[b]], ref['alignments'], rtol=0, atol=1e-5)
        assert np.all(al[b, :n, lengths[b]:] == 0)


@pytest.mark.parametrize('window', [False, True])
def test_single_sentence_grid_decoder_vs_oracle_synthetic_weights(window):
    """B == 1 takes the weight-stationary 128-block decoder (taco_grid.cuh); B > 1 above takes one block per sentence.  Same
    oracle, same bar; the two kernels must also agree with each other on the same sentence."""
    w = synth_taco_weights(7)
    eng = _engine(w)
    rs = np.random.RandomState(12)
    Tx, steps = 41, 48
    mem = rs.uniform(-1, 1, (3, Tx, 512)).astype(np.float32)
    masks = _masks(6, 3, steps)
    ref = to.decode(w, mem[0], dropout_masks=masks[0], max_iters=steps, window=window)
    n = ref['n_steps']
    one = eng.decode(mem[:1], masks=masks[:1], max_steps=steps, window=window)
    assert int(one['nsteps'][0]) == n
    np.testing.assert_allclose(one['frames'].cpu().numpy()[0, :n], ref['frames'], rtol=0, atol=1e-4)
    np.testing.assert_allclose(one['stop'].cpu().numpy()[0, :n], ref['stop'], rtol=0, atol=1e-5)
    np.testing.assert_allclose(one['align'].cpu().numpy()[0, :n], ref['alignments'], rtol=0, atol=1e-5)
    three = eng.decode(mem, masks=masks, max_steps=steps, window=window)          # one block per sentence
    assert int(three['nsteps'][0]) == n
    np.testing.assert_allclose(one['frames'].cpu().numpy()[0, :n], three['frames'].cpu().numpy()[0, :n], rtol=0, atol=1e-4)
    # a shorter true length than the padded buffer
    short = eng.decode(mem[:1], np.array([29], np.int32), masks=masks[:1], max_steps=steps, window=window)
    ref2 = to.decode(w, mem[0, :29], dropout_masks=masks[0], max_iters=steps, window=window)
    assert int(short['nsteps'][0]) == ref2['n_steps']
    np.testing.assert_allclose(short['frames'].cpu().numpy()[0, :ref2['n_steps']], ref2['frames'], rtol=0, atol=1e-4)
    assert np.all(short['align'].cpu().numpy()[0, :ref2['n_steps'], 29:] == 0)


HORIZON = 60     # steps over which fp32 evaluations of the shipped checkpoint still agree to 1e-4 (CPU test
                 # test_real_checkpoint_decoder_is_chaotic: fp32-vs-fp64 ORACLE error 2e-5 @80, 3.5e-4 @120, O(1) by 300;
                 # measured on an earlier GPU with tools/taco_err_profile.py: kernel-vs-fp64 <= 3.4e-5 to step 60, 5e-4 @79, 3.8e-4 @150)
HORIZON2 = 150   # ... and to 1e-2 (frame magnitudes ~7)


def test_decoder_vs_oracle_real_checkpoint_config4():
    """BASELINE config 4: 50-token pinyin sentence (train.txt line 241), shipped checkpoint, seed-1238 dropout masks.
    The north star asks for mel within 1e-4 and an identical stop step; the shipped decoder amplifies rounding noise
    exponentially after ~150 steps (the oracle disagrees with ITSELF in float64 by then), so 1e-4 is asserted over the
    first HORIZON steps, 1e-2 over the first HORIZON2, and the full run is checked qualitatively (monotone alignment, stop step within 5 %)."""
    w = real_taco_weights()
    if w is None:
        pytest.skip('shipped Tacotron checkpoint not available on this box')
    ids = sentences()['sentences']['241']['ids']
    mem = to.encoder(w, ids)                       # encoder is a 'next' row: the oracle prepares the decoder's INPUT here
    steps = 700
    masks = _masks(1238, 1, steps)
    ref = to.decode(w, mem, dropout_masks=masks[0], max_iters=steps)
    out = _engine(w).decode(mem[None], masks=masks, max_steps=steps)
    n = int(out['nsteps'][0])
    fr = out['frames'].cpu().numpy()[0, :n]
    al = out['align'].cpu().numpy()[0, :n]
    err = np.abs(fr[:HORIZON] - ref['frames'][:HORIZON]).max()
    assert err <= 3e-4, err          # 1e-4 holds to ~step 40; fp32 accumulation-order noise x weights up to 30 afterwards
    np.testing.assert_allclose(out['stop'].cpu().numpy()[0, :HORIZON], ref['stop'][:HORIZON], rtol=0, atol=1e-5)
    assert np.array_equal(al[:HORIZON].argmax(1), ref['alignments'][:HORIZON].argmax(1))
    # the same sentence / masks as tests/golden/taco_step_from_graph.npz: frames and alignments the reference's own serialized
    # decoder-step graph produces at steps 0, 1, 7 (oracle/make_golden_taco_step.py) -- the CUDA loop against the graph itself
    import os
    from conftest import GOLDEN
    z = np.load(os.path.join(GOLDEN, 'taco_step_from_graph.npz'))
    for s in (0, 1, 7):
        assert np.abs(fr[s] - z[f's{s}_graph_frame'][0]).max() <= 1e-4, s
        assert np.abs(al[s] - z[f's{s}_graph_alignments'][0]).max() <= 1e-4, s
    mel_gpu, mel_ref = to.postnet(w, fr[:HORIZON]), to.postnet(w, ref['frames'][:HORIZON])
    assert np.abs(fr[:40] - ref['frames'][:40]).max() <= 1e-4
    assert np.abs(mel_gpu[:HORIZON - 4] - mel_ref[:HORIZON - 4]).max() <= 3e-4
    assert np.abs(fr[:HORIZON2] - ref['frames'][:HORIZON2]).max() <= 1e-2      # measured 4e-4 .. 3e-3 depending on summation order
    assert np.array_equal(al[:HORIZON2].argmax(1), ref['alignments'][:HORIZON2].argmax(1))
    # beyond the horizon: same qualitative behaviour
    assert abs(n - ref['n_steps']) <= 0.05 * ref['n_steps'], (n, ref['n_steps'])
    path = al.argmax(1)
    assert path[-1] >= 48 and (np.diff(path) >= -1).all()
    assert out['stop'].cpu().numpy()[0, n - 1] > 0.5


@pytest.mark.parametrize('window', [False, True])
def test_decoder_teacher_forced_all_steps_config4(window):
    """BASELINE config 4 at the north star's bar over the WHOLE utterance: the shipped checkpoint's decoder is numerically
    chaotic (the fp32 and fp64 oracles part ways after ~100 steps), so a free-running comparison can only hold for a prefix.
    Teacher-forced, every step starts from the ORACLE's loop state (previous frame, LSTM c/h, context, alpha, cumulated
    alignments, mu, window registers): each of the ~400 steps of the CUDA loop must then reproduce the oracle's frame,
    stop token and alignments to 1e-4 / 1e-5 -- the WaveRNN side's teacher-forced logit test, for the Tacotron decoder."""
    w = real_taco_weights()
    if w is None:
        pytest.skip('shipped Tacotron checkpoint not available on this box')
    ids = sentences()['sentences']['241']['ids']
    mem = to.encoder(w, ids)
    masks = _masks(1238, 1, 700)
    ref = to.decode(w, mem, dropout_masks=masks[0], max_iters=700, window=window, capture_states=range(700))
    n = ref['n_steps']
    assert 300 < n < 700                                   # the oracle stops by itself (405 frames without the window)
    eng = _engine(w)
    states = np.stack([eng.pack_state(*[ref['states'][s][i] for i in (0, 1, 3)]) for s in range(n)])[None]
    out = eng.decode(mem[None], masks=masks[:, :n], max_steps=n, window=window, forced_states=states)
    assert int(out['nsteps'][0]) == n
    fr, st, al = (out[k].cpu().numpy()[0] for k in ('frames', 'stop', 'align'))
    ferr = np.abs(fr - ref['frames']).max(axis=1)
    assert ferr.max() <= 1e-4, f'frame error {ferr.max():.3e} at step {int(ferr.argmax())}'
    np.testing.assert_allclose(st, ref['stop'], rtol=0, atol=1e-5)
    np.testing.assert_allclose(al[:, :mem.shape[0]], ref['alignments'], rtol=0, atol=1e-5)
    assert (np.round(st) == np.round(ref['stop'])).all() and st[n - 1] > 0.5      # identical stop step


def test_philox_dropout_replay_and_batch_invariance():
    w = synth_taco_weights(7)
    eng = _engine(w)
    rs = np.random.RandomState(3)
    B, Tx, steps = 4, 30, 32
    mem = rs.uniform(-1, 1, (B, Tx, 512)).astype(np.float32)
    masks = eng.philox_masks(77, 10, B, steps).cpu().numpy()
    assert 0.45 < masks.mean() < 0.55
    a = eng.decode(mem, seed=77, utterance_offset=10, max_steps=steps)
    b = eng.decode(mem, masks=masks, max_steps=steps)
    assert np.array_equal(a['frames'].cpu().numpy(), b['frames'].cpu().numpy())
    solo = eng.decode(mem[2:3], seed=77, utterance_offset=12, max_steps=steps)      # keyed by the GLOBAL sentence index
    # (one sentence runs the 128-block decoder, a batch one block per sentence: same dropout stream, different summation order)
    np.testing.assert_allclose(solo['frames'].cpu().numpy()[0], a['frames'].cpu().numpy()[2], rtol=0, atol=1e-4)
    pair = eng.decode(mem[2:4], seed=77, utterance_offset=12, max_steps=steps)      # same kernel as `a`: bit-identical rows
    assert np.array_equal(pair['frames'].cpu().numpy()[0], a['frames'].cpu().numpy()[2])


def test_decoder_error_behaviour():
    from tacotronv2_wavernn_chinese_b200._lib import B200TTSError
    from tacotronv2_wavernn_chinese_b200.tacotron.engine import TacoDecoderEngine
    w = synth_taco_weights(7)
    bad = dict(w)
    del bad['decoder/dense/kernel']
    with pytest.raises(B200TTSError) as e:
        TacoDecoderEngine(bad)
    assert e.value.code == -4
    eng = _engine(w)
    with pytest.raises(ValueError):
        eng.decode(np.zeros((1, 5, 100), np.float32))
    with pytest.raises(B200TTSError):
        eng.decode(np.zeros((1, 600, 512), np.float32), max_steps=4)        # Tx_max > 512


def test_encoder_and_postnet_vs_oracle_real_checkpoint():
    """SURVEY 8f rank 1: encoder (embedding -> 3 x conv+BN -> BiLSTM) and postnet on the GPU vs the oracle."""
    w = real_taco_weights()
    if w is None:
        pytest.skip('shipped Tacotron checkpoint not available on this box')
    eng = _engine(w)
    sent = sentences()['sentences']
    ids = np.zeros((3, 51), dtype=np.int32)
    lengths = np.array([51, 30, 44], dtype=np.int32)
    for b, k in enumerate(('241', '378', '407')):
        ids[b, :lengths[b]] = sent[k]['ids'][:lengths[b]]
    mem = eng.encode(ids, lengths).cpu().numpy()
    for b in range(3):
        ref = to.encoder(w, ids[b, :lengths[b]])
        np.testing.assert_allclose(mem[b, :lengths[b]], ref, rtol=0, atol=2e-5)
        assert np.all(mem[b, lengths[b]:] == 0)
    rs = np.random.RandomState(4)
    frames = rs.uniform(-5, 5, (2, 64, 80)).astype(np.float32)
    nsteps = np.array([64, 37], dtype=np.int32)
    mel = eng.postnet(frames, nsteps).cpu().numpy()
    for b in range(2):
        np.testing.assert_allclose(mel[b, :nsteps[b]], to.postnet(w, frames[b, :nsteps[b]]), rtol=0, atol=5e-5)


def test_synthesizer_and_pipeline_end_to_end(tmp_path):
    """Text -> mel (.npy contract of tacotron_synthesize.py:114-116) -> WaveRNN audio, all on the GPU (config 5 shape, tiny)."""
    import torch
    w = real_taco_weights()
    if w is None:
        pytest.skip('shipped Tacotron checkpoint not available on this box')
    from tacotronv2_wavernn_chinese_b200 import synth as wsynth
    from tacotronv2_wavernn_chinese_b200.engine import WaveRNNEngine
    from tacotronv2_wavernn_chinese_b200.pipeline import synthesize_batch
    from tacotronv2_wavernn_chinese_b200.tacotron.engine import TacoDecoderEngine
    from tacotronv2_wavernn_chinese_b200.tacotron.synthesizer import Synthesizer
    from tacotronv2_wavernn_chinese_b200.tacotron.text import Symbols
    s = sentences()
    syn = Synthesizer()
    syn.symbols = Symbols(s['symbols'])
    syn.engine = TacoDecoderEngine(w)
    syn.step = 206500
    texts = [syn.symbols.sequence_to_text(s['sentences'][k]['ids'][:-1]) for k in ('241', '378')]
    assert syn.symbols.text_to_sequence(texts[0]) == s['sentences']['241']['ids']
    mels, info = syn.mels(texts, seed=3, max_iters=700)
    for m, k in zip(mels, ('241', '378')):
        gt = s['sentences'][k]['frames']
        assert m.dtype == np.float32 and m.shape[1] == 80 and 0.0 <= m.min() and m.max() <= 1.0
        assert abs(m.shape[0] - gt) < 0.25 * gt, (m.shape, gt)              # stops near the ground-truth length
    path, apath = syn.synthesize(texts[0], str(tmp_path), 'abc', seed=3)
    saved = np.load(path)
    # (one sentence runs the 128-block decoder, the pair above one block per sentence: on this numerically chaotic checkpoint the
    #  two summation orders stop a few frames apart, like float32 vs float64 of the oracle -- tests/test_tacotron_oracle.py)
    gt0 = s['sentences']['241']['frames']
    assert path.endswith('step-206500-abc-mel-pred.npy') and saved.shape[1] == 80 and abs(saved.shape[0] - gt0) < 0.25 * gt0
    voc = WaveRNNEngine(wsynth.synth_state_dict(0), wsynth.DEFAULT_DIMS)
    waves, _ = synthesize_batch(syn, voc, texts, seed=3)
    for wv, m in zip(waves, mels):
        assert wv.dtype == np.float64 and wv.shape == ((m.shape[0] - 1) * 275,) and np.isfinite(wv).all() and wv[-1] == 0.0
    # a row of the padded batch == the same utterance vocoded alone (zero padding is what the reference does too)
    solo = voc.generate(torch.as_tensor(mels[1].T[None].copy()), seed=3, utterance_offset=1)['wave'].cpu().numpy()[0]
    np.testing.assert_array_equal(waves[1], solo)
    # ragged scheduler: 5 sentences in length-sorted chunks of 2 rows == the same sentences in one launch, bit for bit
    # (noise keyed by the global sentence index, batch-size-invariant arithmetic); and the sharded entry point with one rank
    from tacotronv2_wavernn_chinese_b200.pipeline import synthesize_sharded
    five = [syn.symbols.sequence_to_text(s['sentences'][k]['ids'][:-1]) for k in ('1', '2', '3', '4', '5')]
    one, m5 = synthesize_batch(syn, voc, five, seed=11)
    two, _ = synthesize_batch(syn, voc, five, seed=11, max_rows=2)
    shd, _ = synthesize_sharded(syn, voc, five, seed=11, max_rows=3)
    assert len({m.shape[0] for m in m5}) > 1                       # genuinely ragged
    for a, b, c3 in zip(one, two, shd):
        np.testing.assert_array_equal(a, b)
        np.testing.assert_array_equal(a, c3)
