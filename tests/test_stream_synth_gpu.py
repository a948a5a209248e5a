"""Batched session opens and the streaming text-to-speech service on the GPU (engine.open_sessions, TacoDecoderEngine.
target_lengths, Synthesizer.decode_device, pipeline.StreamingSynthesizer): sessions opened in one batch from ragged mels are bit
for bit the sessions opened one by one; the 'taco' layout maps a postnet output exactly as the synthesizer's host statements do;
the device stop-token cut is the host rule; the service's pieces are the one-shot runs of its mels and its mels are the
synthesizer's.  Refusals launch nothing; batches leak no device memory.  Shipped vocoder checkpoint, Tacotron travel copy."""
import ctypes

import numpy as np
import pytest

from tacotronv2_wavernn_chinese_b200 import pipeline, synth
from taco_common import real_taco_weights, sentences
from test_wavernn_gpu import engine_for, torch_cuda  # noqa: F401  (torch_cuda is a fixture)

pytestmark = pytest.mark.gpu

HOP = 275


def _padded(mel_tf):
    """[T, feat] -> the [feat, max(T, 21)] mel a one-by-one open takes (zero frames past the end)."""
    T = mel_tf.shape[0]
    out = np.zeros((mel_tf.shape[1], max(T, pipeline.MIN_FRAMES)), dtype=np.float32)
    out[:, :T] = mel_tf.T
    return out


def _full_run(eng, sessions, S):
    """One run of every session to its end -> (labels, waves) as numpy lists."""
    pieces = eng.advance(sessions, S)
    eng.check()
    return [p[0].cpu().numpy() for p in pieces], [p[1].cpu().numpy() for p in pieces]


def _cut_run(eng, sessions, S):
    """Runs of 1 hop, 10 hops, then to S -> concatenated (labels, waves)."""
    labs, waves = [[] for _ in sessions], [[] for _ in sessions]
    for k in (HOP, 10 * HOP, S):
        for i, (lab, wave) in enumerate(eng.advance(sessions, k)):
            labs[i].append(lab.cpu().numpy())
            waves[i].append(wave.cpu().numpy())
    eng.check()
    assert all(s.done for s in sessions)
    return [np.concatenate(x) for x in labs], [np.concatenate(x) for x in waves]


# ---- 1. a batch open is the one-by-one opens ----------------------------------------------------------------------------
RAGGED = (1, 20, 21, 22, 37, 47)
T_MAX = 50                                   # > every frame count


@pytest.mark.parametrize('kernel,n', [('auto', 1), ('auto', 2), ('auto', 31), ('auto', 32),
                                      ('tc', 1), ('tc', 33), ('tc', 128), ('tc', 129), ('tc', 256)])
def test_batch_open_equals_single_opens(torch_cuda, kernel, n):
    eng, _ = engine_for('ckpt')
    seed = 5 + n
    mels = synth.synth_mels(900 + n, n, T_MAX)                                     # [n, 80, T_max]
    frames = [RAGGED[i % len(RAGGED)] for i in range(n)]
    ids = [int(x) for x in np.random.RandomState(n).randint(0, 2 ** 62, size=n, dtype=np.int64)]
    S = max(max(frames), pipeline.MIN_FRAMES) * HOP
    n0 = eng.launch_count
    batch = eng.open_sessions(torch_cuda.as_tensor(mels).cuda(), frames, seed=seed, utterance_ids=ids, kernel=kernel)
    assert eng.launch_count - n0 == 3                                               # whatever n is
    single = [eng.open_session(_padded(mels[i, :, :frames[i]].T), seed=seed, utterance_id=ids[i], kernel=kernel) for i in range(n)]
    for b, s in zip(batch, single):
        assert (b.position, b.steps, b.wave_len) == (s.position, s.steps, s.wave_len)
    ref_lab, ref_wave = _full_run(eng, single, S)
    if kernel == 'auto' and n > 1:               # full runs of the batch-opened sessions too, beside the cut runs below
        lab, wave = _full_run(eng, batch, S)
        batch = eng.open_sessions(torch_cuda.as_tensor(mels).cuda(), frames, seed=seed, utterance_ids=ids, kernel=kernel)
        for i in range(n):
            assert np.array_equal(lab[i], ref_lab[i]) and np.array_equal(wave[i], ref_wave[i]), f'row {i} ({frames[i]} frames)'
    lab, wave = _cut_run(eng, batch, S)
    for i in range(n):
        assert np.array_equal(lab[i], ref_lab[i]), f'labels of row {i} ({frames[i]} frames)'
        assert np.array_equal(wave[i], ref_wave[i]), f'wave of row {i} ({frames[i]} frames)'
    for s in batch + single:
        s.close()


# ---- Tacotron: one loaded synthesizer for the tests below -----------------------------------------------------------------
@pytest.fixture(scope='module')
def syn(torch_cuda):
    w = real_taco_weights()
    if w is None:
        pytest.skip('shipped Tacotron checkpoint not available on this box')
    from tacotronv2_wavernn_chinese_b200.tacotron.engine import TacoDecoderEngine
    from tacotronv2_wavernn_chinese_b200.tacotron.synthesizer import Synthesizer
    from tacotronv2_wavernn_chinese_b200.tacotron.text import Symbols
    s = Synthesizer()
    s.symbols = Symbols(sentences()['symbols'])
    s.engine = TacoDecoderEngine(w)
    s.max_iters = 120
    return s


def _texts(syn, n, first=0):
    """n train.txt sentences cut to 2 .. 25 tokens (so that their decodes stop at different steps, most within max_iters)."""
    ss = sentences()['sentences']
    keys = sorted(ss, key=int)
    out = []
    for i in range(first, first + n):
        ids = ss[keys[i % len(keys)]]['ids'][:-1]
        out.append(syn.symbols.sequence_to_text(ids[:2 + (7 * i) % 24]))
    return out


def _host_cut(stop, nsteps):
    """Synthesizer.mels' rule: first np.round(stop) == 1 below nsteps, else nsteps."""
    out = []
    for b in range(stop.shape[0]):
        r = np.round(stop[b, :nsteps[b]])
        out.append(int(np.argmax(r == 1)) if (r == 1).any() else int(nsteps[b]))
    return out


# ---- 2. the 'taco' layout --------------------------------------------------------------------------------------------------
def test_taco_layout_equals_the_host_statements(torch_cuda, syn):
    from tacotronv2_wavernn_chinese_b200.tacotron.synthesizer import MAX_ABS_VALUE, unit_mel
    eng, _ = engine_for('ckpt')
    texts = _texts(syn, 6)
    ids = [3, 4, 5, 6, 7, 8]
    post, lens = syn.decode_device(texts, ids, seed=2)
    frames = [int(x) for x in lens.cpu()]
    assert all(f >= 1 for f in frames) and len(set(frames)) > 1, frames
    ph = post.cpu().numpy()
    # Synthesizer.mels of the same batch (consecutive ids: the PHILOX stream) is the host conversion of this postnet output
    mels, _ = syn.mels(texts, seed=2, utterance_offset=3)
    for b in range(6):
        assert np.array_equal(mels[b], unit_mel(ph[b, :frames[b]]))
    S = max(max(frames), 21) * HOP
    for kernel in ('auto', 'tc'):
        batch = eng.open_sessions(post, frames, seed=9, utterance_ids=ids, kernel=kernel, layout='taco', max_abs_value=MAX_ABS_VALUE)
        single = [eng.open_session(_padded(mels[b]), seed=9, utterance_id=ids[b], kernel=kernel) for b in range(6)]
        ref_lab, ref_wave = _full_run(eng, single, S)
        lab, wave = _full_run(eng, batch, S)
        for b in range(6):
            assert np.array_equal(lab[b], ref_lab[b]) and np.array_equal(wave[b], ref_wave[b]), (kernel, b, frames[b])
        for s in batch + single:
            s.close()


# ---- 3. target_lengths -------------------------------------------------------------------------------------------------------
def test_target_lengths_is_the_host_rule(torch_cuda, syn):
    eng = syn.engine
    texts = _texts(syn, 8, first=10)
    seqs = [syn.symbols.text_to_sequence(t) for t in texts]
    tok = np.zeros((8, max(map(len, seqs))), dtype=np.int32)
    for b, s in enumerate(seqs):
        tok[b, :len(s)] = s
    ln = np.array([len(s) for s in seqs], dtype=np.int32)
    dec = eng.decode(eng.encode(tok, ln), ln, seed=1, max_steps=120)
    got = eng.target_lengths(dec['stop'], dec['nsteps']).cpu().numpy()
    assert list(got) == _host_cut(dec['stop'].cpu().numpy(), dec['nsteps'].cpu().numpy())
    # constructed rows: exactly 0.5 (np.round gives 0), never above 0.5, above 0.5 at step 0, a hit past nsteps, a failed decode
    stop = np.full((6, 10), 0.1, dtype=np.float32)
    stop[0, 2], stop[0, 6] = 0.5, 0.5000001
    stop[1, :] = 0.5
    stop[2, 0] = 0.75
    stop[3, 5] = 1.0
    stop[4, 9] = 0.51
    nsteps = np.array([10, 10, 10, 3, 10, -1], dtype=np.int32)
    got = eng.target_lengths(torch_cuda.as_tensor(stop), torch_cuda.as_tensor(nsteps)).cpu().numpy()
    assert list(got) == [6, 10, 0, 3, 9, -1]
    assert list(got[:5]) == _host_cut(stop[:5], nsteps[:5])


# ---- 4. the service end to end -----------------------------------------------------------------------------------------------
def _one_shot_waves(eng, mels, ids, seed, tc):
    """{i: one-shot wave of mels[i]} on the kernel family of the sessions: equal-length groups, <= 32 rows on the push kernel."""
    out, by_T = {}, {}
    for i, m in mels.items():
        by_T.setdefault(max(m.shape[0], 21), []).append(i)
    for T, idx in by_T.items():
        for c in range(0, len(idx), 256 if tc else 32):
            part = idx[c:c + (256 if tc else 32)]
            batch = np.stack([_padded(mels[i]) for i in part])
            w = eng.generate(batch, seed=seed, utterance_ids=[ids[i] for i in part], kernel='tc' if tc else 'auto')['wave']
            eng.check()
            assert eng.last_kernel() == ('wavernn_tc_kernel' if tc else 'wavernn_push_kernel')
            for k, i in enumerate(part):
                out[i] = w[k].cpu().numpy()
    return out


@pytest.mark.parametrize('max_rows', [32, 128])
@pytest.mark.parametrize('max_admit', [1, 4, None])
def test_service_end_to_end(torch_cuda, syn, max_rows, max_admit):
    eng, _ = engine_for('ckpt')
    n, seed = 40, 17
    texts = _texts(syn, n, first=20)
    ids = [1000 + i for i in range(n)]
    groups = []
    decode = syn.decode_device

    def recording(tx, ix, seed=0):
        groups.append((list(tx), list(ix)))
        return decode(tx, ix, seed=seed)

    syn.decode_device = recording
    try:
        ss = pipeline.StreamingSynthesizer(syn, eng, seed=seed, chunk_steps=10 * HOP, max_rows=max_rows, max_admit=max_admit)
        got, finished, mels, nxt = {}, [], {}, 0
        while nxt < n or not ss.idle():
            for _ in range(4):                                      # 4 new texts per step until all are in
                if nxt < n:
                    ss.submit(nxt, texts[nxt], ids[nxt])
                    nxt += 1
            out = ss.step()
            for key, piece, fin in out:
                if key not in mels:
                    mels[key] = ss.mel(key)
                assert key not in finished
                got.setdefault(key, []).append(piece)
                if fin:
                    finished.append(key)
            assert ss.active <= max_rows
    finally:
        syn.decode_device = decode
    assert sorted(finished) == list(range(n))
    assert all(len(ix) <= (max_admit or max_rows) for _tx, ix in groups)
    assert [i for _tx, ix in groups for i in ix] == ids                               # first come, first served
    # every mel is Synthesizer.mels of its admission group with the same (consecutive) ids
    for tx, ix in groups:
        ref, _ = syn.mels(tx, seed=seed, utterance_offset=ix[0])
        for t, i in zip(ref, ix):
            assert np.array_equal(mels[i - 1000], t), f'mel of request {i - 1000}'
    ref = _one_shot_waves(eng, {k: m for k, m in mels.items() if m.shape[0] > 0}, {k: ids[k] for k in mels}, seed, max_rows > 32)
    for k in range(n):
        w = np.concatenate(got[k])
        if mels[k].shape[0] == 0:
            assert len(w) == 0
        else:
            assert np.array_equal(w, ref[k]), f'request {k} ({mels[k].shape[0]} frames)'


# ---- 5. refusals and leaks ---------------------------------------------------------------------------------------------------
def _refused(eng, call):
    from tacotronv2_wavernn_chinese_b200._lib import B200TTSError
    n = eng.launch_count
    with pytest.raises(B200TTSError) as e:
        call()
    assert e.value.code == -1, str(e.value)                                   # B200TTS_EINVAL
    assert eng.launch_count == n, f'a refused call launched work: {e.value}'


def test_refusals(torch_cuda):
    from tacotronv2_wavernn_chinese_b200 import _lib
    from tacotronv2_wavernn_chinese_b200.engine import WaveRNNEngine
    eng, _ = engine_for('ckpt')
    mels = torch_cuda.as_tensor(synth.synth_mels(1, 3, 30)).cuda()
    ok = dict(seed=1, utterance_ids=[1, 2, 3])
    mol = WaveRNNEngine(synth.synth_state_dict(3, mode='MOL'), dict(synth.DEFAULT_DIMS, mode='MOL'))
    _refused(mol, lambda: mol.open_sessions(mels, [30, 30, 30], **ok))
    small = dict(synth.DEFAULT_DIMS, rnn_dims=256, fc_dims=256)
    narrow = WaveRNNEngine(synth.synth_state_dict(3, small), small)
    _refused(narrow, lambda: narrow.open_sessions(mels, [30, 30, 30], **ok))
    _refused(eng, lambda: eng.open_sessions(mels, [30, 0, 30], **ok))                # frames < 1
    _refused(eng, lambda: eng.open_sessions(mels, [30, 31, 30], **ok))               # frames > T_max
    big = torch_cuda.zeros(257, 80, 21, device='cuda')
    _refused(eng, lambda: eng.open_sessions(big, [21] * 257, seed=1, utterance_ids=list(range(257)), kernel='tc'))
    # through the C ABI: an unknown layout, a kernel other than AUTO / TC, a non-PHILOX rng, n = 0, a bad max_abs_value
    frames = (ctypes.c_int32 * 3)(30, 30, 30)
    out = (ctypes.c_void_p * 3)()
    rng = _lib.Rng()
    bad = _lib.Rng()
    bad.mode = _lib.RNG_EXT_EXPONENTIAL
    mp = ctypes.c_void_p(mels.data_ptr())
    call = lambda layout=0, mx=4.0, n=3, r=rng, kernel=0: _lib.check(eng.lib.b200tts_wavernn_session_open_batch(   # noqa: E731
        eng._h, mp, layout, mx, frames, n, 30, ctypes.byref(r), 1, kernel, out, None))
    _refused(eng, lambda: call(layout=2))
    _refused(eng, lambda: call(kernel=_lib.KERNEL_GRID))
    _refused(eng, lambda: call(r=bad))
    _refused(eng, lambda: call(n=0))
    _refused(eng, lambda: call(layout=1, mx=0.0))
    assert not any(out)
    mol.close()
    narrow.close()


def test_batches_leak_no_device_memory(torch_cuda):
    eng, _ = engine_for('ckpt')
    mels = torch_cuda.as_tensor(synth.synth_mels(4, 4, 60)).cuda()
    frames = [60, 21, 5, 44]

    def cycle(i, run):
        ss = eng.open_sessions(mels, frames, seed=1, utterance_ids=[4 * i + k for k in range(4)])
        if run:
            eng.advance(ss, 300)
        for s in reversed(ss) if i % 2 else ss:        # the batch's memory goes with whichever session closes last
            s.close()

    for i in range(3):                                  # warm up the allocator and the context's scratch
        cycle(i, True)
    torch_cuda.cuda.synchronize()
    free0, _ = torch_cuda.cuda.mem_get_info()
    for i in range(200):
        cycle(i, i % 20 == 0)
    torch_cuda.cuda.synchronize()
    free1, _ = torch_cuda.cuda.mem_get_info()
    eng.check()
    assert abs(free0 - free1) < 8 << 20, (free0, free1)
