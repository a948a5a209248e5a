"""Generation sessions on the tensor cores (engine.open_session(kernel='tc') / advance, pipeline.StreamingVocoder above 32
rows): a session generated in hop-multiple pieces is bit for bit its one-shot tensor-core run, however the steps are cut,
wherever its row sits among up to 256 sessions and whatever other generate calls run in between.  Refusals launch nothing;
sessions leak no device memory.  Shipped checkpoint."""
import ctypes

import numpy as np
import pytest

from tacotronv2_wavernn_chinese_b200 import pipeline, synth
from test_wavernn_gpu import engine_for, torch_cuda  # noqa: F401  (torch_cuda is a fixture)

pytestmark = pytest.mark.gpu

HOP = 275


def _one_shot(eng, mels, seed, ids):
    """One-shot tensor-core labels [B, S] and wave [B, (T-1)*hop] of equal-length mels [B, 80, T], row b keyed by ids[b]."""
    out = eng.generate(mels, seed=seed, utterance_ids=list(ids), kernel='tc')
    eng.check()
    assert eng.last_kernel() == 'wavernn_tc_kernel'
    return out['labels'].cpu().numpy(), out['wave'].cpu().numpy()


def _cuts(T):
    """Piece ends: 1-hop pieces for the first 10 frames, then 2, 10 and 40 hops, one exactly at (T-1)*hop and the last at S."""
    ends = [k * HOP for k in range(1, 11)]
    for k in (2, 10, 40):
        ends.append(ends[-1] + k * HOP)
    ends += [(T - 1) * HOP, T * HOP]
    return sorted({e for e in ends if 0 < e <= T * HOP})


@pytest.mark.parametrize('T,seed,uid', [(21, 11, 5), (60, 12, 2 ** 40 + 17)])
def test_pieces_concatenate_to_the_one_shot_run(torch_cuda, T, seed, uid):
    eng, _ = engine_for('ckpt')
    assert eng.max_session_rows == 256
    mel = synth.synth_mels(40 + T, 1, T)[0]
    ref_lab, ref_wave = _one_shot(eng, mel[None], seed, [uid])
    S, wave_len = T * HOP, (T - 1) * HOP
    cuts = _cuts(T)
    assert wave_len in cuts and cuts[-1] == S and all(c % HOP == 0 for c in cuts)
    labs, waves = [], []
    with eng.open_session(mel, seed=seed, utterance_id=uid, kernel='tc') as s:
        assert (s.position, s.steps, s.wave_len, s.done) == (0, S, wave_len, False)
        for end in cuts:
            pos = s.position
            n0 = eng.launch_count
            [(lab, wave)] = eng.advance([s], end - pos)
            eng.check()
            assert eng.launch_count - n0 == 2                         # step kernel, wave
            assert eng.last_kernel() == 'wavernn_tc_session_kernel'
            assert s.position == end and len(lab) == end - pos and len(wave) == max(0, min(end, wave_len) - pos)
            labs.append(lab.cpu().numpy())
            waves.append(wave.cpu().numpy())
        assert s.done
        [(lab, wave)] = eng.advance([s], HOP)                       # a finished session takes part with 0 steps
        assert len(lab) == 0 and len(wave) == 0 and s.position == S
    assert np.array_equal(np.concatenate(labs), ref_lab[0])
    assert np.array_equal(np.concatenate(waves), ref_wave[0])


# ---- row placement: up to 256 sessions of different lengths, opened at different runs ---------------------------------
LENGTHS = (21, 34, 47, 60)          # session i has LENGTHS[i % 4] frames
PLACE_SEED = 21


@pytest.fixture(scope='module')
def placement_refs(torch_cuda):
    """256 sessions' mels, ids and one-shot tensor-core labels / waves, from one kernel='tc' call per length."""
    eng, _ = engine_for('ckpt')
    rs = np.random.RandomState(5)
    ids = [int(x) for x in rs.randint(0, 2 ** 62, size=256, dtype=np.int64)]
    mels, labs, waves = [None] * 256, [None] * 256, [None] * 256
    for j, T in enumerate(LENGTHS):
        idx = list(range(j, 256, len(LENGTHS)))
        batch = synth.synth_mels(200 + T, len(idx), T)
        lab, wave = _one_shot(eng, batch, PLACE_SEED, [ids[i] for i in idx])
        for k, i in enumerate(idx):
            mels[i], labs[i], waves[i] = batch[k], lab[k], wave[k]
    return mels, ids, labs, waves


@pytest.mark.parametrize('n', [1, 33, 127, 128, 129, 200, 256])
def test_row_placement(torch_cuda, placement_refs, n):
    """Even sessions open first and run alone for a while; then every session runs, even and odd rows alternating, so both
    128-row groups hold rows at different frame offsets, and rows finish mid-run while their neighbours continue."""
    eng, _ = engine_for('ckpt')
    mels, ids, labs, waves = placement_refs
    sessions = [None] * n
    got_lab = [[] for _ in range(n)]
    got_wave = [[] for _ in range(n)]

    def run(idx, hops):
        for i, (lab, wave) in zip(idx, eng.advance([sessions[i] for i in idx], hops * HOP)):
            got_lab[i].append(lab.cpu().numpy())
            got_wave[i].append(wave.cpu().numpy())

    early = list(range(0, n, 2))
    for i in early:
        sessions[i] = eng.open_session(mels[i], seed=PLACE_SEED, utterance_id=ids[i], kernel='tc')
    run(early, 3)
    run(early, 4)
    for i in range(1, n, 2):
        sessions[i] = eng.open_session(mels[i], seed=PLACE_SEED, utterance_id=ids[i], kernel='tc')
    while not all(s.done for s in sessions):
        run(list(range(n)), 10)
    eng.check()
    assert eng.last_kernel() == 'wavernn_tc_session_kernel'
    for i in range(n):
        sessions[i].close()
        assert np.array_equal(np.concatenate(got_lab[i]), labs[i]), f'session {i} of {n}: labels differ from its one-shot run'
        assert np.array_equal(np.concatenate(got_wave[i]), waves[i]), f'session {i} of {n}: wave differs from its one-shot run'


def test_continuous_batching_is_bit_exact(torch_cuda):
    eng, _ = engine_for('ckpt')
    rs = np.random.RandomState(8)
    n, seed = 300, 13
    lengths = (21, 40, 57, 83, 101, 120)
    frames = [lengths[k] for k in rs.randint(0, len(lengths), size=n)]
    ids = [int(x) for x in rs.randint(0, 2 ** 62, size=n, dtype=np.int64)]
    mels = [synth.synth_mels(300 + i, 1, frames[i])[0] for i in range(n)]                # [80, T]
    sv = pipeline.StreamingVocoder(eng, seed=seed, chunk_steps=2750, max_rows=256)
    got, finished, nxt, runs = {}, [], 0, 0
    while nxt < n or not sv.idle():
        for _ in range(200 if runs == 0 else 12):                  # a burst, then submissions spread over the launches
            if nxt < n:
                sv.submit(nxt, mels[nxt].T, ids[nxt])
                nxt += 1
        for key, piece, fin in sv.step():
            assert key not in finished
            got.setdefault(key, []).append(piece)
            if fin:
                finished.append(key)
        assert sv.active <= 256
        runs += 1
    assert sorted(finished) == list(range(n))
    assert eng.last_kernel() == 'wavernn_tc_session_kernel'
    for T in lengths:
        idx = [i for i in range(n) if frames[i] == T]
        _, ref = _one_shot(eng, np.stack([mels[i] for i in idx]), seed, [ids[i] for i in idx])
        for k, i in enumerate(idx):
            assert np.array_equal(np.concatenate(got[i]), ref[k]), f'utterance {i} ({T} frames) differs from its one-shot run'


def test_generate_between_runs_leaves_the_session_unchanged(torch_cuda):
    eng, _ = engine_for('ckpt')
    mel = synth.synth_mels(3, 1, 30)[0]
    ref_lab, ref_wave = _one_shot(eng, mel[None], 4, [77])
    labs, waves = [], []
    kernels = set()
    with eng.open_session(mel, seed=4, utterance_id=77, kernel='tc') as s:
        k = 0
        while not s.done:
            [(lab, wave)] = eng.advance([s], 5 * HOP)
            labs.append(lab.cpu().numpy())
            waves.append(wave.cpu().numpy())
            eng.check()
            # every step kernel family in between: push, wide grid, tensor cores (each overwrites the context's scratch)
            eng.generate(synth.synth_mels(4, 1 + k % 3, 45), seed=k, max_steps=300, want_wave=False)
            kernels.add(eng.last_kernel())
            eng.generate(synth.synth_mels(5, 40, 21), seed=k, max_steps=50, want_wave=False)
            kernels.add(eng.last_kernel())
            eng.generate(synth.synth_mels(6, 130 + k, 21), seed=k, max_steps=60, want_wave=False, kernel='tc')
            kernels.add(eng.last_kernel())
            eng.check()
            k += 1
    assert kernels == {'wavernn_push_kernel', 'wavernn_grid_kernel', 'wavernn_tc_kernel'}
    assert np.array_equal(np.concatenate(labs), ref_lab[0])
    assert np.array_equal(np.concatenate(waves), ref_wave[0])


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
    mel = synth.synth_mels(1, 1, 21)[0]
    # a MOL context, and a model the tensor-core kernel cannot run
    mol = WaveRNNEngine(synth.synth_state_dict(3, mode='MOL'), dict(synth.DEFAULT_DIMS, mode='MOL'))
    _refused(mol, lambda: mol.open_session(mel, kernel='tc'))
    small = dict(synth.DEFAULT_DIMS, rnn_dims=256, fc_dims=256)
    narrow = WaveRNNEngine(synth.synth_state_dict(3, small), small)
    assert narrow.max_session_rows == 32
    _refused(narrow, lambda: narrow.open_session(mel, kernel='tc'))
    # noise other than PHILOX
    m = torch_cuda.as_tensor(mel).cuda().contiguous()
    rng = _lib.Rng()
    rng.mode = _lib.RNG_EXT_EXPONENTIAL
    h = ctypes.c_void_p()
    _refused(eng, lambda: _lib.check(eng.lib.b200tts_wavernn_session_open_kernel(
        eng._h, ctypes.c_void_p(m.data_ptr()), 21, ctypes.byref(rng), 1, _lib.KERNEL_TC, ctypes.byref(h), None)))
    assert not h.value
    # run arguments: max_steps not a multiple of hop, more than 256 sessions, push and tensor-core sessions mixed
    tc = [eng.open_session(mel, utterance_id=i, kernel='tc') for i in range(257)]
    push = eng.open_session(mel, utterance_id=999)
    _refused(eng, lambda: eng.advance(tc[:1], 1000))
    _refused(eng, lambda: eng.advance(tc[:3], HOP + 1))
    _refused(eng, lambda: eng.advance(tc, HOP))
    _refused(eng, lambda: eng.advance([tc[0], push], HOP))
    _refused(eng, lambda: eng.advance([push, tc[0]], HOP))
    assert all(s.position == 0 for s in tc) and push.position == 0
    eng.advance(tc[:256], HOP)                                              # 256 are accepted
    eng.check()
    assert eng.last_kernel() == 'wavernn_tc_session_kernel'
    assert all(s.position == HOP for s in tc[:256]) and tc[256].position == 0
    for s in tc + [push]:
        s.close()
    mol.close()
    narrow.close()


def test_sessions_leak_no_device_memory(torch_cuda):
    eng, _ = engine_for('ckpt')
    mel = synth.synth_mels(2, 1, 60)[0]
    for i in range(3):                                              # warm up the allocator and the context's scratch
        with eng.open_session(mel, utterance_id=i, kernel='tc') as s:
            eng.advance([s], 2 * HOP)
    torch_cuda.cuda.synchronize()
    free0, _ = torch_cuda.cuda.mem_get_info()
    for i in range(200):
        s = eng.open_session(mel, utterance_id=i, kernel='tc')
        if i % 20 == 0:
            eng.advance([s], 2 * HOP)
        s.close()
    torch_cuda.cuda.synchronize()
    free1, _ = torch_cuda.cuda.mem_get_info()
    eng.check()
    assert abs(free0 - free1) < 8 << 20, (free0, free1)
