"""Generation sessions on the GPU (engine.open_session / advance, pipeline.StreamingVocoder): an utterance generated in pieces
is bit for bit its one-shot run, however the steps are cut, whichever sessions share a launch and whatever other generate calls
run in between.  Refusals launch nothing; sessions leak no device memory.  Shipped checkpoint."""
import ctypes

import numpy as np
import pytest

from tacotronv2_wavernn_chinese_b200 import pipeline, synth
from test_wavernn_gpu import engine_for, torch_cuda  # noqa: F401  (torch_cuda is a fixture)

pytestmark = pytest.mark.gpu

HOP = 275


def _solo(eng, mel, seed, uid):
    """One-shot labels [S] and wave [(T-1)*hop] of mel [80, T] (one row: the push kernel)."""
    out = eng.generate(mel[None], seed=seed, utterance_ids=[uid])
    eng.check()
    return out['labels'][0].cpu().numpy(), out['wave'][0].cpu().numpy()


def _cuts(T):
    """Piece ends: 1-step pieces for the first 300 steps, then 7, 275, 1000, 4096 and the rest, plus an end on a frame boundary,
    one inside the fade region, one exactly at (T-1)*hop and one at S."""
    S, wave_len = T * HOP, (T - 1) * HOP
    ends = list(range(1, 301))
    for k in (7, 275, 1000, 4096):
        ends.append(ends[-1] + k)
    ends += [10 * HOP, wave_len - 20 * HOP + 1234, wave_len, S]
    return sorted({e for e in ends if 0 < e <= S})


@pytest.mark.parametrize('T,seed,uid', [(21, 11, 5), (60, 12, 2 ** 40 + 17)])
def test_pieces_concatenate_to_the_one_shot_run(torch_cuda, T, seed, uid):
    eng, _ = engine_for('ckpt')
    mel = synth.synth_mels(40 + T, 1, T)[0]
    ref_lab, ref_wave = _solo(eng, mel, seed, uid)
    S, wave_len = T * HOP, (T - 1) * HOP
    cuts = _cuts(T)
    fade0 = wave_len - 20 * HOP
    assert any(c % HOP for c in cuts) and any(c % HOP == 0 and c < wave_len for c in cuts)
    assert any(fade0 < c < wave_len for c in cuts) and wave_len in cuts and cuts[-1] == S
    labs, waves = [], []
    with eng.open_session(mel, seed=seed, utterance_id=uid) as s:
        assert (s.position, s.steps, s.wave_len, s.done) == (0, S, wave_len, False)
        for end in cuts:
            pos = s.position
            n0 = eng.launch_count
            [(lab, wave)] = eng.advance([s], end - pos)
            eng.check()
            assert eng.launch_count - n0 == 3                         # exchange init, step kernel, wave
            assert s.position == end and len(lab) == end - pos and len(wave) == max(0, min(end, wave_len) - pos)
            labs.append(lab.cpu().numpy())
            waves.append(wave.cpu().numpy())
        assert s.done
        [(lab, wave)] = eng.advance([s], 100)                       # a finished session takes part with 0 steps
        assert len(lab) == 0 and len(wave) == 0 and s.position == S
    assert np.array_equal(np.concatenate(labs), ref_lab)
    assert np.array_equal(np.concatenate(waves), ref_wave)


def test_continuous_batching_is_bit_exact(torch_cuda):
    eng, _ = engine_for('ckpt')
    rs = np.random.RandomState(7)
    n = 40
    frames = rs.randint(21, 61, size=n)
    ids = [int(x) for x in rs.randint(0, 2 ** 62, size=n, dtype=np.int64)]
    mels = [synth.synth_mels(100 + i, 1, int(frames[i]))[0].T for i in range(n)]          # [T, 80], as Tacotron hands them
    seed = 9
    sv = pipeline.StreamingVocoder(eng, seed=seed, chunk_steps=1000, max_rows=32)
    got, finished, nxt, runs = {}, [], 0, 0
    while nxt < n or not sv.idle():
        for _ in range(10 if runs == 0 else 3):                    # submissions spread over the first launches
            if nxt < n:
                sv.submit(nxt, mels[nxt], ids[nxt])
                nxt += 1
        assert sv.active + min(sv.pending, 32 - sv.active) <= 32
        for key, piece, fin in sv.step():
            assert key not in finished
            got.setdefault(key, []).append(piece)
            if fin:
                finished.append(key)
        runs += 1
    assert sorted(finished) == list(range(n))
    for i in range(n):
        _, ref = _solo(eng, mels[i].T.copy(), seed, ids[i])
        assert np.array_equal(np.concatenate(got[i]), ref), f'utterance {i} ({frames[i]} frames) differs from its solo run'


def test_generate_between_runs_leaves_the_session_unchanged(torch_cuda):
    eng, _ = engine_for('ckpt')
    mel = synth.synth_mels(3, 1, 30)[0]
    ref_lab, ref_wave = _solo(eng, mel, 4, 77)
    other = synth.synth_mels(4, 3, 45)
    labs, waves = [], []
    with eng.open_session(mel, seed=4, utterance_id=77) as s:
        k = 0
        while not s.done:
            [(lab, wave)] = eng.advance([s], 1500)
            labs.append(lab.cpu().numpy())
            waves.append(wave.cpu().numpy())
            eng.check()
            eng.generate(other[: 1 + k % 3], seed=k)               # overwrites the context's scratch (tables, exchange buffers)
            eng.generate(synth.synth_mels(5, 40, 21), seed=k, max_steps=50, want_wave=False)   # and another step kernel
            eng.check()
            k += 1
    assert np.array_equal(np.concatenate(labs), ref_lab)
    assert np.array_equal(np.concatenate(waves), ref_wave)


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
    # a MOL context, and a model the push kernel cannot run
    mol = WaveRNNEngine(synth.synth_state_dict(3, mode='MOL'), dict(synth.DEFAULT_DIMS, mode='MOL'))
    _refused(mol, lambda: mol.open_session(mel))
    small = dict(synth.DEFAULT_DIMS, rnn_dims=256, fc_dims=256)
    narrow = WaveRNNEngine(synth.synth_state_dict(3, small), small)
    _refused(narrow, lambda: narrow.open_session(mel))
    # noise other than PHILOX, and T < 21
    m = torch_cuda.as_tensor(mel).cuda().contiguous()
    rng = _lib.Rng()
    rng.mode = _lib.RNG_EXT_EXPONENTIAL
    h = ctypes.c_void_p()
    _refused(eng, lambda: _lib.check(eng.lib.b200tts_wavernn_session_open(eng._h, ctypes.c_void_p(m.data_ptr()), 21, ctypes.byref(rng),
                                                                          1, ctypes.byref(h), None)))
    assert not h.value
    _refused(eng, lambda: eng.open_session(synth.synth_mels(1, 1, 20)[0]))
    # run arguments: n outside 1..32, max_steps < 1, the same session twice, a session of another context
    sessions = [eng.open_session(mel, utterance_id=i) for i in range(33)]
    _refused(eng, lambda: eng.advance([], 10))
    _refused(eng, lambda: eng.advance(sessions, 10))
    _refused(eng, lambda: eng.advance(sessions[:1], 0))
    _refused(eng, lambda: eng.advance([sessions[0], sessions[1], sessions[0]], 10))
    other = WaveRNNEngine(synth.synth_state_dict(3), synth.DEFAULT_DIMS)
    foreign = other.open_session(mel)
    _refused(eng, lambda: eng.advance([sessions[0], foreign], 10))
    assert all(s.position == 0 for s in sessions) and foreign.position == 0
    for s in sessions:
        s.close()
    other.close()                                                  # frees `foreign` with its context
    foreign.close()
    mol.close()
    narrow.close()


def test_sessions_leak_no_device_memory(torch_cuda):
    eng, _ = engine_for('ckpt')
    mel = synth.synth_mels(2, 1, 60)[0]
    for i in range(3):                                              # warm up the allocator and the context's scratch
        with eng.open_session(mel, utterance_id=i) as s:
            eng.advance([s], 300)
    torch_cuda.cuda.synchronize()
    free0, _ = torch_cuda.cuda.mem_get_info()
    for i in range(200):
        s = eng.open_session(mel, utterance_id=i)
        if i % 20 == 0:
            eng.advance([s], 300)
        s.close()
    torch_cuda.cuda.synchronize()
    free1, _ = torch_cuda.cuda.mem_get_info()
    eng.check()
    assert abs(free0 - free1) < 8 << 20, (free0, free1)
