"""Generation sessions without a GPU: the C-ABI refusals of the session entry points come before any CUDA call, and
pipeline.StreamingVocoder's scheduling (first-come-first-served admission, at most max_rows sessions per launch, requests
joining between launches, pieces that concatenate to each wave) against a stand-in engine."""
import ctypes

import numpy as np
import pytest

from tacotronv2_wavernn_chinese_b200 import pipeline

EINVAL = -1


def _lib():
    from tacotronv2_wavernn_chinese_b200 import build, _lib
    build.build_lib()
    return _lib.load(), _lib


def test_abi_refusals_before_any_cuda_call():
    lib, L = _lib()
    for name in ('b200tts_wavernn_session_open', 'b200tts_wavernn_session_destroy', 'b200tts_wavernn_session_info',
                 'b200tts_wavernn_session_run'):
        assert hasattr(lib, name) and name in L.SIGNATURES
    # the structs the sessions take keep their sizes (ABI 3)
    assert lib.b200tts_abi_version() == 3
    assert ctypes.sizeof(L.Rng) == 40 and ctypes.sizeof(L.GenOpts) == 80 and ctypes.sizeof(L.WaveRNNCfg) == 56
    rng = L.Rng()
    buf = (ctypes.c_float * 16)()
    h = ctypes.c_void_p()
    assert lib.b200tts_wavernn_session_open(None, buf, 21, ctypes.byref(rng), 1, ctypes.byref(h), None) == EINVAL
    assert not h.value and lib.b200tts_last_error()
    assert lib.b200tts_wavernn_session_open(None, None, 21, None, 1, None, None) == EINVAL
    pos = ctypes.c_int64()
    assert lib.b200tts_wavernn_session_info(None, ctypes.byref(pos), None, None) == EINVAL
    handles = (ctypes.c_void_p * 1)()
    assert lib.b200tts_wavernn_session_run(None, handles, 1, 100, None, None, None) == EINVAL
    assert lib.b200tts_wavernn_session_run(None, None, 1, 100, None, None, None) == EINVAL


def test_session_destroy_null_is_safe():
    lib, _ = _lib()
    lib.b200tts_wavernn_session_destroy(None)


# ---- StreamingVocoder against a stand-in engine -------------------------------------------------------------------------
HOP = 275


def _wave_of(uid, T):
    """The stand-in's whole wave of utterance `uid`: sample i is uid * 1e6 + i."""
    return uid * 1e6 + np.arange((T - 1) * HOP, dtype=np.float64)


class FakeSession:
    def __init__(self, T, uid):
        self.T, self.uid, self.position, self.closed = T, uid, 0, False
        self.steps, self.wave_len = T * HOP, (T - 1) * HOP

    @property
    def done(self):
        return self.position >= self.steps

    def close(self):
        assert not self.closed
        self.closed = True


class FakeEngine:
    """open_session / advance / check with the real engine's shapes and counts; records every call."""

    def __init__(self):
        self.opened, self.runs, self.checks = [], [], 0

    def open_session(self, mel, *, seed=0, utterance_id=0, mu_law=True):
        assert mel.ndim == 2 and mel.shape[0] == 80 and mel.shape[1] >= pipeline.MIN_FRAMES
        s = FakeSession(mel.shape[1], utterance_id)
        self.opened.append(utterance_id)
        return s

    def advance(self, sessions, max_steps):
        assert 1 <= len(sessions) <= 32 and len(set(map(id, sessions))) == len(sessions)
        assert not any(s.closed for s in sessions)
        self.runs.append([s.uid for s in sessions])
        out = []
        for s in sessions:
            k = min(max_steps, s.steps - s.position)
            w = max(0, min(s.position + k, s.wave_len) - s.position)
            piece = _wave_of(s.uid, s.T)[s.position:s.position + w]
            s.position += k
            out.append((np.zeros(k, np.int16), piece))
        return out

    def check(self):
        self.checks += 1


def _mel(T):
    return np.full((T, 80), 0.5, dtype=np.float32)


def _drain(sv, got, finished):
    while not sv.idle():
        for key, piece, fin in sv.step():
            assert key not in finished, 'a piece after the finished flag'
            got.setdefault(key, []).append(piece)
            if fin:
                finished.append(key)


def test_stream_admission_is_fifo_and_rows_are_bounded():
    eng = FakeEngine()
    sv = pipeline.StreamingVocoder(eng, seed=3, chunk_steps=1000, max_rows=4)
    frames = [21, 60, 25, 40, 33, 21, 50, 22, 45, 30]
    for k, T in enumerate(frames):
        sv.submit(k, _mel(T), 100 + k)
    got, finished = {}, []
    _drain(sv, got, finished)
    assert eng.opened == [100 + k for k in range(len(frames))]            # admitted in submission order
    assert max(len(r) for r in eng.runs) == 4 and all(1 <= len(r) <= 4 for r in eng.runs)
    assert eng.checks == len(eng.runs)
    assert sorted(finished) == list(range(len(frames)))
    for k, T in enumerate(frames):
        np.testing.assert_array_equal(np.concatenate(got[k]), _wave_of(100 + k, T))


def test_stream_request_submitted_mid_run_joins_at_the_next_step():
    eng = FakeEngine()
    sv = pipeline.StreamingVocoder(eng, chunk_steps=500, max_rows=32)
    sv.submit('a', _mel(30), 7)
    got, finished = {}, []
    for key, piece, fin in sv.step():
        got.setdefault(key, []).append(piece)
    assert eng.runs == [[7]]
    sv.submit('b', _mel(21), 8)
    for key, piece, fin in sv.step():
        got.setdefault(key, []).append(piece)
    assert eng.runs[1] == [7, 8]                                          # 'b' took a free row at once
    _drain(sv, got, finished)
    assert finished == ['b', 'a']                                         # the shorter one leaves first
    np.testing.assert_array_equal(np.concatenate(got['a']), _wave_of(7, 30))
    np.testing.assert_array_equal(np.concatenate(got['b']), _wave_of(8, 21))


def test_stream_full_rows_wait_and_short_mels_are_padded():
    eng = FakeEngine()
    sv = pipeline.StreamingVocoder(eng, chunk_steps=21 * HOP, max_rows=2)
    for k in range(5):
        sv.submit(k, _mel(5 + k), k)                                      # shorter than MIN_FRAMES: padded to 21 frames
    got, finished = {}, []
    _drain(sv, got, finished)
    assert eng.runs == [[0, 1], [2, 3], [4]]                              # one run each: the whole utterance fits a chunk
    assert finished == [0, 1, 2, 3, 4]
    for k in range(5):
        assert len(got[k]) == 1 and len(got[k][0]) == 20 * HOP


def test_stream_argument_checks():
    with pytest.raises(ValueError):
        pipeline.StreamingVocoder(FakeEngine(), max_rows=33)
    with pytest.raises(ValueError):
        pipeline.StreamingVocoder(FakeEngine(), chunk_steps=0)
    sv = pipeline.StreamingVocoder(FakeEngine())
    with pytest.raises(ValueError):
        sv.submit(0, np.zeros(80, np.float32), 0)
    assert sv.step() == [] and sv.idle()
