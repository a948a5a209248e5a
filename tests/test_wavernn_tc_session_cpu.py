"""Tensor-core generation sessions without a GPU: the new C-ABI entry points refuse bad arguments before any CUDA call, and
pipeline.StreamingVocoder, given an engine that takes 256 sessions per launch, admits up to 256 rows first come first served,
opens tensor-core sessions only above 32 rows and requires a hop-multiple chunk there."""
import ctypes

import numpy as np
import pytest

from tacotronv2_wavernn_chinese_b200 import pipeline

EINVAL = -1
HOP = 275


def _lib():
    from tacotronv2_wavernn_chinese_b200 import build, _lib
    build.build_lib()
    return _lib.load(), _lib


def test_abi_entry_points_and_refusals_before_any_cuda_call():
    lib, L = _lib()
    for name in ('b200tts_wavernn_session_open_kernel', 'b200tts_wavernn_session_max_rows'):
        assert hasattr(lib, name) and name in L.SIGNATURES
    assert lib.b200tts_abi_version() == 3
    rng = L.Rng()
    buf = (ctypes.c_float * 16)()
    h = ctypes.c_void_p()
    for kernel in (L.KERNEL_AUTO, L.KERNEL_TC, L.KERNEL_GRID):
        assert lib.b200tts_wavernn_session_open_kernel(None, buf, 21, ctypes.byref(rng), 1, kernel, ctypes.byref(h), None) == EINVAL
        assert not h.value and lib.b200tts_last_error()
    assert lib.b200tts_wavernn_session_max_rows(None) == 32        # no context: the push kernel's limit


class FakeSession:
    def __init__(self, T, uid, kernel):
        self.T, self.uid, self.kernel, self.position, self.closed = T, uid, kernel, 0, False
        self.steps, self.wave_len = T * HOP, (T - 1) * HOP

    @property
    def done(self):
        return self.position >= self.steps

    def close(self):
        assert not self.closed
        self.closed = True


def _wave_of(uid, T):
    return uid * 1e6 + np.arange((T - 1) * HOP, dtype=np.float64)


class FakeTcEngine:
    """An engine whose library takes 256 sessions per run: tensor-core sessions (max_steps a multiple of hop) above 32 rows."""
    hop = HOP
    max_session_rows = 256

    def __init__(self):
        self.opened, self.kernels, self.runs = [], [], []

    def open_session(self, mel, *, seed=0, utterance_id=0, mu_law=True, kernel='auto'):
        assert kernel in ('auto', 'tc')
        self.opened.append(utterance_id)
        self.kernels.append(kernel)
        return FakeSession(mel.shape[1], utterance_id, kernel)

    def advance(self, sessions, max_steps):
        kinds = {s.kernel for s in sessions}
        assert len(kinds) == 1 and len(set(map(id, sessions))) == len(sessions)
        assert 1 <= len(sessions) <= (256 if kinds == {'tc'} else 32)
        assert kinds != {'tc'} or max_steps % HOP == 0
        self.runs.append([s.uid for s in sessions])
        out = []
        for s in sessions:
            k = min(max_steps, s.steps - s.position)
            w = max(0, min(s.position + k, s.wave_len) - s.position)
            out.append((np.zeros(k, np.int16), _wave_of(s.uid, s.T)[s.position:s.position + w]))
            s.position += k
        return out


def _drain(sv, got, finished, bound):
    while not sv.idle():
        for key, piece, fin in sv.step():
            assert key not in finished
            got.setdefault(key, []).append(piece)
            if fin:
                finished.append(key)
        assert sv.active <= bound


def test_fifo_admission_up_to_256_rows():
    eng = FakeTcEngine()
    sv = pipeline.StreamingVocoder(eng, seed=1, chunk_steps=10 * HOP, max_rows=256)
    rs = np.random.RandomState(3)
    frames = [int(x) for x in rs.randint(21, 90, size=300)]
    for k, T in enumerate(frames):
        sv.submit(k, np.full((T, 80), 0.5, np.float32), 1000 + k)
    got, finished = {}, []
    _drain(sv, got, finished, 256)
    assert eng.opened == [1000 + k for k in range(len(frames))]
    assert max(len(r) for r in eng.runs) == 256 and len(eng.runs[0]) == 256
    assert set(eng.kernels) == {'tc'}
    assert sorted(finished) == list(range(len(frames)))
    for k, T in enumerate(frames):
        np.testing.assert_array_equal(np.concatenate(got[k]), _wave_of(1000 + k, T))


@pytest.mark.parametrize('rows,kernel', [(1, 'auto'), (32, 'auto'), (33, 'tc'), (256, 'tc')])
def test_tensor_cores_only_above_32_rows(rows, kernel):
    eng = FakeTcEngine()
    sv = pipeline.StreamingVocoder(eng, chunk_steps=2750, max_rows=rows)
    for k in range(rows + 3):
        sv.submit(k, np.full((21, 80), 0.5, np.float32), k)
    _drain(sv, {}, [], rows)
    assert set(eng.kernels) == {kernel}


def test_chunk_must_be_a_hop_multiple_above_32_rows():
    eng = FakeTcEngine()
    with pytest.raises(ValueError, match='multiple of hop'):
        pipeline.StreamingVocoder(eng, chunk_steps=1000, max_rows=33)
    pipeline.StreamingVocoder(eng, chunk_steps=1000, max_rows=32)          # the push kernel cuts anywhere
    pipeline.StreamingVocoder(eng, chunk_steps=4 * HOP, max_rows=256)
    with pytest.raises(ValueError):
        pipeline.StreamingVocoder(eng, chunk_steps=2750, max_rows=257)
