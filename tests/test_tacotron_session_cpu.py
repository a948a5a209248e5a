"""Tacotron decoder sessions without a GPU: the C-ABI refusals of b200tts_taco_session_*, which come before any CUDA call, and
pipeline.StreamingSynthesizer(decode_steps=k) against stand-ins: decodes admitted first come, first served under max_rows
(decodes plus vocoder sessions) and the 128-session bound, one decoder launch per step advancing each decode by at most k
steps, one finish and one vocoder open per step that finishes decodes, empty mels, and the decode_steps check."""
import ctypes

import numpy as np
import pytest
import torch

from tacotronv2_wavernn_chinese_b200 import pipeline
from tacotronv2_wavernn_chinese_b200.tacotron.text import Symbols

HOP = 275
EINVAL = -1


def _lib():
    from tacotronv2_wavernn_chinese_b200 import build, _lib
    build.build_lib()
    return _lib.load(), _lib


class _FakeSession(ctypes.Structure):
    """Host memory standing in for a b200tts_taco_session, whose first member is its context: the run refusals read nothing
    else of it."""
    _fields_ = [('ctx', ctypes.c_void_p), ('pad', ctypes.c_char * 248)]


def test_abi_refusals_before_any_cuda_call():
    lib, L = _lib()
    assert lib.b200tts_abi_version() == 3
    ctx = ctypes.c_void_p(0x1000)           # never dereferenced: every call below is refused before it is
    mem = (ctypes.c_float * 16)()
    d = L.TacoDropout()
    out = (ctypes.c_void_p * 200)()
    lens = (ctypes.c_int32 * 200)(*([4] * 200))
    F = ctypes.POINTER(ctypes.c_float)

    def open_(n=2, Tx=4, dropout=d, max_steps=100, bias=None, lengths=lens, c=ctx):
        b = None if bias is None else (ctypes.c_float * len(bias))(*bias)
        return lib.b200tts_taco_session_open_batch(c, mem, lengths, n, Tx, ctypes.byref(dropout), None, max_steps, 0,
                                                   None if b is None else ctypes.cast(b, F), out, None)

    assert open_(c=None) == EINVAL and lib.b200tts_last_error()
    assert open_(n=0) == EINVAL and open_(n=129) == EINVAL
    assert open_(Tx=0) == EINVAL and open_(Tx=513) == EINVAL
    assert open_(max_steps=0) == EINVAL
    ext = L.TacoDropout()
    ext.mode = 1
    ext.d_masks = ctypes.addressof(mem)
    assert open_(dropout=ext) == EINVAL and b'PHILOX' in lib.b200tts_last_error()
    assert open_(lengths=(ctypes.c_int32 * 2)(4, 5)) == EINVAL and open_(lengths=(ctypes.c_int32 * 2)(0, 4)) == EINVAL
    for bad in (float('nan'), float('inf'), 1.5, -1.01):
        assert open_(bias=[0.0, bad]) == EINVAL and b'mu_bias[1]' in lib.b200tts_last_error()
    assert not any(out[:4])

    a, b, other = _FakeSession(ctx=0x1000), _FakeSession(ctx=0x1000), _FakeSession(ctx=0x2000)
    P = ctypes.POINTER(ctypes.c_void_p)

    def run(sess, n=None, max_steps=8, c=ctx):
        hs = (ctypes.c_void_p * max(len(sess), 1))(*[ctypes.addressof(s) for s in sess])
        return lib.b200tts_taco_session_run(c, ctypes.cast(hs, P), len(sess) if n is None else n, max_steps, None)

    assert run([a], c=None) == EINVAL
    assert run([a], n=0) == EINVAL and run([a] * 129) == EINVAL
    assert run([a, b, a]) == EINVAL and b'twice' in lib.b200tts_last_error()
    assert run([a, other]) == EINVAL and b'another context' in lib.b200tts_last_error()
    assert run([a, b], max_steps=0) == EINVAL and b'max_steps' in lib.b200tts_last_error()
    assert lib.b200tts_taco_session_run(ctx, None, 1, 8, None) == EINVAL
    buf = (ctypes.c_float * 4)()
    assert lib.b200tts_taco_session_outputs(None, 1, 4, buf, buf, buf, None) == EINVAL
    hs = (ctypes.c_void_p * 2)(ctypes.addressof(a), ctypes.addressof(a))
    assert lib.b200tts_taco_session_outputs(ctypes.cast(hs, P), 2, 4, buf, buf, buf, None) == EINVAL
    pos = ctypes.c_int32()
    assert lib.b200tts_taco_session_info(None, ctypes.byref(pos), None, None) == EINVAL
    lib.b200tts_taco_session_destroy(None)          # null-safe


# ---- the sliced service against stand-ins ---------------------------------------------------------------------------------
def _steps_of(text):
    """The stand-in decoder's length of a text: 3 steps per token; 'silent' decodes one step whose stop fires (an empty mel)."""
    return 1 if text == 'silent' else 3 * len(text.split(' '))


class FakeDecode:
    def __init__(self, text, uid):
        self.uid, self.total, self.position, self.closed = uid, _steps_of(text), 0, False
        self.empty = text == 'silent'

    @property
    def done(self):
        return self.position >= self.total

    def close(self):
        assert not self.closed
        self.closed = True


class FakeTacoEngine:
    def __init__(self):
        self.launches = []          # [(ids, steps)] per advance_decodes

    def advance_decodes(self, sessions, n):
        assert 1 <= len(sessions) <= 128 and not any(s.closed for s in sessions)
        self.launches.append(([s.uid for s in sessions], n))
        for s in sessions:
            s.position = min(s.total, s.position + n)


class FakeSynth:
    def __init__(self):
        self.symbols = Symbols(['_', '~', 'a', 'b', 'silent'])
        self.engine = FakeTacoEngine()
        self.opens, self.finishes, self.biases = [], [], []

    def open_decodes(self, texts, ids, seed=0, mu_bias=None):
        self.opens.append(list(ids))
        self.biases.append(mu_bias)
        return [FakeDecode(t, u) for t, u in zip(texts, ids)]

    def finish_decodes(self, sessions):
        assert all(s.done and not s.closed for s in sessions)
        self.finishes.append([s.uid for s in sessions])
        T = max(s.position for s in sessions)
        post = torch.zeros(len(sessions), T, 80)
        for b, s in enumerate(sessions):
            post[b] = float(s.uid % 5) - 2
        return post, torch.tensor([0 if s.empty else s.position for s in sessions], dtype=torch.int32)


class FakeVocSession:
    def __init__(self, T, uid):
        self.T, self.uid, self.position, self.closed = max(T, pipeline.MIN_FRAMES), uid, 0, False
        self.steps, self.wave_len = self.T * HOP, (self.T - 1) * HOP

    @property
    def done(self):
        return self.position >= self.steps

    def close(self):
        self.closed = True


def _wave_of(uid, T):
    return uid * 1e6 + np.arange((max(T, pipeline.MIN_FRAMES) - 1) * HOP, dtype=np.float64)


class FakeEngine:
    hop = HOP

    def __init__(self, max_session_rows=32):
        self.max_session_rows = max_session_rows
        self.opens, self.runs = [], []

    def open_sessions(self, mels, frames, *, seed=0, utterance_ids, kernel='auto', layout='feat_t'):
        assert layout == 'taco' and mels.shape[0] == len(frames) == len(utterance_ids)
        self.opens.append(list(utterance_ids))
        return [FakeVocSession(f, u) for f, u in zip(frames, utterance_ids)]

    def advance(self, sessions, max_steps):
        self.runs.append([s.uid for s in sessions])
        out = []
        for s in sessions:
            k = min(max_steps, s.steps - s.position)
            w = max(0, min(s.position + k, s.wave_len) - s.position)
            out.append((np.zeros(k, np.int16), _wave_of(s.uid, s.T)[s.position:s.position + w]))
            s.position += k
        return out

    def check(self):
        pass


def _text(n):
    return ' '.join(['a', 'b'] * (n // 2) + ['a'] * (n % 2))


@pytest.mark.parametrize('max_rows,max_admit,k', [(4, None, 5), (6, 2, 1), (32, None, 16), (3, 1, 100)])
def test_sliced_admission_capacity_and_pieces(max_rows, max_admit, k):
    synth, eng = FakeSynth(), FakeEngine()
    ss = pipeline.StreamingSynthesizer(synth, eng, seed=5, chunk_steps=1000, max_rows=max_rows, max_admit=max_admit,
                                       decode_steps=k)
    words = [7, 20, 9, 14, 8, 11, 25, 7, 13, 10]
    for i, n in enumerate(words):
        ss.submit(i, _text(n), 100 + i)
    got, finished, first_piece, step = {}, [], {}, 0
    launches_before = 0
    while not ss.idle():
        out = ss.step()
        step += 1
        # at most one decoder launch per step, each decode advanced by at most k steps
        assert len(synth.engine.launches) - launches_before <= 1
        launches_before = len(synth.engine.launches)
        assert ss.decoding + ss.active <= max_rows and ss.decoding <= 128
        for key, piece, fin in out:
            assert key not in finished
            first_piece.setdefault(key, step)
            got.setdefault(key, []).append(piece)
            if fin:
                finished.append(key)
    assert [u for o in synth.opens for u in o] == [100 + i for i in range(len(words))]     # first come, first served
    assert all(1 <= len(o) <= (max_admit or max_rows) for o in synth.opens)
    assert all(n == k for _ids, n in synth.engine.launches)
    assert synth.biases == [None] * len(synth.opens)
    assert eng.opens == synth.finishes                 # one finish and one vocoder open per step that finishes decodes
    assert sorted(finished) == list(range(len(words)))
    for i, n in enumerate(words):
        np.testing.assert_array_equal(np.concatenate(got[i]), _wave_of(100 + i, 3 * n))
    assert ss.idle() and ss.pending == 0 and ss.active == 0 and ss.decoding == 0


def test_first_piece_in_the_step_the_decode_finishes():
    synth, eng = FakeSynth(), FakeEngine()
    ss = pipeline.StreamingSynthesizer(synth, eng, chunk_steps=1000, max_rows=8, decode_steps=4)
    ss.submit('a', _text(3), 1)          # 9 steps: done in the third slice
    ss.submit('b', _text(1), 2)          # 3 steps: done in the first
    outs = [ss.step() for _ in range(3)]
    assert [k for k, _p, _f in outs[0]] == ['b']
    assert [k for k, _p, _f in outs[1]] == ['b']
    assert [k for k, _p, _f in outs[2]] == ['b', 'a']
    assert synth.engine.launches == [([1, 2], 4), ([1], 4), ([1], 4)]
    np.testing.assert_array_equal(ss.mel('a'), np.full((9, 80), (1 % 5 - 2 + 4) / 8, np.float32))


def test_empty_mels_and_biases():
    synth, eng = FakeSynth(), FakeEngine()
    ss = pipeline.StreamingSynthesizer(synth, eng, chunk_steps=1000, max_rows=8, decode_steps=2)
    ss.submit('x', 'silent', 7)
    ss.submit('y', _text(1), 8, mu_bias=0.25)
    out = ss.step()
    assert [(k, len(p), f) for k, p, f in out] == [('x', 0, True)]
    assert ss.mel('x').shape == (0, 80)
    assert synth.biases == [[0.0, 0.25]]
    assert eng.opens == []                  # nothing to vocode yet: 'y' needs two slices
    out = ss.step()
    assert [k for k, _p, _f in out] == ['y'] and eng.opens == [[8]]


def test_decode_capacity_is_128_sessions():
    synth, eng = FakeSynth(), FakeEngine(max_session_rows=256)
    ss = pipeline.StreamingSynthesizer(synth, eng, chunk_steps=HOP * 10, max_rows=256, decode_steps=1)
    for i in range(200):
        ss.submit(i, _text(5), i)
    ss.step()
    assert ss.decoding == 128 and len(synth.opens[0]) == 128 and ss.pending == 72


def test_decode_steps_validation():
    synth, eng = FakeSynth(), FakeEngine()
    for bad in (0, -3):
        with pytest.raises(ValueError, match='decode_steps'):
            pipeline.StreamingSynthesizer(synth, eng, decode_steps=bad)
    assert pipeline.StreamingSynthesizer(synth, eng).decode_steps is None
