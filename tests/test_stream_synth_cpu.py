"""pipeline.StreamingSynthesizer without a GPU, against a stand-in synthesizer and engine: first-come-first-served admission
under the max_rows and max_admit caps, exactly one Tacotron batch and one batched session open per admitting step, pieces in
admission order that concatenate to each request's wave, finish and idle(); texts over the encoder's bound refused at submit;
the tensor-core hop-multiple rule.  Also the C-ABI refusals of the new entry points, which come before any CUDA call."""
import ctypes

import numpy as np
import pytest
import torch

from tacotronv2_wavernn_chinese_b200 import pipeline
from tacotronv2_wavernn_chinese_b200.tacotron.engine import MAX_TOKENS
from tacotronv2_wavernn_chinese_b200.tacotron.synthesizer import unit_mel
from tacotronv2_wavernn_chinese_b200.tacotron.text import Symbols

HOP = 275
EINVAL = -1


def _frames_of(text):
    """The stand-in decoder's length of a text: 3 frames per token (0 for the text 'silent', whose stop fires at once)."""
    return 0 if text == 'silent' else 3 * len(text.split(' '))


def _post_value(uid, t):
    return (uid % 7) - 3.0 + 0.001 * t


class FakeSynth:
    def __init__(self, ms=200):
        self.symbols = Symbols(['_', '~', 'a', 'b', 'silent'])
        self.ms, self.batches = ms, []

    def decode_device(self, texts, ids, seed=0):
        self.batches.append(list(ids))
        post = torch.zeros(len(texts), self.ms, 80)
        for b, uid in enumerate(ids):
            post[b] = torch.tensor([_post_value(uid, t) for t in range(self.ms)])[:, None]
        return post, torch.tensor([_frames_of(t) for t in texts], dtype=torch.int32)


def _wave_of(uid, T):
    return uid * 1e6 + np.arange((max(T, pipeline.MIN_FRAMES) - 1) * HOP, dtype=np.float64)


class FakeSession:
    def __init__(self, T, uid):
        self.T, self.uid, self.position, self.closed = max(T, pipeline.MIN_FRAMES), uid, 0, False
        self.steps, self.wave_len = self.T * HOP, (self.T - 1) * HOP

    @property
    def done(self):
        return self.position >= self.steps

    def close(self):
        assert not self.closed
        self.closed = True


class FakeEngine:
    hop = HOP

    def __init__(self, max_session_rows=32):
        self.max_session_rows = max_session_rows
        self.opens, self.runs, self.checks = [], [], 0

    def open_sessions(self, mels, frames, *, seed=0, utterance_ids, kernel='auto', layout='feat_t'):
        assert layout == 'taco' and mels.shape[0] == len(frames) == len(utterance_ids) and mels.shape[2] == 80
        assert all(1 <= f <= mels.shape[1] for f in frames)
        self.opens.append((list(utterance_ids), kernel))
        return [FakeSession(f, u) for f, u in zip(frames, utterance_ids)]

    def advance(self, sessions, max_steps):
        assert 1 <= len(sessions) <= self.max_session_rows and not any(s.closed for s in sessions)
        self.runs.append([s.uid for s in sessions])
        out = []
        for s in sessions:
            k = min(max_steps, s.steps - s.position)
            w = max(0, min(s.position + k, s.wave_len) - s.position)
            out.append((np.zeros(k, np.int16), _wave_of(s.uid, s.T)[s.position:s.position + w]))
            s.position += k
        return out

    def check(self):
        self.checks += 1


def _text(n):
    return ' '.join(['a', 'b'] * (n // 2) + ['a'] * (n % 2))


def _drain(ss, got, finished, order):
    steps = 0
    while not ss.idle():
        out = ss.step()
        steps += 1
        order.append([k for k, _p, _f in out])
        for key, piece, fin in out:
            assert key not in finished, 'a piece after the finished flag'
            got.setdefault(key, []).append(piece)
            if fin:
                finished.append(key)
    return steps


@pytest.mark.parametrize('max_rows,max_admit', [(4, None), (4, 1), (32, 3), (6, 2)])
def test_admission_caps_and_pieces(max_rows, max_admit):
    synth, eng = FakeSynth(), FakeEngine()
    ss = pipeline.StreamingSynthesizer(synth, eng, seed=5, chunk_steps=1000, max_rows=max_rows, max_admit=max_admit)
    words = [7, 20, 9, 14, 8, 11, 25, 7, 13, 10]
    for k, n in enumerate(words):
        ss.submit(k, _text(n), 100 + k)
    assert ss.pending == len(words) and not ss.idle()
    got, finished, order = {}, [], []
    _drain(ss, got, finished, order)
    admitted = [u for b in synth.batches for u in b]
    assert admitted == [100 + k for k in range(len(words))]                      # first come, first served
    assert all(1 <= len(b) <= (max_admit or max_rows) for b in synth.batches)
    assert [ids for ids, _k in eng.opens] == synth.batches                        # one open per Tacotron batch
    assert all(kernel == 'auto' for _ids, kernel in eng.opens)
    assert max(len(r) for r in eng.runs) <= max_rows
    assert eng.checks == len(eng.runs)
    for step_keys, run in zip(order, eng.runs):
        assert step_keys == [u - 100 for u in run]                                # pieces in admission order
    assert sorted(finished) == list(range(len(words)))
    for k, n in enumerate(words):
        np.testing.assert_array_equal(np.concatenate(got[k]), _wave_of(100 + k, 3 * n))
    assert ss.idle() and ss.pending == 0 and ss.active == 0


def test_one_tacotron_batch_and_one_open_per_admitting_step():
    synth, eng = FakeSynth(), FakeEngine()
    ss = pipeline.StreamingSynthesizer(synth, eng, chunk_steps=500, max_rows=3)
    for k in range(5):
        ss.submit(k, _text(10), k)
    ss.step()
    assert synth.batches == [[0, 1, 2]] and len(eng.opens) == 1 and eng.runs == [[0, 1, 2]]
    ss.step()                                                   # no free row: no Tacotron batch, no open
    assert len(synth.batches) == 1 and len(eng.opens) == 1 and len(eng.runs) == 2
    ss.submit(9, _text(10), 9)
    got, finished, order = {}, [], []
    _drain(ss, got, finished, order)
    assert [u for b in synth.batches for u in b] == [0, 1, 2, 3, 4, 9]
    assert len(synth.batches) == len(eng.opens)


def test_mel_of_a_request_and_empty_mels():
    synth, eng = FakeSynth(), FakeEngine()
    ss = pipeline.StreamingSynthesizer(synth, eng, chunk_steps=HOP * 30, max_rows=8)
    ss.submit('x', _text(9), 40)
    ss.submit('s', 'silent', 41)
    with pytest.raises(KeyError):
        ss.mel('x')
    out = ss.step()
    assert [k for k, _p, _f in out] == ['x', 's'] and out[1][2] and len(out[1][1]) == 0
    assert eng.opens == [([40], 'auto')]                       # the empty mel opens no session
    post = np.array([[_post_value(40, t)] * 80 for t in range(27)], dtype=np.float32)
    np.testing.assert_array_equal(ss.mel('x'), unit_mel(post))
    assert ss.mel('s').shape == (0, 80)
    got, finished, order = {}, [], []
    _drain(ss, got, finished, order)
    with pytest.raises(KeyError):                              # dropped the step after its last piece
        ss.step()
        ss.mel('x')


def test_overlong_text_refused_at_submit():
    synth, eng = FakeSynth(), FakeEngine()
    ss = pipeline.StreamingSynthesizer(synth, eng)
    ss.submit(0, _text(MAX_TOKENS - 1), 0)                      # + the end mark: exactly MAX_TOKENS symbols
    with pytest.raises(ValueError):
        ss.submit(1, _text(MAX_TOKENS), 1)
    assert ss.pending == 1 and synth.batches == []


def test_tensor_core_rows_need_hop_multiple_chunks():
    synth = FakeSynth()
    eng = FakeEngine(max_session_rows=256)
    with pytest.raises(ValueError):
        pipeline.StreamingSynthesizer(synth, eng, chunk_steps=2750 + 1, max_rows=33)
    with pytest.raises(ValueError):
        pipeline.StreamingSynthesizer(synth, eng, max_rows=257)
    with pytest.raises(ValueError):
        pipeline.StreamingSynthesizer(synth, FakeEngine(), max_rows=33)     # a push-only engine
    with pytest.raises(ValueError):
        pipeline.StreamingSynthesizer(synth, eng, max_admit=0)
    pipeline.StreamingSynthesizer(synth, eng, chunk_steps=2751, max_rows=32)
    ss = pipeline.StreamingSynthesizer(synth, eng, chunk_steps=HOP * 10, max_rows=64)
    ss.submit(0, _text(12), 3)
    ss.step()
    assert eng.opens == [([3], 'tc')]


def _lib():
    from tacotronv2_wavernn_chinese_b200 import _lib, build
    build.build_lib()
    return _lib.load(), _lib


def test_abi_refusals_before_any_cuda_call():
    lib, L = _lib()
    for name in ('b200tts_wavernn_session_open_batch', 'b200tts_taco_target_lengths'):
        assert hasattr(lib, name) and name in L.SIGNATURES
    rng = L.Rng()
    buf = (ctypes.c_float * 16)()
    frames = (ctypes.c_int32 * 2)(21, 21)
    out = (ctypes.c_void_p * 2)()
    assert lib.b200tts_wavernn_session_open_batch(None, buf, 0, 4.0, frames, 2, 21, ctypes.byref(rng), 1, 0, out, None) == EINVAL
    assert lib.b200tts_last_error() and not out[0] and not out[1]
    assert lib.b200tts_wavernn_session_open_batch(None, None, 0, 4.0, None, 2, 21, None, 1, 0, None, None) == EINVAL
    assert lib.b200tts_taco_target_lengths(None, None, 1, 10, None, None) == EINVAL
    assert lib.b200tts_taco_target_lengths(buf, buf, 0, 10, buf, None) == EINVAL
