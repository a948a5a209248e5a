"""Speaking-rate biases through the host layers without a GPU, against stand-ins: the service gives one admission ONE Tacotron
batch with per-row biases in admission order and passes no keyword when every bias is 0; bad biases are refused at submit, in
the Synthesizer and by the C ABI before any CUDA call; synthesize_batch and synthesize_sharded
pass the biases through."""
import ctypes

import numpy as np
import pytest
import torch

from tacotronv2_wavernn_chinese_b200 import pipeline
from tacotronv2_wavernn_chinese_b200.tacotron.engine import mu_bias_array
from tacotronv2_wavernn_chinese_b200.tacotron.synthesizer import Synthesizer
from tacotronv2_wavernn_chinese_b200.tacotron.text import Symbols

BAD = [float('nan'), float('inf'), -float('inf'), 1.0001, -1.5, 2.0]


class RateSynth:
    """decode_device / mels stand-in that records the keyword arguments of every call."""

    def __init__(self):
        self.symbols = Symbols(['_', '~', 'a', 'b'])
        self.calls = []

    def decode_device(self, texts, ids, seed=0, **kw):
        self.calls.append((list(ids), kw))
        post = torch.zeros(len(texts), 40, 80)
        return post, torch.full((len(texts),), 30, dtype=torch.int32)

    def mels(self, texts, seed=0, utterance_offset=0, **kw):
        self.calls.append((utterance_offset, kw))
        return [np.full((25 + b, 80), 0.5, np.float32) for b in range(len(texts))], {}


class Engine:
    hop = 275
    max_session_rows = 32

    def open_sessions(self, mels, frames, *, seed=0, utterance_ids, kernel='auto', layout='taco'):
        return [Session() for _ in frames]

    def advance(self, sessions, max_steps):
        for s in sessions:
            s.done = True
        return [(None, np.zeros(3)) for _ in sessions]


class Session:
    done = False

    def close(self):
        pass


class Voc:
    hop = 275

    def generate(self, mels, seed=0, utterance_ids=None, kernel='auto', utt_frames=None, pack=None):
        return {'wave': torch.zeros(mels.shape[0], (mels.shape[2] - 1) * self.hop, dtype=torch.float64)}

    def check(self):
        pass


def test_mixed_biases_make_one_batch_with_per_row_biases_in_admission_order():
    synth = RateSynth()
    ss = pipeline.StreamingSynthesizer(synth, Engine(), max_rows=8)
    for k, d in enumerate([0.0, -0.04, 0.1, 0.3]):
        ss.submit(k, 'a b a', 10 + k, mu_bias=d)
    ss.step()
    assert len(synth.calls) == 1
    ids, kw = synth.calls[0]
    assert ids == [10, 11, 12, 13] and set(kw) == {'mu_bias'}
    np.testing.assert_array_equal(kw['mu_bias'], np.array([0.0, -0.04, 0.1, 0.3], np.float32))


def test_all_zero_admission_passes_no_keyword():
    synth = RateSynth()
    ss = pipeline.StreamingSynthesizer(synth, Engine(), max_rows=8)
    ss.submit(0, 'a b', 0)
    ss.submit(1, 'a', 1, mu_bias=0.0)
    ss.submit(2, 'b', 2, mu_bias=-0.0)
    ss.step()
    assert synth.calls == [([0, 1, 2], {})]


@pytest.mark.parametrize('bad', BAD + [[0.1], np.zeros(2), 'fast'])
def test_bad_bias_refused_at_submit(bad):
    synth = RateSynth()
    ss = pipeline.StreamingSynthesizer(synth, Engine())
    with pytest.raises(ValueError):
        ss.submit(0, 'a b', 0, mu_bias=bad)
    assert ss.pending == 0 and synth.calls == []


def test_mu_bias_array():
    assert mu_bias_array(None, 3) is None and mu_bias_array(0.0, 3) is None and mu_bias_array([0, -0.0, 0], 3) is None
    np.testing.assert_array_equal(mu_bias_array(0.2, 3), np.full(3, 0.2, np.float32))
    b = mu_bias_array([0, -1, 1], 3)
    assert b.dtype == np.float32 and b.flags['C_CONTIGUOUS'] and list(b) == [0, -1, 1]
    for bad in BAD:
        with pytest.raises(ValueError):
            mu_bias_array(bad, 2)
        with pytest.raises(ValueError):
            mu_bias_array([0.0, bad], 2)
    for wrong_count in ([0.1, 0.2], np.zeros((3, 1)), []):
        with pytest.raises(ValueError):
            mu_bias_array(wrong_count, 3)


class RefusingEngine:
    """Fails the test if anything reaches the device."""

    def __getattr__(self, name):
        raise AssertionError(f'{name} called although the biases were bad')


@pytest.mark.parametrize('bad', [float('nan'), 1.5, [0.1, 0.2, 0.3]])
def test_synthesizer_refuses_bad_bias_before_any_launch(bad):
    syn = Synthesizer()
    syn.symbols = Symbols(['_', '~', 'a', 'b'])
    syn.engine = RefusingEngine()
    with pytest.raises(ValueError):
        syn.mels(['a b', 'b'], mu_bias=bad)
    with pytest.raises(ValueError):
        syn.decode_device(['a b', 'b'], [0, 1], mu_bias=bad)
    with pytest.raises(ValueError):
        syn.synthesize('a b', '/nonexistent/never-created', 'x', mu_bias=bad if np.ndim(bad) == 0 else [0.1, 0.2])


def test_synthesize_batch_and_sharded_pass_biases_through():
    synth = RateSynth()
    pipeline.synthesize_batch(synth, Voc(), ['a', 'b', 'a b'], mu_bias=[0.1, 0.0, -0.04], utterance_offset=5)
    pipeline.synthesize_sharded(synth, Voc(), ['a', 'b', 'a b'], mu_bias=0.2)
    pipeline.synthesize_batch(synth, Voc(), ['a', 'b'], mu_bias=0.0)
    pipeline.synthesize_sharded(synth, Voc(), ['a', 'b'])
    (o1, k1), (o2, k2), (o3, k3), (o4, k4) = synth.calls
    assert o1 == 5 and list(k1['mu_bias']) == list(np.float32([0.1, 0.0, -0.04]))
    assert o2 == 0 and list(k2['mu_bias']) == [np.float32(0.2)] * 3
    assert k3 == {} and k4 == {}
    with pytest.raises(ValueError):
        pipeline.synthesize_batch(synth, Voc(), ['a', 'b'], mu_bias=[0.1])
    assert len(synth.calls) == 4
    gen = pipeline.synthesize_stream(synth, None, 'a b', utterance_id=7, mu_bias=0.3)
    assert next(gen).shape == (25, 80)
    assert synth.calls[-1][0] == 7 and list(synth.calls[-1][1]['mu_bias']) == [np.float32(0.3)]


def test_abi_refuses_bad_biases_before_any_cuda_call():
    from tacotronv2_wavernn_chinese_b200 import _lib, build
    build.build_lib()
    lib = _lib.load()
    assert 'b200tts_taco_decode_biased' in _lib.SIGNATURES
    buf = (ctypes.c_float * 16)()
    d = _lib.TacoDropout()

    def call(bias, B=2):
        arr = None if bias is None else (ctypes.c_float * len(bias))(*bias)
        return lib.b200tts_taco_decode_biased(None, buf, buf, B, 5, ctypes.byref(d), 10, 0, arr, None, buf, buf, None, buf, None)

    assert call(None) == -1 and 'mu_bias' in lib.b200tts_last_error().decode()
    assert call([0.0, 0.0]) == -1                                        # null context: refused before anything else
    assert lib.b200tts_taco_decode_biased(None, None, None, 1, 5, None, 10, 0, None, None, None, None, None, None, None) == -1
