"""Pin of the speaking-rate bias (attention.py:163-165 / forward_attention.py:163-165, the branch the reference ships switched
off) against the reference's own code.

tests/golden/taco_rate_from_reference.npz: loop states of the oracle's biased runs of train.txt line 241 on the shipped
checkpoint, at delta in {-1, -0.3, -0.04, +0.04, +0.3, +1}, without the window (attention.py) and with it
(forward_attention.py), and what the reference's `ForwardLocationSensitiveAttention.__call__` of that file returns for each
with the branch switched on (oracle/ref_harness_taco_rate.py, oracle/make_golden_taco_rate.py).  The oracle of the bias is
oracle/tacotron_rate_oracle.py.
"""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import tacotron_oracle as to
from oracle import tacotron_rate_oracle as tro
from taco_common import real_taco_weights

F32 = np.float32


@pytest.fixture(scope='module')
def fixture():
    return np.load(os.path.join(GOLDEN, 'taco_rate_from_reference.npz'))


def test_rate_fixture_covers_both_files_every_delta_and_both_clip_ends(fixture):
    z = fixture
    deltas = {-1.0, -0.3, -0.04, 0.04, 0.3, 1.0}
    for win in (0, 1):
        assert {round(float(d), 2) for d in z['delta'][z['window'] == win]} == deltas
    biased = z['mu'] + z['delta']
    assert (biased <= 0).any() and (biased >= 1).any() and ((biased > 0) & (biased < 1)).any()   # both clip ends, and inside
    assert (z['step'] == 0).sum() == 2 * len(deltas) and (z['mu'][z['step'] == 0] == F32(0.5)).all()   # step 0: 0.5 + delta
    on = z['window'] == 1
    held = on & (z['ref_max_att'] == z['max_att'])
    advanced = on & (z['ref_max_att'] == z['max_att'] + 1)
    assert held.any() and advanced.any() and (held | advanced)[on].all()
    assert (advanced & (z['pos_rec'] == 9)).any()                                           # forced advance after 10 steps
    off = ~on
    assert len(set(z['ref_max_att'][off] - z['max_att'][off])) > 1                          # without the window: free argmax


def _attention_half(w, memory, keys, alpha, cum, mu, h2, mu_bias, window, max_att, pos_rec):
    """The attention half of oracle.decoder_step driven by a stored query, with the oracle's biased recursion."""
    Wq = w['decoder/Location_Sensitive_Attention/query_layer/kernel']
    v_a = w['decoder/Location_Sensitive_Attention/attention_variable_projection']
    b_a = w['decoder/Location_Sensitive_Attention/attention_bias']
    q = (h2 @ Wq).astype(F32)
    energy = (np.tanh(keys + q + to.location_features(w, cum) + b_a, dtype=F32) * v_a).sum(axis=1).astype(F32)
    e = np.exp(energy - energy.max(), dtype=F32)
    a = (e / e.sum(dtype=F32)).astype(F32)
    shift = np.concatenate([[F32(0)], alpha[:-1]]).astype(F32)
    mu_r = mu if not mu_bias else tro.biased_mu(mu, mu_bias)
    raw = (((F32(1) - mu_r) * alpha + mu_r * shift + F32(1e-10)) * a).astype(F32)
    if window:
        al, new_max, new_pos = to.attention_window(raw, max_att, pos_rec)
    else:
        al, new_max, new_pos = raw, int(np.argmax(raw)), pos_rec
    al = (al / al.sum(dtype=F32)).astype(F32)
    ctxv = (al[None, :] @ memory).astype(F32)
    new_mu = to._sigmoid((np.concatenate([ctxv, h2], axis=1) @ w['decoder/dense/kernel'] + w['decoder/dense/bias']).astype(F32))[0, 0]
    return dict(al=al, cum=(cum + a).astype(F32), ctx=ctxv[0], mu=new_mu, max_att=new_max, pos_rec=new_pos)


def test_biased_attention_step_matches_reference_statements(fixture):
    w = real_taco_weights()
    if w is None:
        pytest.skip('shipped Tacotron checkpoint not available on this box')
    z = fixture
    memory = z['memory']
    keys = (memory @ w['memory_layer/kernel']).astype(F32)
    for i in range(len(z['step'])):
        o = _attention_half(w, memory, keys, z['alpha'][i], z['cum'][i], F32(z['mu'][i]), z['query'][i][None], float(z['delta'][i]),
                            bool(z['window'][i]), int(z['max_att'][i]), int(z['pos_rec'][i]))
        where = (float(z['delta'][i]), int(z['window'][i]), int(z['step'][i]))
        assert (o['max_att'], o['pos_rec']) == (int(z['ref_max_att'][i]), int(z['ref_pos_rec'][i])), where
        np.testing.assert_allclose(o['al'], z['ref_alignments'][i], rtol=0, atol=1e-6, err_msg=str(where))
        np.testing.assert_allclose(o['cum'], z['ref_cum'][i], rtol=0, atol=1e-6, err_msg=str(where))
        np.testing.assert_allclose(o['ctx'], z['ref_context'][i], rtol=0, atol=1e-5, err_msg=str(where))
        assert o['mu'] == z['ref_mu'][i], where                                                 # the carried mu: unbiased sigmoid


def test_biased_mu_is_the_clip_of_one_float32_add():
    mu = np.float32(0.15)
    assert tro.biased_mu(mu, 0.0) == mu and tro.biased_mu(mu, -0.04) == np.float32(mu + np.float32(-0.04))
    assert tro.biased_mu(mu, -1.0) == 0 and tro.biased_mu(mu, 1.0) == 1 and tro.biased_mu(np.float32(0.5), 0.5) == 1
    assert tro.biased_mu(np.float32(1.0), -0.0) == 1 and tro.biased_mu(mu, 0.3).dtype == np.float32


def test_zero_bias_is_the_unbiased_oracle_bit_for_bit(fixture):
    """delta = 0 skips the add: decode and decoder_step are the unbiased ones, bit for bit.  And the biased expression itself
    at 0 reproduces the unbiased alignments of every fixture state exactly (clip(mu + 0, 0, 1) == mu for mu in [0, 1])."""
    w = real_taco_weights()
    if w is None:
        pytest.skip('shipped Tacotron checkpoint not available on this box')
    z = fixture
    memory = z['memory'][:20]
    for window in (False, True):
        a = to.decode(w, memory, seed=3, max_iters=25, window=window)
        b = tro.decode(w, memory, seed=3, max_iters=25, window=window, mu_bias=0.0)
        for k in ('frames', 'stop', 'alignments'):
            assert np.array_equal(a[k], b[k]), (window, k)
    keys = (z['memory'] @ w['memory_layer/kernel']).astype(F32)
    for i in range(0, len(z['step']), 7):
        args = (w, z['memory'], keys, z['alpha'][i], z['cum'][i], F32(z['mu'][i]), z['query'][i][None])
        win = (bool(z['window'][i]), int(z['max_att'][i]), int(z['pos_rec'][i]))
        plain = _attention_half(*args, 0.0, *win)
        mu_r = tro.biased_mu(F32(z['mu'][i]), 0.0)
        assert mu_r == F32(z['mu'][i])
        forced = _attention_half(*args[:5], mu_r, args[6], 0.0, *win)
        assert all(np.array_equal(plain[k], forced[k]) for k in plain)
