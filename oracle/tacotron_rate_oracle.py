"""CPU oracle of the speaking-rate bias -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The reference's forward attention ships a speed control switched off (attention.py:163-165, forward_attention.py:163-165):

    if not self.is_training and False:
        delta_val = -0.04
        mu = tf.clip_by_value(mu + delta_val, 0.0, 1.0)

just before the forward recursion (:167).  Switched on, with delta per sentence, that rebinds only the local `mu` of one step:
the recursion sees the biased value, while the carried mu is the fresh sigmoid of [context | query] (:229).  In
oracle/tacotron_oracle.py's decoder_step the state's `mu` is read by the recursion and nowhere else, so a biased step is that
step on the state with `mu` replaced by biased_mu(mu, delta); the state it returns carries the unbiased new mu.

Pinned against the reference's own `__call__` with the branch switched on (oracle/ref_harness_taco_rate.py,
oracle/make_golden_taco_rate.py -> tests/golden/taco_rate_from_reference.npz, tests/test_tacotron_rate_pins.py).  At delta = 0
both functions below are exactly the unbiased oracle (no add at all).
"""
from __future__ import annotations

import numpy as np

try:
    from oracle import tacotron_oracle as to
except ImportError:                                  # run as a script from oracle/ (the make_golden_* generators)
    import tacotron_oracle as to

F32 = np.float32


def biased_mu(mu, mu_bias):
    """tf.clip_by_value(mu + delta, 0, 1) (attention.py:163-165): a float32 add rounded once, then min with 1 and max with 0
    (clip_by_value's order)."""
    return np.maximum(np.minimum(F32(mu) + F32(mu_bias), F32(1)), F32(0))


def decoder_step(w, memory, keys, x, m, st, zoneout=to.GRAPH_ASSUMPTIONS['zoneout'], modulate=None, mu_bias=0.0):
    """tacotron_oracle.decoder_step with the speaking-rate bias: the recursion uses biased_mu(st['mu'], mu_bias); the
    returned mu (intermediates and new state) is the unbiased sigmoid.  mu_bias = 0: the unbiased step itself."""
    if mu_bias:
        st = dict(st, mu=biased_mu(st['mu'], mu_bias))
    return to.decoder_step(w, memory, keys, x, m, st, zoneout, modulate)


def decode(w, memory, dropout_masks=None, seed=0, max_iters=2000, window=False, zoneout=to.GRAPH_ASSUMPTIONS['zoneout'],
           capture_states=(), mu_bias=0.0):
    """tacotron_oracle.decode with the speaking-rate bias at every step (decoder_step above); same arguments and returns, and
    the captured states hold the unbiased mu, as the reference's loop state does.  mu_bias = 0: tacotron_oracle.decode itself."""
    if not mu_bias:
        return to.decode(w, memory, dropout_masks, seed, max_iters, window, zoneout, capture_states)
    Tx = memory.shape[0]
    keys = (memory @ w['memory_layer/kernel']).astype(F32)
    U = w[to.P + 'decoder_LSTM/multi_rnn_cell/cell_0/decoder_LSTM_1/kernel'].shape[1] // 4
    rs = np.random.RandomState(seed)
    zeros = np.zeros((1, U), dtype=F32)
    alpha0 = np.zeros(Tx, dtype=F32)
    alpha0[0] = 1
    st = dict(c1=zeros, h1=zeros, c2=zeros, h2=zeros, ctx=np.zeros((1, memory.shape[1]), dtype=F32),
              alpha=alpha0, cum=alpha0.copy(), mu=F32(0.5))
    win = dict(max_att=0, pos_rec=0)
    x = np.zeros((1, 80), dtype=F32)
    frames, stops, aligns, masks, captured = [], [], [], [], {}

    def window_modulate(al):
        al, win['max_att'], win['pos_rec'] = to.attention_window(al, win['max_att'], win['pos_rec'])
        return al

    for step in range(max_iters):
        m = dropout_masks[step] if dropout_masks is not None else (rs.uniform(size=(2, 256)) >= to.GRAPH_ASSUMPTIONS['prenet_dropout_rate'])
        m = np.asarray(m, dtype=F32)
        masks.append(m)
        if step in capture_states:
            captured[step] = (x.copy(), {k: np.array(v, copy=True) for k, v in st.items()}, m.copy(), dict(win))
        out, st = decoder_step(w, memory, keys, x, m, st, zoneout, window_modulate if window else None, mu_bias)
        stop = to._sigmoid(out['stop_logit'])[0, 0]
        frames.append(out['frame'][0]); stops.append(stop); aligns.append(out['alignments'])
        x = out['frame']
        if stop > 0.5:
            break
    return dict(frames=np.stack(frames), stop=np.array(stops, dtype=F32), alignments=np.stack(aligns),
                n_steps=len(frames), masks=np.stack(masks), states=captured)
