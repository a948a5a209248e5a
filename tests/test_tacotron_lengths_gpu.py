"""The Tacotron encoder, decoders and postnet at every sentence length the API accepts (up to kTacoMaxTx = 512 tokens) and
over the postnet's 2000 frames, on synthetic weights with the shipped shapes (tacotron_hparams.py), so the file runs without
the checkpoint.

LENGTHS covers the encoder's 8-step conv tile (kConvTile), the 31-tap location window, the two summation branches of
taco_grid_kernel's energy stage (Txp <= 128 and Txp >= 132), the midpoint 256 and the maximum.  A free run of 48 steps keeps
the attention near the start of the sentence (forward attention advances at most one token per step), so each decoder is also
run teacher-forced from loop states whose cumulated and previous alignments are spread over the whole sentence: then the
energy of every position, the last ones included, reaches the frame, the stop token and the alignments.

References: float64 restatements of the encoder and postnet below (oracle/tacotron_oracle.encoder / postnet, which the graph
pins hold to the reference), and the float32 oracle's decoder loop and step (oracle/tacotron_oracle.decode / decoder_step,
oracle/tacotron_gta_oracle.decode_gta)."""
import numpy as np
import pytest

from oracle import tacotron_gta_oracle as gta
from oracle import tacotron_oracle as to
from taco_common import real_taco_weights, sentences, synth_taco_weights

pytestmark = pytest.mark.gpu

LENGTHS = [1, 2, 3, 5, 8, 9, 16, 17, 31, 32, 127, 128, 129, 132, 255, 256, 257, 509, 511, 512]
TXMAX = 512
STEPS = 48           # free-running steps
FORCED = 8           # teacher-forced steps from spread loop states
F32, F64 = np.float32, np.float64
STOP_BIAS = 'decoder/stop_token_projection/projection_stop_token_projection/bias'
ENC = 'encoder_convolutions/conv_layer_{}_encoder_convolutions'
POST = 'postnet_convolutions/conv_layer_{}_postnet_convolutions'
LSTM = 'encoder_LSTM/bidirectional_rnn/{0}/encoder_{0}_LSTM/'
ZONEOUT = float(F32(to.GRAPH_ASSUMPTIONS['zoneout']))
CLIP = [float(F32(v)) for v in to.GRAPH_ASSUMPTIONS['output_clip']]


# ---------------------------------------------------------------- synthetic weights with the shipped shapes

def _conv_bn(w, rs, scope, cin, cout, k=5):
    s = np.sqrt(3.0 / (k * cin))                                     # unit-variance outputs for unit-variance inputs
    w[scope + '/conv1d/kernel'] = rs.uniform(-s, s, (k, cin, cout)).astype(F32)
    w[scope + '/conv1d/bias'] = rs.uniform(-0.1, 0.1, cout).astype(F32)
    bn = scope + '/batch_normalization/'
    w[bn + 'gamma'] = rs.uniform(0.5, 1.5, cout).astype(F32)
    w[bn + 'beta'] = rs.uniform(-0.3, 0.3, cout).astype(F32)
    w[bn + 'moving_mean'] = rs.uniform(-0.3, 0.3, cout).astype(F32)
    w[bn + 'moving_variance'] = rs.uniform(0.5, 2.0, cout).astype(F32)


def synth_full_weights(seed=7, stop_bias=-3.0):
    """synth_taco_weights(seed) for the decoder, plus the encoder (embedding [191, 128], 3 convs k5 128 -> 256 -> 256 -> 256
    with batch norm, BiLSTM kernels [512, 1024]) and the postnet (5 convs k5 80 -> 256 -> ... -> 256 with batch norm,
    projection [256, 80]).  stop_bias None keeps the generator's own stop bias (the stop rule fires within a few steps);
    -3 keeps the stop token below 0.5, so a run lasts all its steps."""
    w = synth_taco_weights(seed)
    if stop_bias is not None:
        w[STOP_BIAS] = np.array([stop_bias], F32)
    rs = np.random.RandomState(1000 + seed)
    w['inputs_embedding'] = rs.uniform(-1, 1, (191, 128)).astype(F32)
    for i, cin in ((1, 128), (2, 256), (3, 256)):
        _conv_bn(w, rs, ENC.format(i), cin, 256)
    s = 1.0 / np.sqrt(512)
    for d in ('fw', 'bw'):
        w[LSTM.format(d) + 'kernel'] = rs.uniform(-s, s, (512, 1024)).astype(F32)
        w[LSTM.format(d) + 'bias'] = rs.uniform(-0.1, 0.1, 1024).astype(F32)
    for i, cin in ((1, 80), (2, 256), (3, 256), (4, 256), (5, 256)):
        _conv_bn(w, rs, POST.format(i), cin, 256)
    s = 1.0 / np.sqrt(256)
    w['postnet_projection/projection_postnet_projection/kernel'] = rs.uniform(-s, s, (256, 80)).astype(F32)
    w['postnet_projection/projection_postnet_projection/bias'] = rs.uniform(-0.1, 0.1, 80).astype(F32)
    return w


# ---------------------------------------------------------------- float64 restatements of the encoder and the postnet

def _block64(x, w, scope, act):
    """conv1d 'same' (k taps, zero padding at both ends of THIS sentence) -> act -> batch norm with moving statistics."""
    K, b = w[scope + '/conv1d/kernel'].astype(F64), w[scope + '/conv1d/bias'].astype(F64)
    k, T, h = K.shape[0], x.shape[0], (K.shape[0] - 1) // 2
    xp = np.zeros((T + k - 1, x.shape[1]))
    xp[h:h + T] = x
    y = act(sum(xp[j:j + T] @ K[j] for j in range(k)) + b)
    bn = {n: w[scope + '/batch_normalization/' + n].astype(F64) for n in ('gamma', 'beta', 'moving_mean', 'moving_variance')}
    return (y - bn['moving_mean']) * (bn['gamma'] / np.sqrt(bn['moving_variance'] + 1e-3)) + bn['beta']


def _sig(v):
    return 1.0 / (1.0 + np.exp(-v))


def encoder64(w, ids):
    """embedding -> 3 x [conv k5 -> ReLU -> BN] -> zoneout BiLSTM 2 x 256 (output = the un-zoned new h), in float64."""
    x = w['inputs_embedding'].astype(F64)[np.asarray(ids)]
    for i in (1, 2, 3):
        x = _block64(x, w, ENC.format(i), lambda v: np.maximum(v, 0.0))
    T, z = x.shape[0], ZONEOUT
    out = np.zeros((T, 512))
    for d, order in ((0, range(T)), (1, range(T - 1, -1, -1))):
        K = w[LSTM.format(('fw', 'bw')[d]) + 'kernel'].astype(F64)
        bias = w[LSTM.format(('fw', 'bw')[d]) + 'bias'].astype(F64)
        c, h = np.zeros(256), np.zeros(256)
        for t in order:
            i_, j_, f_, o_ = np.split(np.concatenate([x[t], h]) @ K + bias, 4)
            cn = _sig(f_ + 1.0) * c + _sig(i_) * np.tanh(j_)
            hn = _sig(o_) * np.tanh(cn)
            c, h = (1 - z) * cn + z * c, (1 - z) * hn + z * h
            out[t, 256 * d:256 * (d + 1)] = hn
    return out


def postnet64(w, dec):
    """clip -> 4 x [conv k5 -> tanh -> BN] -> [conv k5 -> BN] -> projection -> residual add -> clip, in float64."""
    d = np.clip(dec.astype(F64), *CLIP)
    x = d
    for i in (1, 2, 3, 4):
        x = _block64(x, w, POST.format(i), np.tanh)
    x = _block64(x, w, POST.format(5), lambda v: v)
    r = x @ w['postnet_projection/projection_postnet_projection/kernel'].astype(F64) \
        + w['postnet_projection/projection_postnet_projection/bias'].astype(F64)
    return np.clip(d + r, *CLIP)


# ---------------------------------------------------------------- shared inputs and oracle runs

_W = {}
_ORACLE = {}


def _weights():
    if 'w' not in _W:
        _W['w'] = synth_full_weights()
    return _W['w']


def _engine(w):
    from tacotronv2_wavernn_chinese_b200.tacotron.engine import TacoDecoderEngine
    return TacoDecoderEngine(w)


def _bank():
    """One memory row per entry of LENGTHS ([len(LENGTHS), 512, 512]; row i is a sentence of LENGTHS[i] tokens, the rest is
    padding that must not be read) and its dropout keep flags."""
    if 'bank' not in _W:
        _W['bank'] = (np.random.default_rng(5).random((len(LENGTHS), TXMAX, 512), dtype=F32) * 2 - 1,
                      (np.random.RandomState(6).uniform(size=(len(LENGTHS), STEPS, 2, 256)) >= 0.5).astype(np.uint8))
    return _W['bank']


def _oracle(i, window):
    """The oracle's free run of bank row i (its own length, its own keep flags), computed once per file."""
    if (i, window) not in _ORACLE:
        mem, masks = _bank()
        _ORACLE[(i, window)] = to.decode(_weights(), mem[i, :LENGTHS[i]], dropout_masks=masks[i], max_iters=STEPS, window=window)
    return _ORACLE[(i, window)]


def _check_free(out, b, ref, length, tag):
    """Row b of a decoder output against an oracle run: identical step count, frames 1e-4, stop and alignments 1e-5, and
    alignment columns at or beyond the sentence's length exactly 0.  Returns the three maximum errors."""
    n = ref['n_steps']
    fr, st, al = (out[k][b].cpu().numpy() for k in ('frames', 'stop', 'align'))
    assert int(out['nsteps'][b]) == n, (tag, int(out['nsteps'][b]), n)
    errs = (float(np.abs(fr[:n] - ref['frames']).max()), float(np.abs(st[:n] - ref['stop']).max()),
            float(np.abs(al[:n, :length] - ref['alignments']).max()))
    assert errs[0] <= 1e-4 and errs[1] <= 1e-5 and errs[2] <= 1e-5, (tag, errs)
    assert not al[:n, length:].any(), tag
    return errs


def _spread_states(seed, length, n, window):
    """n independent decoder loop states over a sentence of `length` tokens, with the previous alignments (alpha) and the
    cumulated alignments spread over every position; float32 throughout, so the records and the oracle see the same values.
    With the window, the first two records put it over the last positions of the sentence, the others anywhere."""
    rs = np.random.RandomState(seed)
    u = lambda lo, hi, shape: rs.uniform(lo, hi, shape).astype(F32)
    recs = []
    for k in range(n):
        alpha = u(0.2, 1.0, length)
        st = dict(c1=u(-1, 1, (1, 256)), h1=u(-1, 1, (1, 256)), c2=u(-1, 1, (1, 256)), h2=u(-1, 1, (1, 256)),
                  ctx=u(-1, 1, (1, 512)), alpha=(alpha / alpha.sum(dtype=F32)).astype(F32), cum=u(0, 3, length),
                  mu=F32(rs.uniform(0.05, 0.95)))
        at = max(length - 1 - 2 * k, 0) if k < 2 else int(rs.randint(0, length))
        win = dict(max_att=at, pos_rec=int(rs.randint(0, 12))) if window else {}
        recs.append((u(-2, 2, (1, 80)), st, win))
    return recs


def _forced_reference(w, mem, recs, masks, window):
    """The oracle's decoder step from each record: (frames [n, 80], stop [n], alignments [n, Tx])."""
    keys = (mem @ w['memory_layer/kernel']).astype(F32)
    frames, stops, aligns = [], [], []
    for s, (x, st, win) in enumerate(recs):
        mod = (lambda al, win=win: to.attention_window(al, win['max_att'], win['pos_rec'])[0]) if window else None
        out, _ = to.decoder_step(w, mem, keys, x, np.asarray(masks[s], F32), st, modulate=mod)
        frames.append(out['frame'][0]); stops.append(to._sigmoid(out['stop_logit'])[0, 0]); aligns.append(out['alignments'])
    return np.stack(frames), np.array(stops, F32), np.stack(aligns)


def _check_forced(out, b, ref, length, tag):
    fr, st, al = (out[k][b].cpu().numpy() for k in ('frames', 'stop', 'align'))
    n = len(ref[0])
    assert int(out['nsteps'][b]) == n, tag
    errs = (float(np.abs(fr[:n] - ref[0]).max()), float(np.abs(st[:n] - ref[1]).max()),
            float(np.abs(al[:n, :length] - ref[2]).max()))
    assert errs[0] <= 1e-4 and errs[1] <= 1e-5 and errs[2] <= 1e-5, (tag, errs)
    assert not al[:n, length:].any(), tag
    return errs


def _report(title, rows):
    """rows: (label, errors...) -> one printed line per row (pytest -s shows them)."""
    print(f'\n{title}')
    for r in rows:
        print('  ' + str(r[0]).rjust(12) + '  ' + '  '.join(f'{e:.2e}' for e in r[1:]))


# ---------------------------------------------------------------- 1. encoder

def test_encoder_every_length_vs_float64():
    """One ragged [20, 512] call with one sentence per length of LENGTHS; padding positions hold valid non-zero ids, so a read
    past a sentence's end would change its rows.  2e-5 abs against float64; rows at and beyond each length exactly 0."""
    w = _weights()
    eng = _engine(w)
    rs = np.random.RandomState(21)
    ids = rs.randint(1, 191, (len(LENGTHS), TXMAX)).astype(np.int32)
    mem = eng.encode(ids, np.array(LENGTHS, np.int32)).cpu().numpy()
    rows = []
    for b, n in enumerate(LENGTHS):
        err = float(np.abs(mem[b, :n] - encoder64(w, ids[b, :n])).max())
        rows.append((n, err))
        assert not mem[b, n:].any(), n
    _report('encoder vs float64, max abs error per length', rows)
    assert max(e for _, e in rows) <= 2e-5, rows


def test_encoder_140_sentences_match_each_sentence_alone():
    """B = 140 (280 BiLSTM blocks of 1024 threads: more than one wave on 132 SMs), lengths cycling over 1 ... 512: every row
    equals the same sentence encoded alone in a buffer of its own length, bit for bit, and is 0 beyond its length."""
    import torch
    w = _weights()
    eng = _engine(w)
    B = 140
    lengths = (1 + (np.arange(B) * 11) % TXMAX).astype(np.int32)
    assert lengths.min() == 1 and lengths.max() == TXMAX
    ids = np.random.RandomState(22).randint(1, 191, (B, TXMAX)).astype(np.int32)
    mem = eng.encode(ids, lengths)
    for b in range(B):
        n = int(lengths[b])
        solo = eng.encode(ids[b:b + 1, :n], lengths[b:b + 1])
        assert torch.equal(mem[b, :n], solo[0]), b
        assert not bool(mem[b, n:].any()), b


# ---------------------------------------------------------------- 2. postnet

def test_postnet_2000_frames_vs_float64():
    """max_steps = 2000, frames uniform in [-6, 6] (both clips active), step counts at the conv tile edges, 1000, 1999, 2000,
    and 0 and -1 (the count of a failed decode), which leave the whole row 0.  5e-5 abs against float64; rows at and beyond
    each count exactly 0."""
    w = _weights()
    eng = _engine(w)
    ms = 2000
    nsteps = np.array([1, 2, 3, 5, 8, 9, 1000, 1999, 2000, 0, -1], np.int32)
    frames = np.random.RandomState(23).uniform(-6, 6, (len(nsteps), ms, 80)).astype(F32)
    mel = eng.postnet(frames, nsteps).cpu().numpy()
    rows = []
    for b, n in enumerate(nsteps):
        n0 = max(int(n), 0)
        assert not mel[b, n0:].any(), n
        if n0:
            rows.append((int(n), float(np.abs(mel[b, :n0] - postnet64(w, frames[b, :n0])).max())))
    _report('postnet vs float64, max abs error per step count', rows)
    assert max(e for _, e in rows) <= 5e-5, rows


# ---------------------------------------------------------------- 3. single-sentence grid decoder (B = 1)

GRID_CASES = [(n, False) for n in LENGTHS] + [(5, True), (129, True), (512, True)]


@pytest.mark.parametrize('length,window', GRID_CASES, ids=[f'{n}{"-window" if wd else ""}' for n, wd in GRID_CASES])
def test_grid_decoder_vs_oracle(length, window):
    """taco_grid_kernel (B = 1, Txp = length rounded up to 4): 48 free steps against the oracle's loop, then FORCED steps from
    spread loop states against the oracle's step.  Frames 1e-4, stop and alignments 1e-5, identical step counts."""
    w = _weights()
    eng = _engine(w)
    i = LENGTHS.index(length)
    mem, masks = _bank()
    out = eng.decode(mem[i:i + 1, :length], masks=masks[i:i + 1], max_steps=STEPS, window=window)
    free = _check_free(out, 0, _oracle(i, window), length, 'free')
    recs = _spread_states(100 + length, length, FORCED, window)
    states = np.stack([eng.pack_state(x, st, win) for x, st, win in recs])[None]
    out = eng.decode(mem[i:i + 1, :length], masks=masks[i:i + 1, :FORCED], max_steps=FORCED, window=window, forced_states=states)
    forced = _check_forced(out, 0, _forced_reference(w, mem[i, :length], recs, masks[i], window), length, 'forced')
    _report(f'grid decoder, {length} tokens, window {window}: frame / stop / alignment errors', [('free', *free), ('forced', *forced)])


@pytest.mark.parametrize('buffer,length', [(512, 130), (130, 3)])
def test_grid_decoder_shorter_than_its_buffer(buffer, length):
    """The padded buffer sets Txp (exchange slots, energy partials) while the kernel attends over lengths[0] only."""
    w = _weights()
    eng = _engine(w)
    mem = np.random.default_rng(buffer + length).random((1, buffer, 512), dtype=F32) * 2 - 1
    masks = (np.random.RandomState(buffer).uniform(size=(1, STEPS, 2, 256)) >= 0.5).astype(np.uint8)
    ln = np.array([length], np.int32)
    out = eng.decode(mem, ln, masks=masks, max_steps=STEPS)
    ref = to.decode(w, mem[0, :length], dropout_masks=masks[0], max_iters=STEPS)
    free = _check_free(out, 0, ref, length, 'free')
    recs = _spread_states(200 + length, length, FORCED, False)
    states = np.stack([eng.pack_state(x, st, win, Tx_max=buffer) for x, st, win in recs])[None]
    out = eng.decode(mem, ln, masks=masks[:, :FORCED], max_steps=FORCED, forced_states=states)
    forced = _check_forced(out, 0, _forced_reference(w, mem[0, :length], recs, masks[0], False), length, 'forced')
    _report(f'grid decoder, {length} tokens in a buffer of {buffer}', [('free', *free), ('forced', *forced)])


# ---------------------------------------------------------------- 4. one block per sentence

@pytest.mark.parametrize('window', [False, True])
def test_batch_decoder_ragged_every_length_vs_oracle(window):
    """taco_decoder_kernel on one ragged batch of every length of LENGTHS at Tx_max = 512: 48 free steps against the oracle,
    then FORCED steps from spread loop states against the oracle's step."""
    w = _weights()
    eng = _engine(w)
    mem, masks = _bank()
    lengths = np.array(LENGTHS, np.int32)
    out = eng.decode(mem, lengths, masks=masks, max_steps=STEPS, window=window)
    rows = [(n, *_check_free(out, b, _oracle(b, window), n, f'free {n}')) for b, n in enumerate(LENGTHS)]
    _report(f'batch decoder, window {window}, free run: frame / stop / alignment errors per length', rows)
    recs = [_spread_states(300 + n, n, FORCED, window) for n in LENGTHS]
    states = np.stack([np.stack([eng.pack_state(x, st, win, Tx_max=TXMAX) for x, st, win in r]) for r in recs])
    out = eng.decode(mem, lengths, masks=masks[:, :FORCED], max_steps=FORCED, window=window, forced_states=states)
    rows = [(n, *_check_forced(out, b, _forced_reference(w, mem[b, :n], recs[b], masks[b], window), n, f'forced {n}'))
            for b, n in enumerate(LENGTHS)]
    _report(f'batch decoder, window {window}, forced steps: frame / stop / alignment errors per length', rows)


def test_batch_decoder_140_sentences_philox():
    """B = 140 sentences (two waves of one 1024-thread block per SM), lengths cycling over 1 ... 512, Philox dropout: 16 rows
    spread over the batch against the oracle (fed the keep flags Philox draws), and every row bit-identical to the same
    sentence decoded in a batch of 2 with the same global sentence index (same kernel, same summation order)."""
    w = _weights()
    eng = _engine(w)
    B, seed = 140, 31
    lengths = (1 + (np.arange(B) * 11) % TXMAX).astype(np.int32)
    mem = np.random.default_rng(32).random((B, TXMAX, 512), dtype=F32) * 2 - 1
    out = eng.decode(mem, lengths, seed=seed, max_steps=STEPS)
    host = {k: out[k].cpu().numpy() for k in ('frames', 'stop', 'align', 'nsteps')}
    masks = eng.philox_masks(seed, 0, B, STEPS).cpu().numpy()
    rows = []
    for b in np.linspace(0, B - 1, 16).astype(int).tolist() + [int(np.argmax(lengths))]:
        n = int(lengths[b])
        ref = to.decode(w, mem[b, :n], dropout_masks=masks[b], max_iters=STEPS)
        rows.append((f'row {b} ({n})', *_check_free(out, b, ref, n, f'row {b}')))
    _report('batch of 140, Philox dropout: frame / stop / alignment errors', rows)
    for b in range(0, B, 2):
        t = int(lengths[b:b + 2].max())
        pair = eng.decode(mem[b:b + 2, :t], lengths[b:b + 2], seed=seed, utterance_offset=b, max_steps=STEPS)
        for j in range(2):
            n, steps = int(lengths[b + j]), int(host['nsteps'][b + j])
            assert int(pair['nsteps'][j]) == steps, b + j
            assert np.array_equal(pair['frames'][j].cpu().numpy(), host['frames'][b + j]), b + j
            assert np.array_equal(pair['stop'][j].cpu().numpy(), host['stop'][b + j]), b + j
            assert np.array_equal(pair['align'][j, :steps, :n].cpu().numpy(), host['align'][b + j, :steps, :n]), b + j


def test_stop_rule_fires_at_long_lengths():
    """The generator's own stop bias: the stop token crosses 0.5 after a few steps (by more than 2e-3 at every step of this
    sentence), so both decoders must stop at the oracle's step, at 512 tokens and in a buffer of 512 at 257."""
    w = synth_full_weights(stop_bias=None)
    eng = _engine(w)
    mem = np.random.default_rng(1014).random((TXMAX, 512), dtype=F32) * 2 - 1
    masks = (np.random.RandomState(2014).uniform(size=(STEPS, 2, 256)) >= 0.5).astype(np.uint8)
    refs = [to.decode(w, mem[:n], dropout_masks=masks, max_iters=STEPS) for n in (TXMAX, 257)]
    assert 1 < refs[0]['n_steps'] < STEPS and 1 < refs[1]['n_steps'] < STEPS
    one = eng.decode(mem[None], masks=masks[None], max_steps=STEPS)
    _check_free(one, 0, refs[0], TXMAX, 'grid')
    two = eng.decode(np.stack([mem, mem]), np.array([TXMAX, 257], np.int32), masks=np.stack([masks, masks]), max_steps=STEPS)
    for b, n in enumerate((TXMAX, 257)):
        _check_free(two, b, refs[b], n, f'batch {n}')


# ---------------------------------------------------------------- 5. teacher forced at 512 tokens, shipped checkpoint

def test_teacher_forced_512_tokens_real_checkpoint():
    """A 512-token sentence made of shipped sentences end to end: encoded on the GPU against float64 (2e-5), then ~100
    teacher-forced steps from the oracle's own loop states in the grid decoder (B = 1) and in a batch of 2, at the bars of
    test_decoder_teacher_forced_all_steps_config4 (frames 1e-4, stop and alignments 1e-5)."""
    w = real_taco_weights()
    if w is None:
        pytest.skip('shipped Tacotron checkpoint not available on this box')
    s = sentences()['sentences']
    eos = s['1']['ids'][-1]
    ids = []
    for k in sorted(s, key=int):
        ids += s[k]['ids'][:-1]
        if len(ids) >= TXMAX - 1:
            break
    ids = np.array(ids[:TXMAX - 1] + [eos], np.int32)
    assert len(ids) == TXMAX
    eng = _engine(w)
    mem = eng.encode(ids[None]).cpu().numpy()[0]
    eerr = float(np.abs(mem - encoder64(w, ids)).max())
    _report('real checkpoint, 512 tokens: encoder vs float64', [('encoder', eerr)])
    assert eerr <= 2e-5
    masks = (np.random.RandomState(512).uniform(size=(1, 100, 2, 256)) >= 0.5).astype(np.uint8)
    ref = to.decode(w, mem, dropout_masks=masks[0], max_iters=100, capture_states=range(100))
    n = ref['n_steps']
    assert n > 50
    states = np.stack([eng.pack_state(*[ref['states'][t][i] for i in (0, 1, 3)]) for t in range(n)])[None]
    refs = (ref['frames'], ref['stop'], ref['alignments'])
    one = eng.decode(mem[None], masks=masks[:, :n], max_steps=n, forced_states=states)
    two = eng.decode(np.stack([mem, mem]), masks=np.concatenate([masks, masks])[:, :n], max_steps=n,
                     forced_states=np.concatenate([states, states]))
    rows = [('grid', *_check_forced(one, 0, refs, TXMAX, 'grid'))]
    rows += [(f'batch row {b}', *_check_forced(two, b, refs, TXMAX, f'batch {b}')) for b in range(2)]
    _report(f'real checkpoint, 512 tokens, {n} teacher-forced steps: frame / stop / alignment errors', rows)


# ---------------------------------------------------------------- 6. GTA at long inputs

def test_gta_long_inputs_vs_oracle():
    """decode_gta on a ragged batch of 1, 129 and 512 tokens, Ty = 64: frames 1e-4 and alignments 1e-5 against
    tacotron_gta_oracle.decode_gta, zeros beyond each sentence and each step count; each row equals the sentence alone."""
    w = _weights()
    eng = _engine(w)
    rs = np.random.RandomState(41)
    lengths = np.array([1, 129, 512], np.int32)
    tlen = np.array([64, 50, 64], np.int32)
    Ty = 64
    mem = np.random.default_rng(42).random((3, TXMAX, 512), dtype=F32) * 2 - 1
    targets = rs.uniform(-4, 4, (3, Ty, 80)).astype(F32)
    masks = (rs.uniform(size=(3, Ty, 2, 256)) >= 0.5).astype(np.uint8)
    out = eng.decode_gta(mem, lengths, targets, tlen, masks=masks, want_align=True)
    fr, al = out['frames'].cpu().numpy(), out['align'].cpu().numpy()
    rows = []
    for b in range(3):
        n, t = int(lengths[b]), int(tlen[b])
        ref = gta.decode_gta(w, mem[b, :n], targets[b, :t], dropout_masks=masks[b])
        rows.append((n, float(np.abs(fr[b, :t] - ref['frames']).max()), float(np.abs(al[b, :t, :n] - ref['alignments']).max())))
        assert rows[-1][1] <= 1e-4 and rows[-1][2] <= 1e-5, rows[-1]
        assert not al[b, :, n:].any() and not fr[b, t:].any() and not al[b, t:].any()
        solo = eng.decode_gta(mem[b:b + 1, :n], None, targets[b:b + 1, :t], None, masks=masks[b:b + 1, :t], want_align=True)
        assert np.array_equal(solo['frames'].cpu().numpy()[0], fr[b, :t])
        assert np.array_equal(solo['align'].cpu().numpy()[0], al[b, :t, :n])
    _report('GTA, Ty = 64: frame / alignment errors per length', rows)


# ---------------------------------------------------------------- 7. refusals

class _NoLibrary:
    """Stands in for the library handle: any call into it fails the test."""

    def __getattr__(self, name):
        raise AssertionError(f'{name} was called')


def test_out_of_range_arguments_are_refused_before_any_library_call():
    from tacotronv2_wavernn_chinese_b200._lib import B200TTSError
    from tacotronv2_wavernn_chinese_b200.tacotron.engine import TacoDecoderEngine
    w = _weights()
    eng = _engine(w)
    ids = np.random.RandomState(51).randint(1, 191, (2, 9)).astype(np.int32)
    bad_id = ids.copy(); bad_id[1, 4] = 191
    neg_id = ids.copy(); neg_id[0, 0] = -1
    frames = np.zeros((2, 6, 80), F32)
    lib, eng.lib = eng.lib, _NoLibrary()
    try:
        for kw in (dict(ids=ids, lengths=[9, 10]), dict(ids=ids, lengths=[0, 9]), dict(ids=ids, lengths=[-3, 9]),
                   dict(ids=ids, lengths=[9]), dict(ids=ids[0], lengths=[9]), dict(ids=bad_id, lengths=[9, 9]),
                   dict(ids=neg_id, lengths=[9, 9])):
            with pytest.raises(ValueError):
                eng.encode(**kw)
        for n in ([7, 1], [3], [[3, 3]]):
            with pytest.raises(ValueError):
                eng.postnet(frames, np.array(n, np.int32))
        with pytest.raises(ValueError):
            eng.postnet(frames[:, :, :79], np.array([3, 3], np.int32))
    finally:
        eng.lib = lib
    # ids at or beyond a sentence's length are padding: any value is accepted and none is read
    pad = bad_id.copy(); pad[0, 5:] = 10 ** 6
    a = eng.encode(pad, [5, 4]).cpu().numpy()
    b = eng.encode(ids, [5, 4]).cpu().numpy()
    assert np.array_equal(a, b)
    # location features of a 512-token sentence x 64 filters would overflow taco_decoder_kernel's partial buffer
    small = dict(w)
    rs = np.random.RandomState(52)
    L = 'decoder/Location_Sensitive_Attention/'
    for k, shp in ((L + 'query_layer/kernel', (256, 64)), (L + 'location_features_convolution/kernel', (15, 1, 64)),
                   (L + 'location_features_convolution/bias', (64,)), (L + 'location_features_layer/kernel', (64, 64)),
                   (L + 'attention_variable_projection', (64,)), (L + 'attention_bias', (64,)), ('memory_layer/kernel', (512, 64))):
        small[k] = rs.uniform(-0.1, 0.1, shp).astype(F32)
    with pytest.raises(B200TTSError) as e:
        TacoDecoderEngine(small, cfg=dict(attn_filters=64, attn_dim=64, attn_kernel=15))
    assert e.value.code == -1 and 'attn_filters' in str(e.value)
