"""Tacotron decoder sessions on the GPU (TacoDecoderEngine.open_decode_sessions / advance_decodes / decode_outputs,
Synthesizer.open_decodes / finish_decodes, StreamingSynthesizer(decode_steps=k)).  Every comparison is np.array_equal against the
one-shot batch decoder (taco_decoder_kernel, B >= 2): frames, stop values and step counts, however the steps are cut, whichever
sessions share a slice, with the window on or off and with per-row speaking-rate biases.  The service's mels and pieces equal
the one-shot decode, postnet, stop cut and generate.  Open / run / close cycles leak no device memory."""
import numpy as np
import pytest

from taco_common import real_taco_weights, sentences, synth_taco_weights
from test_stream_synth_gpu import HOP, _one_shot_waves, _texts
from test_wavernn_gpu import engine_for, torch_cuda  # noqa: F401  (torch_cuda is a fixture)
from tacotronv2_wavernn_chinese_b200 import pipeline

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def never(torch_cuda):
    """Synthetic decoder whose stop token never fires: every decode runs to max_steps."""
    from tacotronv2_wavernn_chinese_b200.tacotron.engine import TacoDecoderEngine
    w = synth_taco_weights(3)
    w['decoder/stop_token_projection/projection_stop_token_projection/bias'][:] = -1e4
    return TacoDecoderEngine(w)


@pytest.fixture(scope='module')
def syn(torch_cuda):
    w = real_taco_weights()
    if w is None:
        pytest.skip('shipped Tacotron checkpoint not available on this box')
    from tacotronv2_wavernn_chinese_b200.tacotron.engine import TacoDecoderEngine
    from tacotronv2_wavernn_chinese_b200.tacotron.synthesizer import Synthesizer
    from tacotronv2_wavernn_chinese_b200.tacotron.text import Symbols
    s = Synthesizer()
    s.symbols = Symbols(sentences()['symbols'])
    s.engine = TacoDecoderEngine(w)
    s.max_iters = 150
    return s


def _memory(torch, n, Tx, seed):
    rs = np.random.RandomState(seed)
    return torch.as_tensor(rs.uniform(-1, 1, size=(n, Tx, 512)).astype(np.float32)).cuda()


def _one_shot(eng, mem, lengths, ids, seed, max_steps, window=False, bias=None):
    """Row i's one-shot run on the batch decoder: a batch of two copies of row i (B = 2), row 0 keyed by ids[i]."""
    out = []
    for i in range(mem.shape[0]):
        kw = {} if bias is None or bias[i] == 0 else {'mu_bias': [bias[i], bias[i]]}
        d = eng.decode(mem[[i, i]], [lengths[i]] * 2, seed=seed, utterance_offset=ids[i], max_steps=max_steps, window=window,
                       want_align=False, **kw)
        n = int(d['nsteps'][0])
        out.append((d['frames'][0, :n].cpu().numpy(), d['stop'][0, :n].cpu().numpy(), n))
    return out


def _check(eng, sessions, ref):
    got = eng.decode_outputs(sessions)
    fr, st, ns = got['frames'].cpu().numpy(), got['stop'].cpu().numpy(), got['nsteps'].cpu().numpy()
    for i, (s, (rf, rs, rn)) in enumerate(zip(sessions, ref)):
        assert s.done and s.position == rn == ns[i], (i, s.position, rn)
        assert np.array_equal(fr[i, :rn], rf) and np.array_equal(st[i, :rn], rs), f'row {i}'
        assert not fr[i, rn:].any() and not st[i, rn:].any()


def _run_cuts(eng, sessions, cuts):
    for k in cuts:
        eng.advance_decodes(sessions, k)
    while not all(s.done for s in sessions):
        eng.advance_decodes(sessions, 1000)


# ---- 1. one sentence, cut every way, up to max_steps ---------------------------------------------------------------------
@pytest.mark.parametrize('window', [False, True])
@pytest.mark.parametrize('bias', [0.0, 0.2, -0.05])
@pytest.mark.parametrize('cuts', [[1] * 40, [3, 7, 1, 13, 2, 9, 5], [40], [39, 1], [100]])
def test_one_sentence_in_slices_to_max_steps(torch_cuda, never, window, bias, cuts):
    mem = _memory(torch_cuda, 1, 37, 11)
    ref = _one_shot(never, mem, [37], [(1 << 40) + 5], 7, 40, window, [bias])
    assert ref[0][2] == 40                                   # the stop never fires
    ss = never.open_decode_sessions(mem, [37], [(1 << 40) + 5], seed=7, max_steps=40, window=window, mu_bias=bias)
    _run_cuts(never, ss, cuts)
    _check(never, ss, ref)
    never.advance_decodes(ss, 5)                             # a finished session takes part with 0 steps
    assert ss[0].position == 40
    ss[0].close()


# ---- 2. cuts at and around the stop step (shipped checkpoint) ------------------------------------------------------------
def _encoded(syn, texts):
    seqs = [syn.symbols.text_to_sequence(t) for t in texts]
    tok = np.zeros((len(seqs), max(map(len, seqs))), dtype=np.int32)
    for b, s in enumerate(seqs):
        tok[b, :len(s)] = s
    ln = np.array([len(s) for s in seqs], dtype=np.int32)
    return syn.engine.encode(tok, ln), ln


@pytest.mark.parametrize('window', [False, True])
def test_cuts_at_the_stop_step(torch_cuda, syn, window):
    eng = syn.engine
    mem, ln = _encoded(syn, _texts(syn, 8, first=5))
    ids = [9, 1 << 33, 77, 5, 6, 1 << 50, 12, 13]
    bias = [0.0, 0.1, -0.03, 0.0, 0.2, 0.05, 0.0, 0.1]
    ref = _one_shot(eng, mem, ln, ids, 4, 250, window, bias)
    rows = [i for i in range(8) if ref[i][2] < 250][:3]      # sentences whose stop fires
    assert len(rows) >= 2, [r[2] for r in ref]
    mem, ln, ids, bias, ref = mem[rows], ln[rows], [ids[i] for i in rows], [bias[i] for i in rows], [ref[i] for i in rows]
    stops = [r[2] for r in ref]
    for i in range(len(rows)):
        s = stops[i]
        for cuts in ([s], [s + 1], [s - 1, 1], [s - 1, 2], [1] * s, [2, 5, 1, s]):
            ses = eng.open_decode_sessions(mem[i:i + 1], ln[i:i + 1], ids[i:i + 1], seed=4, max_steps=250, window=window,
                                           mu_bias=bias[i])
            for k in cuts:
                if not ses[0].done:
                    eng.advance_decodes(ses, max(k, 1))
            assert ses[0].done, (i, cuts)
            _check(eng, ses, ref[i:i + 1])
            ses[0].close()


# ---- 3. many sessions of mixed lengths, opened at different slices, sharing launches -------------------------------------
@pytest.mark.parametrize('n', [1, 2, 33, 128])
def test_sessions_share_slices(torch_cuda, syn, n):
    eng = syn.engine
    rs = np.random.RandomState(n)
    lengths = [int(x) for x in rs.randint(1, 513, size=n)]
    lengths[0] = 512
    ids = [int(x) for x in rs.randint(0, 2 ** 62, size=n, dtype=np.int64)]
    bias = [float(x) for x in rs.choice([0.0, 0.0, 0.15, -0.04], size=n)]
    mem = _memory(torch_cuda, n, max(lengths), 100 + n)
    for i, L in enumerate(lengths):
        mem[i, L:] = 0
    ref = _one_shot(eng, mem, lengths, ids, 6, 60, False, bias)
    half = (n + 1) // 2
    a = eng.open_decode_sessions(mem[:half], lengths[:half], ids[:half], seed=6, max_steps=60, mu_bias=bias[:half])
    eng.advance_decodes(a, 5)
    b = eng.open_decode_sessions(mem[half:], lengths[half:], ids[half:], seed=6, max_steps=60, mu_bias=bias[half:]) if n > 1 else []
    for k in (3, 11, 1, 17):
        eng.advance_decodes(a + b, k)                        # one launch for both opens
    _run_cuts(eng, a + b, [7])
    _check(eng, a + b, ref)
    for s in a + b:
        s.close()


# ---- 4. the sliced service end to end -------------------------------------------------------------------------------------
@pytest.mark.parametrize('max_rows,decode_steps', [(32, 9), (128, 25)])
def test_sliced_service_end_to_end(torch_cuda, syn, max_rows, decode_steps):
    from tacotronv2_wavernn_chinese_b200.tacotron.synthesizer import unit_mel
    eng, _ = engine_for('ckpt')
    n, seed = 24, 17
    texts = _texts(syn, n, first=20)
    ids = [3 * i + 1000 for i in range(n)]
    biases = [(0.0, 0.12, -0.04)[i % 3] for i in range(n)]
    groups = []
    opener = syn.open_decodes

    def recording(tx, ix, seed=0, mu_bias=None):
        groups.append((list(tx), list(ix), mu_bias))
        return opener(tx, ix, seed=seed, mu_bias=mu_bias)

    syn.open_decodes = recording
    try:
        ss = pipeline.StreamingSynthesizer(syn, eng, seed=seed, chunk_steps=10 * HOP, max_rows=max_rows, decode_steps=decode_steps)
        got, finished, mels, nxt = {}, [], {}, 0
        while nxt < n or not ss.idle():
            for _ in range(3):
                if nxt < n:
                    ss.submit(nxt, texts[nxt], ids[nxt], mu_bias=biases[nxt])
                    nxt += 1
            for key, piece, fin in ss.step():
                if key not in mels:
                    mels[key] = ss.mel(key)
                got.setdefault(key, []).append(piece)
                if fin:
                    finished.append(key)
            assert ss.active + ss.decoding <= max_rows
    finally:
        syn.open_decodes = opener
    assert sorted(finished) == list(range(n))
    assert [i for _tx, ix, _b in groups for i in ix] == ids
    # reference: each admission group's encoder output, the one-shot batch decode of every row, postnet, stop cut
    eng_t = syn.engine
    for tx, ix, gb in groups:
        mem, ln = _encoded(syn, tx)
        bias = [0.0] * len(ix) if gb is None else [float(x) for x in gb]
        for i, (uid, b) in enumerate(zip(ix, bias)):
            kw = {} if b == 0 else {'mu_bias': [b, b]}
            d = eng_t.decode(mem[[i, i]], [ln[i]] * 2, seed=seed, utterance_offset=uid, max_steps=syn.max_iters, want_align=False, **kw)
            post = eng_t.postnet(d['frames'], d['nsteps'])
            T = int(eng_t.target_lengths(d['stop'], d['nsteps'])[0])
            k = ids.index(uid)
            assert np.array_equal(mels[k], unit_mel(post[0, :T].cpu().numpy())), f'mel of request {k}'
    ref = _one_shot_waves(eng, {k: m for k, m in mels.items() if m.shape[0] > 0}, {k: ids[k] for k in mels}, seed, max_rows > 32)
    for k in range(n):
        w = np.concatenate(got[k])
        assert (len(w) == 0) if mels[k].shape[0] == 0 else np.array_equal(w, ref[k]), f'request {k}'


# ---- 5. refusals with real sessions, and leaks ---------------------------------------------------------------------------
def test_refusals_with_real_sessions(torch_cuda, never):
    from tacotronv2_wavernn_chinese_b200._lib import B200TTSError
    from tacotronv2_wavernn_chinese_b200.tacotron.engine import TacoDecoderEngine
    other = TacoDecoderEngine(synth_taco_weights(3))
    mem = _memory(torch_cuda, 2, 8, 1)
    a = never.open_decode_sessions(mem, [8, 5], [1, 2], max_steps=10)
    b = other.open_decode_sessions(mem, [8, 5], [1, 2], max_steps=10)
    for call in (lambda: never.advance_decodes(a + [a[0]], 3), lambda: never.advance_decodes([a[0], b[0]], 3),
                 lambda: never.advance_decodes(a, 0), lambda: never.open_decode_sessions(mem, [8, 9], [1, 2]),
                 lambda: never.open_decode_sessions(mem, [8, 5], [1, 2], mu_bias=[0.0, 2.0])):
        with pytest.raises((B200TTSError, ValueError)):
            call()
    assert all(s.position == 0 for s in a + b)
    other.close()
    with pytest.raises(ValueError):
        b[0].position                                        # closing the engine closed its sessions
    for s in a:
        s.close()


def test_cycles_leak_no_device_memory(torch_cuda, never):
    mem = _memory(torch_cuda, 4, 64, 2)

    def cycle(i):
        ss = never.open_decode_sessions(mem, [64, 30, 7, 1], [4 * i + k for k in range(4)], max_steps=12)
        never.advance_decodes(ss, 5)
        never.decode_outputs(ss)
        for s in reversed(ss) if i % 2 else ss:
            s.close()

    for i in range(3):
        cycle(i)
    torch_cuda.cuda.synchronize()
    free0, _ = torch_cuda.cuda.mem_get_info()
    for i in range(200):
        cycle(i)
    torch_cuda.cuda.synchronize()
    free1, _ = torch_cuda.cuda.mem_get_info()
    assert abs(free0 - free1) < 8 << 20, (free0, free1)
