"""sm_90a speaking-rate control: the biased instantiations of taco_decoder_kernel and taco_grid_kernel through
b200tts_taco_decode_biased, TacoDecoderEngine.decode(mu_bias=...) and the streaming service.  The oracle's biased attention
step is pinned against the reference's own statements with the branch switched on (tests/test_tacotron_rate_pins.py)."""
import ctypes as C

import numpy as np
import pytest

from oracle import tacotron_oracle as to
from oracle import tacotron_rate_oracle as tro
from taco_common import real_taco_weights, sentences, synth_taco_weights

pytestmark = pytest.mark.gpu

FIXTURE_DELTAS = (-1.0, -0.3, -0.04, 0.04, 0.3, 1.0)          # the deltas of tests/golden/taco_rate_from_reference.npz
RESPONSE_DELTAS = (-0.06, -0.04, 0.0, 0.04, 0.1, 0.2, 0.3)
RESPONSE_SEED = 5


def _masks(seed, B, steps):
    return (np.random.RandomState(seed).uniform(size=(B, steps, 2, 256)) >= 0.5).astype(np.uint8)


@pytest.fixture(scope='module')
def real():
    w = real_taco_weights()
    if w is None:
        pytest.skip('shipped Tacotron checkpoint not available on this box')
    from tacotronv2_wavernn_chinese_b200.tacotron.engine import TacoDecoderEngine
    return w, TacoDecoderEngine(w)


def _weights_and_memory(B, seed=3):
    """Shipped checkpoint and real encoder outputs when available, portable synthetic weights and random memory otherwise."""
    from tacotronv2_wavernn_chinese_b200.tacotron.engine import TacoDecoderEngine
    w = real_taco_weights()
    if w is not None:
        eng = TacoDecoderEngine(w)
        ss = sentences()['sentences']
        seqs = [ss[k]['ids'] for k in ('241', '378', '407', '12')[:B]]
        tok = np.zeros((B, max(map(len, seqs))), np.int32)
        for b, s in enumerate(seqs):
            tok[b, :len(s)] = s
        ln = np.array([len(s) for s in seqs], np.int32)
        return eng, eng.encode(tok, ln).cpu().numpy(), ln
    eng = TacoDecoderEngine(synth_taco_weights(7))
    rs = np.random.RandomState(seed)
    ln = np.array([37, 20, 29, 33][:B], np.int32)
    return eng, rs.uniform(-1, 1, (B, 37, 512)).astype(np.float32), ln


def _biased_raw(eng, mem, ln, bias, *, masks=None, seed=0, steps, window, states=None):
    """b200tts_taco_decode_biased called directly (also at bias 0, which the Python layer would route to the plain entry)."""
    import torch
    from tacotronv2_wavernn_chinese_b200 import _lib
    dev = torch.device('cuda', eng.device)
    m = torch.as_tensor(mem, device=dev).contiguous()
    B, Tx, _ = m.shape
    lt = torch.as_tensor(ln, dtype=torch.int32, device=dev)
    d = _lib.TacoDropout()
    d.seed = seed
    md = None
    if masks is not None:
        md = torch.as_tensor(masks, device=dev).contiguous()
        d.mode, d.d_masks = 1, md.data_ptr()
    fs = None if states is None else torch.as_tensor(states, dtype=torch.float32, device=dev).contiguous()
    out = dict(frames=torch.zeros(B, steps, 80, device=dev), stop=torch.zeros(B, steps, device=dev),
               align=torch.zeros(B, steps, Tx, device=dev), nsteps=torch.zeros(B, dtype=torch.int32, device=dev))
    hb = np.ascontiguousarray(np.broadcast_to(np.asarray(bias, np.float32), (B,)))
    p = lambda t: C.c_void_p(t.data_ptr() if t is not None else 0)
    _lib.check(eng.lib.b200tts_taco_decode_biased(eng._h, p(m), p(lt), B, Tx, C.byref(d), steps, int(window),
                                                  hb.ctypes.data_as(C.POINTER(C.c_float)), p(fs), p(out['frames']), p(out['stop']),
                                                  p(out['align']), p(out['nsteps']), eng._stream()))
    return {k: v.cpu().numpy() for k, v in out.items()}


def _host(out):
    return {k: v.cpu().numpy() for k, v in out.items() if v is not None}


# ---- 1. delta = 0 is today's decoder ----------------------------------------------------------------------------------------
@pytest.mark.parametrize('B', [1, 3])
@pytest.mark.parametrize('window', [False, True])
def test_zero_bias_is_the_unbiased_decoder_bit_for_bit(B, window):
    eng, mem, ln = _weights_and_memory(B)
    steps = 160
    plain = _host(eng.decode(mem, ln, seed=11, max_steps=steps, window=window))
    zero = _biased_raw(eng, mem, ln, 0.0, seed=11, steps=steps, window=window)
    for k in ('frames', 'stop', 'align', 'nsteps'):
        assert np.array_equal(plain[k], zero[k]), k
    assert np.array_equal(_host(eng.decode(mem, ln, seed=11, max_steps=steps, window=window, mu_bias=[0.0] * B))['frames'],
                          plain['frames'])


# ---- 2. whole utterances, teacher-forced ------------------------------------------------------------------------------------
@pytest.mark.parametrize('window', [False, True])
def test_teacher_forced_whole_utterance_at_every_fixture_delta(real, window):
    """Every step of the oracle's own biased run, from the oracle's loop state, on both kernels: the bars of
    test_decoder_teacher_forced_all_steps_config4.  A run that never stops (delta = -1 without the window: mu' = 0, attention
    never moves) is compared over its first CAP steps."""
    w, eng = real
    mem = to.encoder(w, sentences()['sentences']['241']['ids'])
    Tx, CAP = mem.shape[0], 600
    masks = _masks(1238, 1, CAP)
    refs, states = [], []
    for delta in FIXTURE_DELTAS:
        ref = tro.decode(w, mem, dropout_masks=masks[0], max_iters=CAP, window=window, capture_states=range(CAP), mu_bias=delta)
        refs.append(ref)
        states.append(np.stack([eng.pack_state(*[ref['states'][s][i] for i in (0, 1, 3)]) for s in range(ref['n_steps'])]))
    n_max = max(r['n_steps'] for r in refs)

    def check(out, b, ref, kernel):
        n = ref['n_steps']
        ferr = np.abs(out['frames'][b, :n] - ref['frames']).max(axis=1)
        where = f'{kernel}, delta {FIXTURE_DELTAS[b] if kernel == "batch" else ""}, {n} steps'
        assert ferr.max() <= 1e-4, f'{where}: frame error {ferr.max():.3e} at step {int(ferr.argmax())}'
        np.testing.assert_allclose(out['stop'][b, :n], ref['stop'], rtol=0, atol=1e-5, err_msg=where)
        np.testing.assert_allclose(out['align'][b, :n, :Tx], ref['alignments'], rtol=0, atol=1e-5, err_msg=where)
        assert (np.round(out['stop'][b, :n]) == np.round(ref['stop'])).all(), where             # identical stop step

    for delta, ref, st in zip(FIXTURE_DELTAS, refs, states):                                     # B = 1: taco_grid_kernel
        n = ref['n_steps']
        out = _biased_raw(eng, mem[None], [Tx], delta, masks=masks[:, :n], steps=n, window=window, states=st[None])
        assert int(out['nsteps'][0]) == n
        check(out, 0, ref, f'grid delta {delta}')
    # all six deltas as the rows of ONE batch (taco_decoder_kernel), records past a row's own end repeat its last state
    B = len(FIXTURE_DELTAS)
    pad = np.stack([np.concatenate([st, np.repeat(st[-1:], n_max - len(st), axis=0)]) for st in states])
    out = _biased_raw(eng, np.repeat(mem[None], B, axis=0), [Tx] * B, np.float32(FIXTURE_DELTAS),
                      masks=np.repeat(masks[:, :n_max], B, axis=0), steps=n_max, window=window, states=pad)
    for b, ref in enumerate(refs):
        check(out, b, ref, 'batch')
    assert any(r['n_steps'] < CAP for r in refs)


# ---- 3. free-run prefix -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('window', [False, True])
def test_free_run_prefix_vs_oracle(real, window):
    w, eng = real
    mem = to.encoder(w, sentences()['sentences']['241']['ids'])
    Tx, steps = mem.shape[0], 40
    masks = _masks(1238, 1, steps)
    deltas = (0.1, -0.1)
    refs = [tro.decode(w, mem, dropout_masks=masks[0], max_iters=steps, window=window, mu_bias=d) for d in deltas]
    batch = _host(eng.decode(np.repeat(mem[None], 2, axis=0), masks=np.repeat(masks, 2, axis=0), max_steps=steps, window=window,
                             mu_bias=deltas))
    for b, (d, ref) in enumerate(zip(deltas, refs)):
        one = _host(eng.decode(mem[None], masks=masks, max_steps=steps, window=window, mu_bias=d))
        for kernel, out, r in (('grid', one, 0), ('batch', batch, b)):
            assert int(out['nsteps'][r]) == ref['n_steps'] == steps
            err = np.abs(out['frames'][r] - ref['frames']).max()
            assert err <= 1e-4, f'{kernel} delta {d}: frame error {err:.3e}'
            np.testing.assert_allclose(out['align'][r, :, :Tx], ref['alignments'], rtol=0, atol=1e-5)


# ---- 4. per-row biases in one batch -----------------------------------------------------------------------------------------
@pytest.mark.parametrize('window', [False, True])
def test_per_row_biases_in_one_ragged_batch(window):
    eng, mem, ln = _weights_and_memory(4, seed=8)
    deltas = np.float32([0.0, -0.04, 0.1, 0.3])
    steps = 300
    mixed = _host(eng.decode(mem, ln, seed=21, max_steps=steps, window=window, mu_bias=deltas))
    for b, d in enumerate(deltas):
        uniform = _host(eng.decode(mem, ln, seed=21, max_steps=steps, window=window, mu_bias=float(d)))
        n = int(mixed['nsteps'][b])
        assert n == int(uniform['nsteps'][b]) and n > 0
        for k in ('frames', 'stop', 'align'):
            assert np.array_equal(mixed[k][b, :n], uniform[k][b, :n]), (float(d), k)
    plain = _host(eng.decode(mem, ln, seed=21, max_steps=steps, window=window))
    n = int(plain['nsteps'][0])
    assert n == int(mixed['nsteps'][0])
    for k in ('frames', 'stop', 'align'):
        assert np.array_equal(mixed[k][0, :n], plain[k][0, :n]), k
    assert len(set(int(x) for x in mixed['nsteps'])) > 1


# ---- 5. the service ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('max_rows', [32, 128])
def test_service_with_mixed_biases(max_rows):
    import torch
    if not torch.cuda.is_available():
        pytest.fail('GPU tests need a CUDA device')
    w = real_taco_weights()
    if w is None:
        pytest.skip('shipped Tacotron checkpoint not available on this box')
    from test_stream_synth_gpu import _one_shot_waves, _texts
    from test_wavernn_gpu import engine_for
    from tacotronv2_wavernn_chinese_b200 import pipeline
    from tacotronv2_wavernn_chinese_b200.tacotron.engine import TacoDecoderEngine
    from tacotronv2_wavernn_chinese_b200.tacotron.synthesizer import Synthesizer
    from tacotronv2_wavernn_chinese_b200.tacotron.text import Symbols
    syn = Synthesizer()
    syn.symbols = Symbols(sentences()['symbols'])
    syn.engine = TacoDecoderEngine(w)
    syn.max_iters = 160
    eng, _ = engine_for('ckpt')
    n, seed = 16, 23
    texts = _texts(syn, n, first=30)
    ids = [500 + i for i in range(n)]
    deltas = [(0.0, -0.04, 0.1, 0.3)[i % 4] for i in range(n)]
    groups, decode = [], syn.decode_device

    def recording(tx, ix, seed=0, **kw):
        groups.append((list(tx), list(ix), kw.get('mu_bias')))
        return decode(tx, ix, seed=seed, **kw)

    syn.decode_device = recording
    try:
        ss = pipeline.StreamingSynthesizer(syn, eng, seed=seed, chunk_steps=10 * 275, max_rows=max_rows, max_admit=6)
        got, mels, nxt = {}, {}, 0
        while nxt < n or not ss.idle():
            for _ in range(3):
                if nxt < n:
                    ss.submit(nxt, texts[nxt], ids[nxt], mu_bias=deltas[nxt])
                    nxt += 1
            for key, piece, _fin in ss.step():
                if key not in mels:
                    mels[key] = ss.mel(key)
                got.setdefault(key, []).append(piece)
    finally:
        syn.decode_device = decode
    assert any(b is not None for _t, _i, b in groups)
    for tx, ix, bias in groups:
        want = [deltas[i - 500] for i in ix]
        assert (bias is None) == (not any(want)) and (bias is None or list(bias) == list(np.float32(want)))
        ref, _ = syn.mels(tx, seed=seed, utterance_offset=ix[0], mu_bias=want)
        for t, i in zip(ref, ix):
            assert np.array_equal(mels[i - 500], t), f'mel of request {i - 500}'
    ref = _one_shot_waves(eng, {k: m for k, m in mels.items() if m.shape[0] > 0}, {k: ids[k] for k in mels}, seed, max_rows > 32)
    for k in range(n):
        wv = np.concatenate(got[k])
        assert (len(wv) == 0) if mels[k].shape[0] == 0 else np.array_equal(wv, ref[k]), f'request {k}'


# ---- 6. length response on the shipped checkpoint ---------------------------------------------------------------------------
def length_response(eng, window, deltas=RESPONSE_DELTAS, seed=RESPONSE_SEED, max_steps=2000):
    """Every sentence of taco_symbols.json at every delta (one batch per delta, Philox keyed by sentence index): dict
    delta -> (cut lengths [n], nsteps [n], attention argmax at the stop step [n]) and the token counts [n]."""
    ss = sentences()['sentences']
    seqs = [ss[k]['ids'] for k in sorted(ss, key=int)]
    tok = np.zeros((len(seqs), max(map(len, seqs))), np.int32)
    for b, s in enumerate(seqs):
        tok[b, :len(s)] = s
    ln = np.array([len(s) for s in seqs], np.int32)
    mem = eng.encode(tok, ln)
    out = {}
    for d in deltas:
        dec = eng.decode(mem, ln, seed=seed, max_steps=max_steps, window=window, mu_bias=d)
        cut = eng.target_lengths(dec['stop'], dec['nsteps']).cpu().numpy()
        ns = dec['nsteps'].cpu().numpy()
        al = dec['align'].cpu().numpy()
        am = np.array([al[b, max(ns[b] - 1, 0), :ln[b]].argmax() for b in range(len(seqs))])
        out[d] = (cut, ns, am)
    return out, ln


@pytest.mark.parametrize('window', [False, True])
def test_length_response_on_the_shipped_checkpoint(real, window):
    _w, eng = real
    res, ln = length_response(eng, window)
    base = res[0.0][0].astype(np.float64)
    med = {d: float(np.median(res[d][0] / base)) for d in RESPONSE_DELTAS}
    for d, (cut, ns, am) in res.items():
        assert (ns < 2000).all() and (ns >= 1).all(), f'delta {d}: a stop never fired'
        assert (am >= ln - 3).all(), f'delta {d}: attention at the cut short of the last 3 tokens in {np.flatnonzero(am < ln - 3)}'
    chain = (-0.06, 0.0, 0.1, 0.3) if not window else (0.0, 0.1, 0.3)
    assert all(med[a] > med[b] for a, b in zip(chain, chain[1:])), med


# ---- 7. refusals ------------------------------------------------------------------------------------------------------------
def test_refusals_launch_nothing():
    import torch
    from tacotronv2_wavernn_chinese_b200._lib import B200TTSError
    eng, mem, ln = _weights_and_memory(2)
    sentinel = torch.full((2,), -7, dtype=torch.int32, device='cuda')
    for bad in ([float('nan'), 0.0], [0.0, float('inf')], [1.5, 0.0], [0.0, -1.01]):
        with pytest.raises(B200TTSError) as e:
            _biased_raw(eng, mem, ln, np.float32(bad), steps=8, window=False)
        assert e.value.code == -1, str(e.value)
        with pytest.raises(ValueError):
            eng.decode(mem, ln, max_steps=8, mu_bias=bad)
    with pytest.raises(ValueError):
        eng.decode(mem, ln, max_steps=8, mu_bias=[0.1, 0.2, 0.3])                                 # wrong count
    # the C entry refuses before anything is enqueued: an output it would write stays as it was
    import ctypes
    from tacotronv2_wavernn_chinese_b200 import _lib
    m = torch.as_tensor(mem, device='cuda')
    lt = torch.as_tensor(ln, device='cuda')
    fr = torch.zeros(2, 8, 80, device='cuda')
    stp = torch.zeros(2, 8, device='cuda')
    hb = (ctypes.c_float * 2)(0.2, float('nan'))
    d = _lib.TacoDropout()
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    rc = eng.lib.b200tts_taco_decode_biased(eng._h, p(m), p(lt), 2, m.shape[1], ctypes.byref(d), 8, 0, hb, None, p(fr), p(stp), None,
                                            p(sentinel), eng._stream())
    torch.cuda.synchronize()
    assert rc == -1 and (sentinel == -7).all() and 'mu_bias[1]' in eng.lib.b200tts_last_error().decode()
