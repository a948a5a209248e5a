"""sm_90a ground-truth-aligned (GTA) decoding: taco_decoder_kernel<true> through b200tts_taco_decode_gta, Synthesizer.gta_mels
and wavernn_preprocess.py.  The oracle's decode_gta is pinned against the reference's serialized graph over whole
utterances (tests/test_tacotron_gta_pins.py), and teacher forcing keeps float32 within 2e-5 of float64 over every step, so
the GPU is held to the graph over the WHOLE utterance, not a prefix as in free running."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import tacotron_gta_oracle as gta
from oracle import tacotron_oracle as to
from taco_common import REF_CKPT_DIR, TRAVEL_COPY, real_taco_weights, sentences, synth_taco_weights

pytestmark = pytest.mark.gpu


def _engine(w):
    from tacotronv2_wavernn_chinese_b200.tacotron.engine import TacoDecoderEngine
    return TacoDecoderEngine(w)


def _weights():
    w = real_taco_weights()
    if w is None:
        pytest.skip('shipped Tacotron checkpoint not available on this box')
    return w


def _gta_fixture():
    z = np.load(os.path.join(GOLDEN, 'taco_gta_from_graph.npz'))
    n = int(z['n_steps'])
    masks = np.unpackbits(z['masks'], axis=1)[:, :512].reshape(n, 2, 256)
    src = np.load(os.path.join(GOLDEN, str(z['target_file'])))[str(z['target_key'])]
    return z, n, masks, np.clip(src, -4.0, 4.0).astype(np.float32)


def test_whole_utterance_parity_with_the_graph_demo03():
    """Demo-03, 323 teacher-forced steps from the serialized graph's encoder memory: frames within 1e-4 over every step,
    alignments within 1e-5 of the oracle (which equals the graph), the postnet mel within 1e-4 of the graph's."""
    w = _weights()
    z, n, masks, targets = _gta_fixture()
    eng = _engine(w)
    out = eng.decode_gta(z['memory_graph'][None], None, targets[None], None, masks=masks[None], want_align=True)
    assert int(out['nsteps'][0]) == n
    fr, al = out['frames'].cpu().numpy()[0], out['align'].cpu().numpy()[0]
    ferr = np.abs(fr - z['frames']).max(axis=1)
    print(f'demo-03 GTA frames vs graph: max {ferr.max():.2e} at step {int(ferr.argmax())}')
    assert ferr.max() <= 1e-4, (int(ferr.argmax()), float(ferr.max()))
    ref = gta.decode_gta(w, z['memory_graph'], targets, dropout_masks=masks.astype(np.float32))
    np.testing.assert_allclose(al, ref['alignments'], rtol=0, atol=1e-5)
    assert np.array_equal(al.argmax(1), z['align_argmax'])
    np.testing.assert_allclose(al.max(1), z['align_peak'], rtol=0, atol=1e-5)
    mel = eng.postnet(out['frames'], out['nsteps']).cpu().numpy()[0]
    merr = np.abs(mel - z['mel_graph']).max()
    print(f'demo-03 GTA postnet mel vs graph: max {merr:.2e}')
    assert merr <= 1e-4


def test_gta_mels_end_to_end_demo03():
    """Synthesizer.gta_mels: text -> GPU encoder -> GTA decoder (Philox seed 0) -> postnet -> the reference's glue; against
    the oracle's encoder -> decode_gta with the same keep flags -> postnet -> the same glue, over the whole utterance."""
    from tacotronv2_wavernn_chinese_b200.tacotron.synthesizer import Synthesizer
    from tacotronv2_wavernn_chinese_b200.tacotron.text import Symbols
    w = _weights()
    z, n, _, targets = _gta_fixture()
    syn = Synthesizer()
    syn.symbols = Symbols(sentences()['symbols'])
    syn.engine = _engine(w)
    assert syn.symbols.text_to_sequence(str(z['pinyin'])) == list(z['ids'])
    mel = syn.gta_mels([str(z['pinyin'])], [np.load(os.path.join(GOLDEN, str(z['target_file'])))[str(z['target_key'])]])[0]
    assert mel.dtype == np.float32 and mel.shape == (n, 80) and mel.min() >= 0 and mel.max() <= 1
    masks = syn.engine.philox_masks(0, 0, 1, n).cpu().numpy()[0].astype(np.float32)
    ref = gta.decode_gta(w, to.encoder(w, z['ids']), targets, dropout_masks=masks)
    want = np.clip((np.clip(to.postnet(w, ref['frames']), -4, 4) + 4) / 8, 0, 1)
    err = np.abs(mel - want).max()
    print(f'gta_mels vs oracle on the [0, 1] scale: max {err:.2e}')
    assert err <= 1e-4


def _replay(w, mem, lengths, seed, offset, max_steps):
    eng = _engine(w)
    free = eng.decode(mem, lengths, seed=seed, utterance_offset=offset, max_steps=max_steps, want_align=True)
    n = free['nsteps'].cpu().numpy()
    gta = eng.decode_gta(mem, lengths, free['frames'], n, seed=seed, utterance_offset=offset, want_align=True)
    assert np.array_equal(gta['nsteps'].cpu().numpy(), n)
    ff, fa = free['frames'].cpu().numpy(), free['align'].cpu().numpy()
    gf, ga = gta['frames'].cpu().numpy(), gta['align'].cpu().numpy()
    for b in range(len(n)):
        assert np.array_equal(gf[b, :n[b]], ff[b, :n[b]]), b             # bit for bit over the whole run
        assert np.array_equal(ga[b, :n[b]], fa[b, :n[b]]), b
        assert not gf[b, n[b]:].any()                                   # rows beyond the step count untouched (zeros)
    return n


def test_gta_replays_a_free_run_bit_for_bit_real_checkpoint():
    """Three sentences decoded free-running at B = 3 (one block per sentence), then GTA on each row's own raw frames with the
    same Philox seed and offset: the same kernel source with the frame fed from memory instead of from the step before."""
    w = _weights()
    eng = _engine(w)
    s = sentences()['sentences']
    lengths = np.array([len(s[k]['ids']) for k in ('241', '48', '42')], dtype=np.int32)
    ids = np.zeros((3, lengths.max()), dtype=np.int32)
    for b, k in enumerate(('241', '48', '42')):
        ids[b, :lengths[b]] = s[k]['ids']
    mem = eng.encode(ids, lengths)
    n = _replay(w, mem, lengths, seed=1238, offset=5, max_steps=700)
    assert (n > 100).all() and (n < 700).all() and len(set(n.tolist())) == 3      # each row stopped by itself


def test_gta_replays_a_free_run_bit_for_bit_synthetic():
    w = synth_taco_weights(7)
    w['decoder/stop_token_projection/projection_stop_token_projection/bias'] = np.array([-3.0], dtype=np.float32)
    mem = np.random.RandomState(4).uniform(-1, 1, (3, 33, 512)).astype(np.float32)
    _replay(w, mem, np.array([33, 17, 25], np.int32), seed=9, offset=100, max_steps=64)


def test_ragged_batch_vs_oracle_and_batch_invariance():
    w = synth_taco_weights(7)
    eng = _engine(w)
    rs = np.random.RandomState(11)
    B, Tx, Ty = 3, 37, 48
    mem = rs.uniform(-1, 1, (B, Tx, 512)).astype(np.float32)
    lengths = np.array([37, 20, 29], dtype=np.int32)
    tlen = np.array([48, 30, 41], dtype=np.int32)
    targets = rs.uniform(-4, 4, (B, Ty, 80)).astype(np.float32)
    masks = (np.random.RandomState(5).uniform(size=(B, Ty, 2, 256)) >= 0.5).astype(np.uint8)
    out = eng.decode_gta(mem, lengths, targets, tlen, masks=masks, want_align=True)
    fr, al = out['frames'].cpu().numpy(), out['align'].cpu().numpy()
    for b in range(B):
        ref = gta.decode_gta(w, mem[b, :lengths[b]], targets[b, :tlen[b]], dropout_masks=masks[b])
        np.testing.assert_allclose(fr[b, :tlen[b]], ref['frames'], rtol=0, atol=1e-4)
        np.testing.assert_allclose(al[b, :tlen[b], :lengths[b]], ref['alignments'], rtol=0, atol=1e-5)
        assert not al[b, :, lengths[b]:].any() and not fr[b, tlen[b]:].any() and not al[b, tlen[b]:].any()
        solo = eng.decode_gta(mem[b:b + 1, :lengths[b]], None, targets[b:b + 1, :tlen[b]], None, masks=masks[b:b + 1, :tlen[b]],
                              want_align=True)
        assert np.array_equal(solo['frames'].cpu().numpy()[0], fr[b, :tlen[b]])
        assert np.array_equal(solo['align'].cpu().numpy()[0], al[b, :tlen[b], :lengths[b]])
    # Philox mode == EXT mode fed the keep flags Philox draws; rows keyed by the global sentence index
    ph = eng.decode_gta(mem, lengths, targets, tlen, seed=77, utterance_offset=10)['frames'].cpu().numpy()
    ext = eng.decode_gta(mem, lengths, targets, tlen, masks=eng.philox_masks(77, 10, B, Ty))['frames'].cpu().numpy()
    assert np.array_equal(ph, ext)
    one = eng.decode_gta(mem[1:2], lengths[1:2], targets[1:2], tlen[1:2], seed=77, utterance_offset=11)['frames'].cpu().numpy()
    assert np.array_equal(one[0], ph[1])
    # target lengths are clamped to [0, Ty_max]: 0 steps leaves the row untouched, > Ty_max runs Ty_max steps
    cl = eng.decode_gta(mem, lengths, targets, np.array([0, 1000, 48], np.int32), seed=77, utterance_offset=10)
    assert cl['nsteps'].cpu().numpy().tolist() == [0, Ty, Ty] and not cl['frames'].cpu().numpy()[0].any()


def test_gta_argument_errors_launch_nothing():
    import torch
    from tacotronv2_wavernn_chinese_b200 import _lib
    from tacotronv2_wavernn_chinese_b200._lib import TacoDropout
    w = synth_taco_weights(7)
    eng = _engine(w)
    lib = eng.lib
    B, Tx, Ty = 2, 9, 6
    dev = torch.device('cuda', eng.device)
    mem = torch.zeros(B, Tx, 512, device=dev)
    ln = torch.full((B,), Tx, dtype=torch.int32, device=dev)
    tg = torch.zeros(B, Ty, 80, device=dev)
    tl = torch.full((B,), Ty, dtype=torch.int32, device=dev)
    frames = torch.full((B, Ty, 80), 7.5, device=dev)
    align = torch.full((B, Ty, Tx), 7.5, device=dev)
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)
    good = TacoDropout()
    bad_mode = TacoDropout(); bad_mode.mode = 7
    ext_null = TacoDropout(); ext_null.mode = 1
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    base = dict(ctx=eng._h, mem=mem, ln=ln, B=B, Tx=Tx, d=C.byref(good), tg=tg, tl=tl, Ty=Ty, fr=frames, al=align)
    cases = [dict(ctx=None), dict(mem=None), dict(ln=None), dict(d=None), dict(tg=None), dict(tl=None), dict(fr=None),
             dict(B=0), dict(Tx=513), dict(Tx=0), dict(Ty=0), dict(d=C.byref(bad_mode)), dict(d=C.byref(ext_null))]
    for case in cases:
        a = dict(base, **case)
        ctx = a['ctx'] if a['ctx'] is not None else C.c_void_p(0)
        rc = lib.b200tts_taco_decode_gta(ctx, p(a['mem']), p(a['ln']), a['B'], a['Tx'], a['d'], p(a['tg']), p(a['tl']), a['Ty'],
                                         p(a['fr']), p(a['al']), stream)
        assert rc == -1, case
        assert lib.b200tts_last_error().decode(), case
    torch.cuda.synchronize()
    assert bool((frames == 7.5).all()) and bool((align == 7.5).all())
    # the same through the Python wrapper
    with pytest.raises(_lib.B200TTSError) as e:
        eng.decode_gta(np.zeros((1, 600, 512), np.float32), None, np.zeros((1, 4, 80), np.float32), None)
    assert e.value.code == -1
    with pytest.raises(ValueError):
        eng.decode_gta(np.zeros((1, 5, 512), np.float32), None, np.zeros((1, 4, 79), np.float32), None)


# ---------------------------------------------------------------- wavernn_preprocess.py end to end

def _checkpoint():
    if os.path.isfile(TRAVEL_COPY):
        return TRAVEL_COPY
    if os.path.isdir(REF_CKPT_DIR):
        return REF_CKPT_DIR
    pytest.skip('shipped Tacotron checkpoint not available on this box')


def _data_dir(root):
    """Three training lines in the layout tacotron_preprocess.py writes, made from the fixture PCMs with audio.preprocess_wav."""
    from tacotron_hparams import hparams
    from tacotronv2_wavernn_chinese_b200.tacotron import audio
    z = np.load(os.path.join(GOLDEN, 'mel_analysis_from_reference.npz'))
    pcms = [z['speech_pcm'], z['padded_pcm'], z['speech_pcm'][20000:60000]]
    texts = ['如果打穿地球，那么从一头到另一头h ui4发生什么？', '卡尔普陪外孙玩滑梯。', '假语村言别再拥抱我。']
    os.makedirs(root)
    lines = []
    for i, (pcm, text) in enumerate(zip(pcms, texts), 1):
        mel, out, _ = audio.preprocess_wav(pcm.astype(np.float32) / 32768.0, hparams)
        np.save(os.path.join(root, f'audio-{i:06d}.npy'), out, allow_pickle=False)
        np.save(os.path.join(root, f'mel-{i:06d}.npy'), mel, allow_pickle=False)
        lines.append(f'audio-{i:06d}.npy|mel-{i:06d}.npy|{len(out)}|{len(mel)}|{text}|-')
    with open(os.path.join(root, 'train.txt'), 'w', encoding='utf-8') as f:
        f.write('\n'.join(lines) + '\n')
    return root


def test_wavernn_preprocess_cli_end_to_end(tmp_path):
    import wavernn_preprocess
    ck = _checkpoint()
    data = _data_dir(str(tmp_path / 'data'))
    runs = {}
    for batch in (1, 3):
        out = tmp_path / f'out{batch}'
        idx = tmp_path / f'index{batch}.txt'
        wavernn_preprocess.main(['--data_dir', data, '--out_dir', str(out), '--index', str(idx), '--checkpoint', ck,
                                 '--symbols_json', os.path.join(GOLDEN, 'taco_symbols.json'), '--seed', '3',
                                 '--batch', str(batch)])
        rows = [l.split('|') for l in idx.read_text(encoding='utf-8').splitlines()]
        assert len(rows) == 3
        preds = []
        for i, row in enumerate(rows, 1):
            wav_path, mel_path, pred_path, text = row
            assert all(os.path.isabs(p) for p in row[:3])
            assert wav_path == str(out / f'audio-{i:06d}.npy') and mel_path == str(out / f'mel-{i:06d}.npy')
            assert pred_path == str(out / f'mel-{i:06d}-pred.npy') and text
            q = np.load(wav_path)
            src = np.load(os.path.join(data, f'audio-{i:06d}.npy'))
            assert q.shape == src.shape and (q == np.floor(q)).all() and q.min() >= 0 and q.max() <= 1023
            target = np.load(os.path.join(data, f'mel-{i:06d}.npy'))
            np.testing.assert_array_equal(np.load(mel_path), np.clip((target + 4.0) / 8.0, 0, 1))
            pred = np.load(pred_path)
            assert pred.dtype == np.float32 and pred.shape == target.shape and pred.min() >= 0 and pred.max() <= 1
            if i == 1:                                                          # the demo recording with its own text
                assert np.abs(pred - np.load(mel_path)).mean() < 0.1            # GTA: close to the recording frame for frame
            preds.append(open(pred_path, 'rb').read())
        runs[batch] = preds
    assert runs[1] == runs[3]                                                   # independent of --batch, byte for byte
