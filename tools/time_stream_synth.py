"""The streaming text-to-speech service on one GPU: batched against one-by-one session opens, then
pipeline.StreamingSynthesizer fed train.txt sentences at a fixed arrival rate.

    python tools/time_stream_synth.py [--frames 401] [--opens 1,32,128,256] [--rows 32,128] [--rate 6,24] [--requests 48,128]
                                      [--chunk 2750] [--decode_steps whole,8,32] [--slices 1,3,8,32,128] [--out FILE]

Prints the card name and power limit first, and writes the whole report as JSON to --out.
  * opens: host time (synchronised, median of 4 repeats after one warm-up) to open N sessions of `frames` frames one by one
    (open_session) and in one batch (open_sessions), push sessions up to 32 and tensor-core sessions above.  The sessions of
    both are run to their first piece and compared bit for bit.  Then where a one-by-one open's time goes: the Python call, the
    C call alone, its three launches (CUDA events) and a cudaMalloc + cudaFree of its one allocation, table and state (libcudart,
    median of 20).
  * service: at each max_rows, `requests` sentences of tests/golden/taco_symbols.json (cut from train.txt) arrive at `rate`
    per second, in order, round robin over the set.  Per request the time from arrival to its first piece on the host
    (p50 / p95); per admitting step the admission time (Tacotron encode + decode + postnet, stop cut and batched open, timed
    with a synchronisation around it) and the Tacotron batch size; per step its wall time against the audio each active stream
    received (chunk / sample rate): a stream keeps real time while step wall <= that duration.  The service runs once per
    --decode_steps value: 'whole' decodes each admission whole (the default service), k slices the decodes (decode_steps=k),
    and the per-step Tacotron time is then that of the slice, the finishing postnet and cut and the vocoder open.
  * slices: the Tacotron decoder sessions' step time at 1, 3, 8, 32 and 128 sessions, as the slope between slices of 8 and 40
    steps (CUDA events), on synthetic decoder weights whose stop never fires.
Synthetic vocoder weights (time does not depend on their values); the Tacotron travel copy oracle/_ref/tacotron_weights.npz,
whose stop tokens decide the mel lengths.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tacotronv2_wavernn_chinese_b200 import pipeline, synth                 # noqa: E402
from tacotronv2_wavernn_chinese_b200.engine import WaveRNNEngine              # noqa: E402

SR = 22050


def _sync():
    torch.cuda.synchronize()


def _median_ms(f, reps=4):
    t = []
    for rep in range(reps + 1):
        _sync()
        t0 = time.perf_counter()
        out = f()
        _sync()
        if rep:
            t.append(time.perf_counter() - t0)
        for s in out:
            s.close()
    return float(np.median(t)) * 1e3


def opens(eng, frames, ns):
    res = []
    for n in ns:
        kernel = 'auto' if n <= 32 else 'tc'
        mels = synth.synth_mels(n, n, frames)
        d = torch.as_tensor(mels).cuda()
        ids = list(range(n))
        one = lambda: [eng.open_session(d[i], seed=1, utterance_id=i, kernel=kernel) for i in range(n)]   # noqa: E731
        batch = lambda: eng.open_sessions(d, [frames] * n, seed=1, utterance_ids=ids, kernel=kernel)       # noqa: E731
        t_one, t_batch = _median_ms(one), _median_ms(batch)
        a, b = one(), batch()
        pa = eng.advance(a, 2750)
        pb = eng.advance(b, 2750)
        equal = all(torch.equal(x[1], y[1]) for x, y in zip(pa, pb))
        eng.check()
        for s in a + b:
            s.close()
        res.append(dict(n=n, kernel=kernel, one_by_one_ms=t_one, batch_ms=t_batch, first_piece_equal=bool(equal)))
        print(f'open {n:3d} x {frames} frames ({kernel}): one by one {t_one:8.2f} ms, one batch {t_batch:7.2f} ms, equal {equal}')
    return res


def open_split(eng, frames):
    """Where one session_open's time goes."""
    import ctypes as C
    from tacotronv2_wavernn_chinese_b200 import _lib
    from tacotronv2_wavernn_chinese_b200.engine import _rng
    d = torch.as_tensor(synth.synth_mels(3, 1, frames)[0]).cuda().contiguous()
    st = torch.cuda.current_stream()
    py, capi, kern = [], [], []
    for rep in range(21):
        _sync()
        t0 = time.perf_counter()
        s = eng.open_session(d, seed=1, utterance_id=rep)
        _sync()
        py.append(time.perf_counter() - t0)
        s.close()
        rng = _rng(_lib.RNG_PHILOX, 1, rep)
        h = C.c_void_p()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        _sync()
        t0 = time.perf_counter()
        e0.record(st)
        _lib.check(eng.lib.b200tts_wavernn_session_open(eng._h, C.c_void_p(d.data_ptr()), frames, C.byref(rng), 1, C.byref(h),
                                                        C.c_void_p(st.cuda_stream)))
        e1.record(st)
        _sync()
        capi.append(time.perf_counter() - t0)
        kern.append(e0.elapsed_time(e1) * 1e-3)
        eng.lib.b200tts_wavernn_session_destroy(h)
    out = dict(python_call_ms=float(np.median(py[1:])) * 1e3, c_call_ms=float(np.median(capi[1:])) * 1e3,
               launches_gpu_ms=float(np.median(kern[1:])) * 1e3)
    try:
        rt = ctypes.CDLL('libcudart.so.12')
        nbytes = ((frames + 1) * 128 * 52 + 4160) * 4         # the table of 128 CTAs, then the state (4 100 floats, 256-byte aligned)
        t = []
        p = ctypes.c_void_p()
        for rep in range(21):
            t0 = time.perf_counter()
            assert rt.cudaMalloc(ctypes.byref(p), ctypes.c_size_t(nbytes)) == 0
            assert rt.cudaFree(p) == 0
            t.append(time.perf_counter() - t0)
        out['cudaMalloc_free_ms'] = float(np.median(t[1:])) * 1e3
    except OSError as e:
        out['cudaMalloc'] = f'not measured: {e}'
    print('one open of', frames, 'frames:', json.dumps(out))
    return out


def slices(ns, Tx=64, k1=8, k2=40):
    """us per decoder step of a slice of n sessions: (t(k2) - t(k1)) / (k2 - k1), each the median of 5 (CUDA events)."""
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    from taco_common import synth_taco_weights
    from tacotronv2_wavernn_chinese_b200.tacotron.engine import TacoDecoderEngine
    w = synth_taco_weights(3)
    w['decoder/stop_token_projection/projection_stop_token_projection/bias'][:] = -1e4
    te = TacoDecoderEngine(w, device=0)
    res = []
    for n in ns:
        mem = torch.as_tensor(np.random.RandomState(n).uniform(-1, 1, (n, Tx, 512)).astype(np.float32)).cuda()
        ms = {}
        for k in (k1, k2):
            t = []
            for rep in range(6):
                ss = te.open_decode_sessions(mem, None, list(range(n)), max_steps=k)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                _sync()
                e0.record()
                te.advance_decodes(ss, k)
                e1.record()
                _sync()
                if rep:
                    t.append(e0.elapsed_time(e1))
                for s in ss:
                    s.close()
            ms[k] = float(np.median(t))
        us = (ms[k2] - ms[k1]) / (k2 - k1) * 1e3
        res.append(dict(sessions=n, us_per_step=us, slice_ms={str(k): v for k, v in ms.items()}))
        print(f'decoder slice, {n:3d} sessions: {us:7.1f} us per step')
    te.close()
    return res


def service(syn, eng, texts, rows, rate, nreq, chunk, decode_steps=None):
    ss = pipeline.StreamingSynthesizer(syn, eng, seed=3, chunk_steps=chunk, max_rows=rows, decode_steps=decode_steps)
    admits = []
    name = '_admit' if decode_steps is None else '_decode_slice'
    admit = getattr(ss, name)

    def timed_admit():
        k = len(ss._queue)
        busy = k and ss.max_rows > len(ss._active) + len(ss._decoding) or ss._decoding
        _sync()
        t0 = time.perf_counter()
        out = admit()
        _sync()
        if busy:
            admits.append(dict(n=k - len(ss._queue), ms=(time.perf_counter() - t0) * 1e3))
        return out

    setattr(ss, name, timed_admit)
    arrival = [i / rate for i in range(nreq)]
    first, steps = {}, []
    t0 = time.perf_counter()
    nxt = 0
    while nxt < nreq or not ss.idle():
        now = time.perf_counter() - t0
        while nxt < nreq and arrival[nxt] <= now:
            ss.submit(nxt, texts[nxt % len(texts)], nxt)
            nxt += 1
        if ss.idle():
            time.sleep(max(0.0, arrival[nxt] - now))
            continue
        s0 = time.perf_counter()
        queued = ss.pending
        active = ss.active
        out = ss.step()
        s1 = time.perf_counter()
        for key, piece, _fin in out:
            if key not in first and len(piece):
                first[key] = s1 - t0 - arrival[key]
        steps.append(dict(wall_ms=(s1 - s0) * 1e3, streams=len(out), admitted=ss.pending < queued, active_before=active))
    audio_ms = chunk / SR * 1e3
    ttfa = np.array([first[k] for k in sorted(first)]) * 1e3
    walls = np.array([s['wall_ms'] for s in steps])
    adm = np.array([s['admitted'] for s in steps])
    res = dict(decode_steps=decode_steps or 'whole', max_rows=rows, rate_per_s=rate, requests=nreq, chunk_steps=chunk,
               chunk_audio_ms=audio_ms,
               ttfa_ms_p50=float(np.percentile(ttfa, 50)), ttfa_ms_p95=float(np.percentile(ttfa, 95)),
               taco_steps=len(admits), taco_ms_p50=float(np.median([a['ms'] for a in admits])),
               taco_ms_max=float(max(a['ms'] for a in admits)),
               admit_batch_mean=float(np.mean([a['n'] for a in admits if a['n']] or [0])),
               admit_per_batch=[(a['n'], round(a['ms'], 2)) for a in admits],
               steps=len(steps), step_wall_ms_p50=float(np.median(walls)), step_wall_ms_p95=float(np.percentile(walls, 95)),
               step_wall_ms_p50_admitting=float(np.median(walls[adm])) if adm.any() else None,
               step_wall_ms_p50_not_admitting=float(np.median(walls[~adm])) if (~adm).any() else None,
               real_time_steps=float(np.mean(walls <= audio_ms)),
               real_time_steps_admitting=float(np.mean(walls[adm] <= audio_ms)) if adm.any() else None,
               real_time_steps_not_admitting=float(np.mean(walls[~adm] <= audio_ms)) if (~adm).any() else None,
               max_active=int(max(s['active_before'] for s in steps)))
    print('service:', json.dumps({k: v for k, v in res.items() if k != 'admit_per_batch'}))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=401)
    ap.add_argument('--opens', default='1,32,128,256')
    ap.add_argument('--rows', default='32,128')
    ap.add_argument('--rate', default='6,24', help='arrivals per second, one per --rows entry')
    ap.add_argument('--requests', default='48,128', help='requests, one per --rows entry')
    ap.add_argument('--chunk', type=int, default=2750)
    ap.add_argument('--decode_steps', default='whole', help="'whole' and / or slice lengths k, comma-separated")
    ap.add_argument('--slices', default='1,3,8,32,128', help='session counts of the decoder slice timing (empty: none)')
    ap.add_argument('--out', default='')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('time_stream_synth.py needs a CUDA device')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    card = q.stdout.strip() or 'unknown'
    print('card:', card)
    torch.cuda.set_device(0)
    eng = WaveRNNEngine(synth.synth_state_dict(0), synth.DEFAULT_DIMS, device=0)
    report = dict(card=card, frames=a.frames, opens=opens(eng, a.frames, [int(x) for x in a.opens.split(',')]),
                  one_open_split=open_split(eng, a.frames), service=[])
    w = os.path.join(ROOT, 'oracle', '_ref', 'tacotron_weights.npz')
    if os.path.isfile(w):
        from tacotronv2_wavernn_chinese_b200.tacotron.engine import TacoDecoderEngine
        from tacotronv2_wavernn_chinese_b200.tacotron.synthesizer import Synthesizer
        from tacotronv2_wavernn_chinese_b200.tacotron.text import Symbols
        gold = json.load(open(os.path.join(ROOT, 'tests', 'golden', 'taco_symbols.json')))
        syn = Synthesizer()
        syn.symbols = Symbols(gold['symbols'])
        syn.engine = TacoDecoderEngine(dict(np.load(w)), device=0)
        texts = [syn.symbols.sequence_to_text(v['ids'][:-1]) for _k, v in sorted(gold['sentences'].items(), key=lambda kv: int(kv[0]))]
        syn.decode_device(texts[:2], [0, 1])                    # warm-up
        for ds in a.decode_steps.split(','):
            for rows, rate, nreq in zip(*[[int(x) for x in v.split(',')] for v in (a.rows, a.rate, a.requests)]):
                report['service'].append(service(syn, eng, texts, rows, rate, nreq, a.chunk, None if ds == 'whole' else int(ds)))
    else:
        report['service'] = 'not measured: no Tacotron weights at oracle/_ref/tacotron_weights.npz'
        print(report['service'])
    report['slices'] = slices([int(x) for x in a.slices.split(',')]) if a.slices else []
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(report, f, indent=1)


if __name__ == '__main__':
    main()
