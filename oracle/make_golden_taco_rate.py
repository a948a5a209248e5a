"""Golden vectors for the speaking-rate bias of the forward attention (attention.py:163-165, forward_attention.py:163-165: the
branch the reference ships switched off with `and False`), produced by the reference's own
`ForwardLocationSensitiveAttention.__call__` of BOTH attention files with that branch switched on at a given delta
(oracle/ref_harness_taco_rate.py: an edit of the parsed file in memory; every other statement runs unmodified on numpy
arrays).  The oracle side is oracle/tacotron_rate_oracle.py.  TEST INFRASTRUCTURE; run HERE (needs /root/reference).

States come from the oracle's own biased runs of train.txt line 241 on the shipped checkpoint (seed-1238 masks), without the
window through attention.py and with it through forward_attention.py, at every delta of DELTAS.  Each state is what the
recursion sees at one step (query, alpha, cumulated alignments, the UNBIASED mu, window registers); the record is what the
reference's `__call__` returns for it: alignments, new mu, context, cumulated alignments, max_attentions, pos_rec.  At
delta = +-1 every step clips (mu + delta >= 1 or <= 0).

    python oracle/make_golden_taco_rate.py        ->  tests/golden/taco_rate_from_reference.npz
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)

import ref_harness_taco_attention as R                     # noqa: E402
import ref_harness_taco_rate as RR                         # noqa: E402
import tacotron_oracle as to                               # noqa: E402
import tacotron_rate_oracle as tro                         # noqa: E402
from tacotronv2_wavernn_chinese_b200.tacotron import ckpt  # noqa: E402

CKPT_DIR = os.path.join(R.REF_ROOT, 'logs-Tacotron-2/taco_pretrained')
DELTAS = (-1.0, -0.3, -0.04, 0.04, 0.3, 1.0)
FILES = (('attention.py', False), ('forward_attention.py', True))     # (reference file, window)
N_RUN = 150                                                            # steps of each biased run the states are taken from


def _state(st, win):
    return R.State(alignments=st['alpha'][None], cumulated_alignments=st['cum'][None], alpha=st['alpha'][None],
                   mu=np.reshape(st['mu'], (1, 1)).astype(np.float32), max_attentions=np.array([win['max_att']], np.int32),
                   pos_rec=np.array([win['pos_rec']], np.int32))


def main():
    w = ckpt.load_tacotron_weights(CKPT_DIR)
    ids = np.array(json.load(open(os.path.join(ROOT, 'tests', 'golden', 'taco_symbols.json')))['sentences']['241']['ids'])
    memory = to.encoder(w, ids)
    keys = (memory @ w['memory_layer/kernel']).astype(np.float32)
    rows, worst = [], {}
    for file, window in FILES:
        # delta = 0 with the branch switched on is the shipped file: same outputs, bit for bit
        d0 = to.decode(w, memory, seed=1238, max_iters=12, window=window, capture_states=range(12))
        plain, on0 = RR.ReferenceRateAttention(w, memory, file, None), RR.ReferenceRateAttention(w, memory, file, 0.0)
        for s in sorted(d0['states']):
            x, st, m, win = d0['states'][s]
            o, _ = to.decoder_step(w, memory, keys, x, m, st)
            a, b = plain(o['new_h2'], _state(st, win)), on0(o['new_h2'], _state(st, win))
            assert all(np.array_equal(np.asarray(u), np.asarray(v)) for u, v in zip(a, b)), (file, s)
            if window:                          # the class re-executed from the parsed file is the imported one
                c = R.ReferenceAttention(w, memory)(o['new_h2'], _state(st, win))
                assert all(np.array_equal(np.asarray(u), np.asarray(v)) for u, v in zip(a, c)), (file, s)
        for delta in DELTAS:
            d = tro.decode(w, memory, seed=1238, max_iters=N_RUN, window=window, capture_states=range(N_RUN), mu_bias=delta)
            att = RR.ReferenceRateAttention(w, memory, file, delta)
            n = d['n_steps']
            keep = sorted({s for s in range(n) if s < 3 or s % 19 == 0} | {n - 1})
            for s in keep:
                x, st, m, win = d['states'][s]
                mod = (lambda al, win=win: to.attention_window(al, win['max_att'], win['pos_rec'])[0]) if window else None
                o, _ = tro.decoder_step(w, memory, keys, x, m, st, modulate=mod, mu_bias=delta)
                new_max, new_pos = (to.attention_window(o['forward_raw'], win['max_att'], win['pos_rec'])[1:] if window
                                    else (int(np.argmax(o['forward_raw'])), win['pos_rec']))
                al, mu, ctx, cum, mx, pr = att(o['new_h2'], _state(st, win))
                rows.append(dict(delta=np.float32(delta), window=np.int32(window), step=s, query=o['new_h2'][0], alpha=st['alpha'],
                                 cum=st['cum'], mu=np.float32(st['mu']), max_att=win['max_att'], pos_rec=win['pos_rec'],
                                 ref_alignments=np.asarray(al)[0], ref_mu=np.asarray(mu)[0, 0], ref_context=np.asarray(ctx)[0],
                                 ref_cum=np.asarray(cum)[0], ref_max_att=int(mx[0]), ref_pos_rec=int(pr[0])))
                for k, (u, v) in dict(alignments=(o['alignments'], al[0]), mu=(o['mu'], mu[0, 0]), context=(o['context'][0], ctx[0]),
                                      max_att=(new_max, mx[0]), pos_rec=(new_pos, pr[0])).items():
                    worst[k] = max(worst.get(k, 0.0), float(np.abs(np.asarray(u, np.float64) - np.asarray(v, np.float64)).max()))
            print(f'{file:22s} delta {delta:+.2f}: run of {n} steps (cap {N_RUN}), {len(keep)} states', flush=True)
    out = {'ids': ids, 'memory': memory}
    for k in rows[0]:
        out[k] = np.stack([np.asarray(r[k]) for r in rows])
    path = os.path.join(ROOT, 'tests', 'golden', 'taco_rate_from_reference.npz')
    np.savez_compressed(path, **out)
    lo = int(((out['mu'] + out['delta']) <= 0).sum())
    hi = int(((out['mu'] + out['delta']) >= 1).sum())
    print(f'wrote {path} ({os.path.getsize(path)} bytes, {len(rows)} states; {lo} clip at 0, {hi} clip at 1); '
          f'oracle vs the reference statements, max abs difference:')
    for k, v in worst.items():
        print(f'  {k:11s} {v:.3e}')


if __name__ == '__main__':
    main()
