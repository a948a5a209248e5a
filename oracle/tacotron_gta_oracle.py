"""CPU oracle for ground-truth-aligned (GTA) decoding, the teacher-forced decoder loop of the reference's wavernn_preprocess.py
-- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The per-step arithmetic is oracle/tacotron_oracle.py's `decoder_step` (pinned against the reference's serialized graph, see
that module); this file adds only the loop driver of `TacoTrainingHelper`.  Its float type is `tacotron_oracle.F32`, read at
call time, so a test that evaluates that module in float64 evaluates this loop in float64 too.  Pins:
  * tests/test_tacotron_gta_pins.py: `decode_gta` reproduces every frame and attended position of the demo recording
    teacher-forced through the serialized step graph with the reference's own TacoTrainingHelper (oracle/make_golden_taco_gta.py
    -> tests/golden/taco_gta_from_graph.npz; measured difference 0.0 over 323 steps), and fed the 405 frames of the free-running
    graph run (tests/golden/taco_run_from_graph.npz) it replays that run exactly.

Only tests/ and oracle/ may import this module.  Reference citations are relative to the reference root.
"""
from __future__ import annotations

import numpy as np

import oracle.tacotron_oracle as to


def decode_gta(w, memory, targets, dropout_masks=None, seed=0, zoneout=to.GRAPH_ASSUMPTIONS['zoneout']):
    """The teacher-forced decoder loop of wavernn_preprocess.py for ONE sentence: dynamic_decode(CustomDecoder(
    TacotronDecoderCell, TacoTrainingHelper)) with `is_evaluating=True` (wavernn_preprocess.py:46-47; tacotron.py:86-103).
    TacoTrainingHelper (helpers.py:69-151), restated:
      * first input: the all-zero GO frame (initialize, :124 -> _go_frames, :149-151);
      * next input after step `time`: always targets[:, time, :] (:142; the teacher-forcing-ratio branch is commented out,
        :136-141), r = 1 so the targets are not subsampled (:84);
      * finished = time + 1 >= len(targets) (:132, :93) with max_iters None (tacotron.py:96): exactly len(targets) steps, no
        stop rule.
    The attention is built with is_training=True (tacotron.py:66), so no inference window; prenet dropout stays on
    (modules.py:249) and draws the same RandomState stream as `tacotron_oracle.decode`.

    memory [Tx, 512]; targets [Ty, 80] used as given (the caller clips, wavernn_preprocess.py:79).
    Returns dict(frames [Ty,80] raw decoder outputs, alignments [Ty,Tx], n_steps, masks)."""
    F32 = to.F32
    Tx = memory.shape[0]
    keys = (memory @ w['memory_layer/kernel']).astype(F32)
    U = w[to.P + 'decoder_LSTM/multi_rnn_cell/cell_0/decoder_LSTM_1/kernel'].shape[1] // 4
    rs = np.random.RandomState(seed)
    zeros = np.zeros((1, U), dtype=F32)
    alpha0 = np.zeros(Tx, dtype=F32)
    alpha0[0] = 1
    st = dict(c1=zeros, h1=zeros, c2=zeros, h2=zeros, ctx=np.zeros((1, memory.shape[1]), dtype=F32),
              alpha=alpha0, cum=alpha0.copy(), mu=F32(0.5))
    x = np.zeros((1, 80), dtype=F32)                                                         # _go_frames (helpers.py:149)
    frames, aligns, masks = [], [], []
    for step in range(len(targets)):
        if dropout_masks is not None:
            m = dropout_masks[step]
        else:
            m = rs.uniform(size=(2, 256)) >= to.GRAPH_ASSUMPTIONS['prenet_dropout_rate']
        m = np.asarray(m, dtype=F32)
        masks.append(m)
        out, st = to.decoder_step(w, memory, keys, x, m, st, zoneout)
        frames.append(out['frame'][0])
        aligns.append(out['alignments'])
        x = np.asarray(targets[step], dtype=F32)[None]                                       # helpers.py:142
    return dict(frames=np.stack(frames), alignments=np.stack(aligns), n_steps=len(frames), masks=np.stack(masks))
