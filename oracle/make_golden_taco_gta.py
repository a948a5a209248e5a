"""WHOLE-RUN golden for ground-truth-aligned (GTA) decoding, the teacher-forced loop of the reference's
`wavernn_preprocess.py`, produced by driving the reference's own serialized decoder-step graph -- container only (needs
/root/reference).

TEST INFRASTRUCTURE.  The case is the reference's demo recording `demo/03-forward-griffin_lim.wav` with its own text
(TEXT below): the target mel is `speech_mel` of tests/golden/mel_analysis_from_reference.npz (the reference's
`_process_utterance_v1` on that recording, oracle/make_golden_mel_analysis.py), clipped to +-4 as wavernn_preprocess.py:79
does; it is NOT copied into this fixture, which names the key instead.  Per step:
  * cells, attention and projections: the serialized `decoder/while/CustomDecoderStep/*` sub-graph evaluated by
    oracle/tf_graph_eval.py on the shipped checkpoint (oracle/make_golden_taco_step.run_graph_step), inference zoneout between
    steps (modules.py:137-138), as in oracle/make_golden_taco_run.py;
  * the next input and the step count: the reference's OWN `TacoTrainingHelper` (tacotron/models/helpers.py:69-151; hparams of
    the shipped model, is_evaluating=True as wavernn_preprocess.py:46-47 builds it) executed on numpy values through a
    stand-in for the few tensorflow ops it touches -- its `initialize` gives the GO frame, its `next_inputs` the next input and
    `finished`.  The serialized graph is the training graph and does contain the helper, but its next-input slice reads the
    targets through the while-loop's frame ops, which the op interpreter does not evaluate.
The encoder memory is the serialized encoder's (make_golden_taco_run.encoder_through_graph), the mel the serialized postnet's.
The prenet keep-masks are RandomState(SEED) draws, [steps, 2, 256], packed like tests/golden/taco_run_from_graph.npz.

    python oracle/make_golden_taco_gta.py        ->  tests/golden/taco_gta_from_graph.npz
                                                     tests/golden/train_txt_lengths.npz

The second file is the length distribution of the reference's train.txt -- mel frames (4th field) and pinyin tokens (6th
field) of each of its 10 000 lines -- the workload tools/time_taco_gta.py times GTA decoding on.
"""
from __future__ import annotations

import contextlib
import importlib.util
import json
import os
import sys
import time
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)

import tacotron_oracle as to                               # noqa: E402
from oracle.tacotron_gta_oracle import decode_gta           # noqa: E402
import tf_graph_eval as E                                   # noqa: E402
from make_golden_taco_graph import DEFAULT_META            # noqa: E402
from make_golden_taco_step import CKPT_DIR, run_graph_step  # noqa: E402
from make_golden_taco_run import encoder_through_graph, postnet_through_graph   # noqa: E402
from ref_harness_taco_attention import REF_ROOT            # noqa: E402
from tacotronv2_wavernn_chinese_b200.tacotron import ckpt  # noqa: E402
from tacotronv2_wavernn_chinese_b200.tacotron.pinyin import get_pyin   # noqa: E402
from tacotronv2_wavernn_chinese_b200.tacotron.text import Symbols      # noqa: E402

F32 = np.float32
SEED = 1238
TEXT = '如果打穿地球，那么从一头到另一头h ui4发生什么？'      # demo/03-forward-griffin_lim.wav's text (index.html:106)
TARGET = ('mel_analysis_from_reference.npz', 'speech_mel')
PROBES = (0, 1, 2, 161, 321, 322)                           # times at which the helper's next input is recorded


def reference_training_helper(targets):
    """The reference's own `TacoTrainingHelper` (helpers.py:69-146) for a batch of targets [B, T, 80], on numpy values:
    hparams of the shipped model (outputs_per_step 1, use_all_outputs False, natural eval, constant teacher forcing),
    gta=False and evaluating=True as Tacotron.initialize passes them (tacotron.py:33, :87-88)."""
    tf = types.ModuleType('tensorflow')
    tf.name_scope = lambda *a, **k: contextlib.nullcontext()
    tf.tile = lambda x, m: np.tile(np.asarray(x), m)
    tf.shape = lambda x: np.array(np.shape(x), dtype=np.int32)
    tf.convert_to_tensor = lambda x, dtype=None: np.asarray(x)
    tf.TensorShape = lambda x: tuple(x)
    seq2seq = types.ModuleType('tensorflow.contrib.seq2seq')
    seq2seq.Helper = type('Helper', (), {})
    fake = {'tensorflow': tf, 'tensorflow.contrib': types.ModuleType('tensorflow.contrib'), 'tensorflow.contrib.seq2seq': seq2seq}
    saved = {k: sys.modules.get(k) for k in fake}
    sys.modules.update(fake)
    try:
        spec = importlib.util.spec_from_file_location('_ref_helpers', os.path.join(REF_ROOT, 'tacotron/models/helpers.py'))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    hp = types.SimpleNamespace(outputs_per_step=1, use_all_outputs=False, num_mels=80, tacotron_teacher_forcing_ratio=1.,
                               tacotron_natural_eval=True, tacotron_teacher_forcing_mode='constant')
    return mod.TacoTrainingHelper(batch_size=np.shape(targets)[0], targets=np.asarray(targets), hparams=hp, gta=False,
                                  evaluating=True, global_step=None)


def drive_graph_gta(nodes, variables, memory, keys, targets, masks, zoneout=0.1):
    """The teacher-forced loop: graph step, zoneout, then the helper picks the next input and decides `finished`."""
    Tx, U = memory.shape[0], 256
    z = F32(zoneout)
    zeros = np.zeros((1, U), dtype=F32)
    alpha0 = np.zeros(Tx, dtype=F32)
    alpha0[0] = 1
    st = dict(c1=zeros, h1=zeros, c2=zeros, h2=zeros, ctx=np.zeros((1, memory.shape[1]), dtype=F32), alpha=alpha0, cum=alpha0.copy(),
              mu=F32(0.5))
    zoned = lambda new, prev: ((F32(1) - z) * new + z * prev).astype(F32)
    helper = reference_training_helper(targets[None])
    finished, x = helper.initialize()
    go = np.asarray(x, dtype=F32).copy()
    x = go
    frames, aligns, fin, probes = [], [], [], {}
    step = 0
    while True:
        g = run_graph_step(nodes, variables, memory, keys, np.asarray(x, dtype=F32).reshape(1, 80), masks[step].astype(F32), st)
        st = dict(c1=zoned(g['new_c1'], st['c1']), h1=zoned(g['new_h1'], st['h1']), c2=zoned(g['new_c2'], st['c2']),
                  h2=zoned(g['new_h2'], st['h2']), ctx=np.asarray(g['context'], dtype=F32).reshape(1, -1),
                  alpha=np.asarray(g['alignments'], dtype=F32).reshape(-1), cum=np.asarray(g['cum'], dtype=F32).reshape(-1),
                  mu=F32(np.asarray(g['mu']).reshape(-1)[0]))
        frame = np.asarray(g['frame'], dtype=F32).reshape(1, 80)
        frames.append(frame[0]); aligns.append(st['alpha'].copy())
        finished, x, _ = helper.next_inputs(step, frame, None, None, None)
        fin.append(bool(np.all(finished)))
        if step in PROBES:
            probes[step] = np.asarray(x, dtype=F32).reshape(80).copy()
        if np.all(finished):
            break
        step += 1
    return np.stack(frames), np.stack(aligns), go[0], np.array(fin), probes


def write_train_txt_lengths():
    frames, tokens = [], []
    with open(os.path.join(REF_ROOT, 'train.txt'), encoding='utf-8') as f:
        for line in f:
            fields = line.strip().split('|')
            frames.append(int(fields[3]))
            tokens.append(len(fields[5].split()))
    path = os.path.join(ROOT, 'tests', 'golden', 'train_txt_lengths.npz')
    np.savez_compressed(path, mel_frames=np.array(frames, np.int16), pinyin_tokens=np.array(tokens, np.int16))
    print(f'wrote {path}: {len(frames)} lines, {min(frames)}-{max(frames)} frames ({sum(frames)} in all), '
          f'{min(tokens)}-{max(tokens)} tokens')


def main():
    write_train_txt_lengths()
    nodes = E.load_graph(DEFAULT_META)
    variables = ckpt.load_bundle(CKPT_DIR)
    w = ckpt.load_tacotron_weights(CKPT_DIR)
    symbols = Symbols(json.load(open(os.path.join(ROOT, 'tests', 'golden', 'taco_symbols.json')))['symbols'])
    pyin, _ = get_pyin(TEXT)
    ids = np.array(symbols.text_to_sequence(pyin))
    targets = np.clip(np.load(os.path.join(ROOT, 'tests', 'golden', TARGET[0]))[TARGET[1]], -4.0, 4.0).astype(F32)
    n = targets.shape[0]
    mem_g = encoder_through_graph(nodes, variables, ids)
    keys = (mem_g @ w['memory_layer/kernel']).astype(F32)
    masks = (np.random.RandomState(SEED).uniform(size=(n, 2, 256)) >= 0.5)
    t0 = time.time()
    frames, aligns, go, fin, probes = drive_graph_gta(nodes, variables, mem_g, keys, targets, masks)
    print(f'graph-driven teacher-forced run: {len(frames)} steps ({n} target frames) in {time.time() - t0:.1f} s')
    d = decode_gta(w, mem_g, targets, dropout_masks=masks.astype(F32))
    err = np.abs(d['frames'] - frames).max(axis=1)
    print(f'  oracle decode_gta vs graph: frames max {err.max():.3e} (step {int(err.argmax())}), alignments max '
          f'{np.abs(d["alignments"] - aligns).max():.3e}, attention ends on token {int(aligns[-1].argmax())} of {len(ids)}')
    mel_g = postnet_through_graph(nodes, variables, frames)
    print(f'  postnet mel: graph vs oracle {np.abs(mel_g - to.postnet(w, frames)).max():.3e}')
    path = os.path.join(ROOT, 'tests', 'golden', 'taco_gta_from_graph.npz')
    np.savez_compressed(path, text=np.array(TEXT), pinyin=np.array(pyin), ids=ids, target_file=np.array(TARGET[0]),
                        target_key=np.array(TARGET[1]), target_clip=np.array(4.0), seed=np.array(SEED), n_steps=np.array(len(frames)),
                        memory_graph=mem_g, frames=frames, mel_graph=mel_g,
                        align_argmax=aligns.argmax(1).astype(np.int16), align_peak=aligns.max(1).astype(F32),
                        masks=np.packbits(masks.reshape(n, -1), axis=1),
                        helper_go=go, helper_finished=fin, helper_probe_times=np.array(sorted(probes)),
                        helper_probe_next=np.stack([probes[t] for t in sorted(probes)]))
    print(f'wrote {path} ({os.path.getsize(path)} bytes)')


if __name__ == '__main__':
    main()
