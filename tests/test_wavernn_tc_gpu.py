"""The tensor-core WaveRNN step (`wavernn_tc_kernel`, csrc/wavernn_tc.cuh) against the float32 oracle where short runs do not reach:
whole utterances at the benchmark's shape (the last frames: FIR taps past the end, the last frame's aux rows, the wave epilogue),
external noise beyond the first 128-row group, a lone live row in the second group, step counts that end inside a conditioning
block, per-row utterance ids, and a real mel.  Shipped checkpoint; the oracle is pinned to the reference by
tests/test_oracle_golden.py."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import wavernn_oracle as wo
from tacotronv2_wavernn_chinese_b200 import synth
from test_wavernn_gpu import _distinct_cond, _padded, engine_for, torch_cuda  # noqa: F401  (torch_cuda is a fixture)

pytestmark = pytest.mark.gpu

HOP, NC = 275, 1024
TC = 'wavernn_tc_kernel'
NEAR_TIE_CAP = 5          # draws per case that may differ from the oracle, each a confirmed sampling near-tie (config 2 allows 5)


def _bar(want):
    """The logit bar of every WaveRNN parity test: 5e-6 * max|logit| + 1e-4."""
    return 5e-6 * max(1.0, float(np.abs(want).max())) + 1e-4


def _philox_rows(eng, seed, rows, steps, chunk=20000):
    """The Exp(1) noise PHILOX mode draws for the given global rows, [steps, len(rows), NC] on the host (copied chunk by chunk)."""
    q = np.empty((steps, len(rows), NC), np.float32)
    for i, r in enumerate(rows):
        for s0 in range(0, steps, chunk):
            n = min(chunk, steps - s0)
            q[s0:s0 + n, i] = eng.philox_exponential(seed, r, 1, s0, n)[:, 0].cpu().numpy()
    return q


def _draws_agree(p, mels, q, teacher, cond, got, want, logits=None, what=''):
    """The oracle, teacher-forced on `teacher` [R, S] with noise `q` [steps, R, NC], drew `want` [R, steps]; the kernel, fed the same
    labels, drew `got`.  Each step is then an independent draw from the same state, so every step where the two differ must be a
    near-tie of the sampling race in the oracle's own logits (top-2 gap of l - log q below 1e-3 * max(1, |top|)), and there may be
    at most NEAR_TIE_CAP of them.  `logits` ({step: [R, NC]}) may hold the oracle's logits already; missing steps are recomputed in
    one pass.  Returns the (row, step, gap) of each accepted near-tie."""
    rr, tt = np.nonzero(got != want)
    where = list(zip(rr.tolist()[:8], tt.tolist()[:8]))
    assert rr.size <= NEAR_TIE_CAP, f'{what}: {rr.size} draws differ from the oracle; first (row, step): {where}'
    logits = dict(logits or {})
    need = sorted(set(tt.tolist()) - set(logits))
    if need:
        logits.update(wo.generate(p, mels, q=q[:need[-1] + 1], teacher=teacher, keep_logits=need, max_steps=need[-1] + 1,
                                  cond=cond)['logits'])
    ties = []
    for i, t in zip(rr.tolist(), tt.tolist()):
        key = logits[t][i].astype(np.float64) - np.log(q[t, i].astype(np.float64))
        top = np.sort(key)[-2:]
        gap = float(top[1] - top[0])
        assert gap < 1e-3 * max(1.0, abs(top[1])), f'{what}: row {i} step {t}: the draw differs without a sampling near-tie (gap {gap:.3e})'
        ties.append((i, t, gap))
    return ties


def _whole_utterance_vs_oracle(torch, mels, seed, rows, probe):
    """Free-run all rows with Philox; teacher-force the kernel on its own labels (it must redraw them bit for bit); teacher-force
    the oracle on the kernel's labels of `rows` over every step with the replayed noise.  Asserts draws (near-ties only), logits at
    the `probe` steps (none: labels and wave only) and the wave of every row."""
    eng, p = engine_for('ckpt')
    B, _, T = mels.shape
    S = T * HOP
    out = eng.generate(mels, seed=seed)
    eng.check()
    assert eng.last_kernel() == TC
    lab, wave = out['labels'].cpu().numpy(), out['wave'].cpu().numpy()
    del out
    np.testing.assert_allclose(wave, wo.finish_wave(lab, NC, (T - 1) * HOP, HOP), rtol=0, atol=1e-12)
    torch.cuda.empty_cache()
    tf = eng.generate(mels, seed=seed, teacher=lab, return_logits=bool(probe), want_wave=False)
    eng.check()
    assert eng.last_kernel() == TC
    assert np.array_equal(tf['labels'].cpu().numpy(), lab), 'teacher-forced on its own labels, the kernel must redraw them bit for bit'
    lg = None
    if probe:      # only the probed steps of the oracle's rows leave the device (the whole buffer is S x B x 4 KB)
        dev = tf['logits'].device
        lg = tf['logits'].index_select(0, torch.as_tensor(probe, device=dev)).index_select(1, torch.as_tensor(rows, device=dev))
        lg = lg.cpu().numpy()
    del tf
    torch.cuda.empty_cache()
    q = _philox_rows(eng, seed, rows, S)
    mu = np.unique(mels[rows], axis=0, return_inverse=True)
    up, aux = wo.upsample(p, _padded(mu[0]))                      # one conditioning-network run per distinct mel
    inv = mu[1].reshape(-1)
    cond = (np.ascontiguousarray(up[inv]), np.ascontiguousarray(aux[inv]))
    from threadpoolctl import threadpool_limits
    with threadpool_limits(limits=min(16, os.cpu_count() or 1)):
        ref = wo.generate(p, mels[rows], q=q, teacher=lab[rows], keep_logits=probe or (), cond=cond)
        ties = _draws_agree(p, mels[rows], q, lab[rows], cond, lab[rows], ref['labels'], ref['logits'], what=f'B={B} T={T}')
    report = 'labels and wave only'
    if probe:
        want = np.stack([ref['logits'][s] for s in probe])
        tol = _bar(want)
        e = np.abs(lg - want)
        worst = np.unravel_index(int(e.argmax()), e.shape)
        assert e.max() <= tol, f'logit error {e.max():.3e} > {tol:.3e} at (step, row, class) = ({probe[worst[0]]}, {rows[worst[1]]}, {worst[2]})'
        report = f'worst logit error {e.max():.3e} (bar {tol:.3e})'
    print(f'\n[tc] B={B} T={T} rows={rows}: {report}, near-ties (row, step, gap) {ties}')


# ------------------------------------------------------------------------------------------------
# a. whole utterances at the benchmark's shape
# ------------------------------------------------------------------------------------------------
def test_whole_utterance_256_rows_21_frames(torch_cuda):
    """256 rows x 5 775 steps: oracle rows at both edges of every 64-row quarter of both groups; logits at the first steps, around
    the 3-step block that ends frame 0 (272-276), at step 2 000 and at every step of the last three frames."""
    T = 21
    S = T * HOP
    probe = [0, 1, 272, 273, 274, 275, 276, 2000] + list(range(S - 3 * HOP, S))
    _whole_utterance_vs_oracle(torch_cuda, synth.synth_mels(2101, 256, T), 2102, [0, 63, 64, 127, 128, 191, 192, 255], probe)


def test_whole_utterance_256_rows_80_frames(torch_cuda):
    """The benchmark's workload and kernel: 256 rows x 22 000 steps.  Labels and wave only (a logits buffer would be 23 GB)."""
    _whole_utterance_vs_oracle(torch_cuda, synth.synth_mels(8001, 256, 80), 8002, [0, 127, 128, 255], None)


# ------------------------------------------------------------------------------------------------
# b. a real mel through the partial second group
# ------------------------------------------------------------------------------------------------
def test_real_mel_lone_row_of_the_second_group(torch_cuda):
    """The demo recording's features (323 frames, 88 825 steps), converted as wavernn_gen.wav_to_mel does and tiled to 129 rows:
    kernel=auto picks the tensor cores, and row 128 is the only live row of group 1.  Real speech drives the shipped model to
    |logit| ~ 450, far peakier than uniform-random mels, which is what the split-fp16 operands must survive.  The teacher-forced
    logits buffer is 47 GB."""
    mel = np.load(os.path.join(GOLDEN, 'mel_analysis_from_reference.npz'))['speech_mel']
    mel = np.clip((mel + 4.0) / 8.0, 0, 1).T.astype(np.float32)
    mels = np.ascontiguousarray(np.tile(mel[None], (129, 1, 1)))
    S = mels.shape[2] * HOP
    probe = [0, 1, 272, 273, 274, 275, 276, 2000, S // 2] + list(range(S - 3 * HOP, S))
    _whole_utterance_vs_oracle(torch_cuda, mels, 323, [128], probe)


# ------------------------------------------------------------------------------------------------
# c. external noise beyond one group
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('B', [129, 256])
def test_external_noise_all_rows_vs_oracle(torch_cuda, B):
    """EXT_EXPONENTIAL noise q[t][row]: teacher-forced logits of every row for 300 steps, and the draws of that run (fc3 indexes q
    by the global row, so a group-1 row reading another row's noise draws different labels)."""
    eng, p = engine_for('ckpt')
    T, steps = 21, 300
    mels, cond = _distinct_cond(p, B, T, 6000 + B)
    q = synth.synth_exponential_noise(6100 + B, steps, B)
    teacher = np.random.RandomState(6200 + B).randint(0, NC, size=(B, T * HOP)).astype(np.int16)
    out = eng.generate(mels, q=q, teacher=teacher, return_logits=True, max_steps=steps, kernel='tc')
    eng.check()
    assert eng.last_kernel() == TC
    ref = wo.generate(p, mels, q=q, teacher=teacher, keep_logits='all', max_steps=steps, cond=cond)
    want = np.stack([ref['logits'][s] for s in range(steps)])
    e = np.abs(out['logits'].cpu().numpy() - want)
    tol = _bar(want)
    assert e.max() <= tol, f'B={B}: logit error {e.max():.3e} > {tol:.3e} at (step, row, class) = {np.unravel_index(int(e.argmax()), e.shape)}'
    ties = _draws_agree(p, mels, q, teacher, cond, out['labels'].cpu().numpy()[:, :steps], ref['labels'], ref['logits'], what=f'B={B}')
    print(f'\n[tc] external noise B={B}: worst logit error {e.max():.3e} (bar {tol:.3e}), near-ties {ties}')


# ------------------------------------------------------------------------------------------------
# d. step counts that end inside a conditioning block
# ------------------------------------------------------------------------------------------------
STEP_EDGES = [1, 2, 9, 274, 276, 283]      # blocks are <= 8 steps, cut at frame ends: 274 = 34*8 + 2, 283 = 275 + 8


def test_step_count_edges_vs_oracle(torch_cuda):
    """kernel=tc, 129 rows, Philox: for each step count, the teacher-forced logits of every step and the draws (the last one is
    collected on the loop's extra trip) against one oracle run; nothing is written past the last step."""
    eng, p = engine_for('ckpt')
    B, T, seed = 129, 21, 2830
    n = max(STEP_EDGES)
    mels, cond = _distinct_cond(p, B, T, 7000)
    teacher = np.random.RandomState(7001).randint(0, NC, size=(B, T * HOP)).astype(np.int16)
    q = eng.philox_exponential(seed, 0, B, 0, n).cpu().numpy()
    ref = wo.generate(p, mels, q=q, teacher=teacher, keep_logits='all', max_steps=n, cond=cond)
    want = np.stack([ref['logits'][s] for s in range(n)])
    for m in STEP_EDGES:
        out = eng.generate(mels, seed=seed, teacher=teacher, return_logits=True, max_steps=m, kernel='tc')
        eng.check()
        lg, lab = out['logits'].cpu().numpy(), out['labels'].cpu().numpy()
        assert lg.shape == (m, B, NC)
        e = np.abs(lg - want[:m])
        tol = _bar(want[:m])
        assert e.max() <= tol, f'max_steps={m}: logit error {e.max():.3e} > {tol:.3e} at {np.unravel_index(int(e.argmax()), e.shape)}'
        assert not lab[:, m:].any(), f'max_steps={m}: labels written past the last step'
        ties = _draws_agree(p, mels, q, teacher, cond, lab[:, :m], ref['labels'][:, :m], ref['logits'], what=f'max_steps={m}')
        print(f'\n[tc] max_steps={m}: worst logit error {e.max():.3e} (bar {tol:.3e}), near-ties {ties}')


# ------------------------------------------------------------------------------------------------
# e. utterance ids
# ------------------------------------------------------------------------------------------------
def _ids(seed, n):
    """n distinct arbitrary 64-bit utterance ids (as int64: the negative ones have the top bit set)."""
    ids = np.random.RandomState(seed).randint(np.iinfo(np.int64).min, np.iinfo(np.int64).max, size=n, dtype=np.int64)
    assert np.unique(ids).size == n
    return ids


def test_utterance_ids_rows_equal_solo_runs(torch_cuda):
    """kernel=tc, 200 rows keyed by d_utterance_ids: a row is bit-identical to the same row run alone under its id, although it sits
    at another position (and in group 1 for rows >= 128) -- a row's tensor-core arithmetic depends on neither its batch nor its
    position.  Full length, labels and wave."""
    eng, _ = engine_for('ckpt')
    B, T, seed = 200, 21, 2001
    mels = synth.synth_mels(2002, B, T)
    ids = _ids(2003, B)
    full = eng.generate(mels, seed=seed, utterance_ids=ids, kernel='tc')
    eng.check()
    lab, wave = full['labels'].cpu().numpy(), full['wave'].cpu().numpy()
    for b in (0, 1, 127, 128, 199):
        solo = eng.generate(mels[b:b + 1], seed=seed, utterance_ids=ids[b:b + 1], kernel='tc')
        eng.check()
        assert np.array_equal(solo['labels'].cpu().numpy()[0], lab[b]), f'row {b}'
        np.testing.assert_array_equal(solo['wave'].cpu().numpy()[0], wave[b])
    plain = eng.generate(mels[:1], seed=seed, kernel='tc')['labels'].cpu().numpy()[0]     # global index 0 instead of ids[0]
    assert not np.array_equal(plain, lab[0]), 'the utterance id does not reach the noise'


def test_utterance_ids_through_the_256_row_slices(torch_cuda):
    """kernel=auto, 300 rows with ids: one launch of 256 rows on the tensor cores plus a tail, each slice taking its own ids.  The
    result equals the two slices called by hand."""
    eng, _ = engine_for('ckpt')
    B, T, seed = 300, 21, 3001
    mels = synth.synth_mels(3002, B, T)
    ids = _ids(3003, B)
    full = eng.generate(mels, seed=seed, utterance_ids=ids)
    eng.check()
    lab, wave = full['labels'].cpu().numpy(), full['wave'].cpu().numpy()
    for lo, hi in ((0, 256), (256, B)):
        part = eng.generate(mels[lo:hi], seed=seed, utterance_ids=ids[lo:hi])
        eng.check()
        if lo == 0:
            assert eng.last_kernel() == TC
        assert np.array_equal(part['labels'].cpu().numpy(), lab[lo:hi]), f'rows {lo}:{hi}'
        np.testing.assert_array_equal(part['wave'].cpu().numpy(), wave[lo:hi])


# ------------------------------------------------------------------------------------------------
# f. argument errors
# ------------------------------------------------------------------------------------------------
def test_tc_argument_errors(torch_cuda):
    """kernel=tc refuses folding, packed rows and more than 256 rows with B200TTS_EINVAL, and launches nothing."""
    from tacotronv2_wavernn_chinese_b200 import pipeline as pl
    from tacotronv2_wavernn_chinese_b200._lib import B200TTSError
    eng, _ = engine_for('ckpt')
    frames = [21, 25, 22]
    packed = synth.synth_mels(3, len(frames), max(frames))
    calls = {
        'fold': lambda: eng.generate(synth.synth_mels(1, 1, 30), seed=1, kernel='tc', fold=(2750, 550)),
        'pack': lambda: eng.generate(packed, seed=1, kernel='tc', utt_frames=np.array(frames, np.int32),
                                     pack=pl.pack_schedule(frames, 2)),
        '257 rows': lambda: eng.generate(synth.synth_mels(2, 257, 21), seed=1, kernel='tc'),
    }
    for what, call in calls.items():
        n = eng.launch_count
        with pytest.raises(B200TTSError) as e:
            call()
        assert e.value.code == -1 and 'kernel=tc needs' in str(e.value), f'{what}: {e.value}'      # -1 = B200TTS_EINVAL
        assert eng.launch_count == n, f'{what}: a refused call launched work'
