"""Fold-with-overlap generation (the reference's generate(batched=True), fatchord_version.py:293-405) on every step kernel that
serves it, against the oracle.

One utterance is cut into n_folds rows of L = target + 2 * overlap samples, generated as a batch and cross-faded back together.
Each step kernel gets its fold rows through its own code: the utterance kernel through fold_cond_kernel, the push kernel (up to
32 folds) through its conditioning table read at sample u * stride + t, the wide grid kernel through fold_cond_T_kernel.  Every
path ends in xfade_unfold_kernel.  The geometries below put the fold count at every dispatch boundary and the last fold at every
edge of fold_with_overlap's padding, with small folds so that every step of every fold is compared.  Synthetic weights, plus the
shipped checkpoint where it is present."""
import ctypes

import numpy as np
import pytest

from oracle import wavernn_oracle as wo
from tacotronv2_wavernn_chinese_b200 import synth
from test_wavernn_gpu import _padded, engine_for, torch_cuda  # noqa: F401  (torch_cuda is a fixture)

pytestmark = pytest.mark.gpu

HOP, NC = 275, 1024
UTT, GRID, PUSH = 'wavernn_utt_kernel', 'wavernn_grid_kernel', 'wavernn_push_kernel'

# (T frames, target, overlap), teacher-forced over every step of every fold.  "remaining" is fold_with_overlap's
# S - (n_folds' * stride + overlap) before it adds the padded last fold: 0 means the last fold ends exactly at S, 1 that it
# holds overlap + 1 real samples, stride - 1 that it is one padded sample short of L.
FOLD_CASES = [
    (21, 5775, 550),    # 1 fold, longer than the utterance; stride 23 hops       push G = 8
    (21, 2883, 3),      # 2 folds, remaining 0, odd overlap (flen 2)               push G = 8
    (21, 713, 8),       # 8 folds, remaining stride - 1                           push G = 8
    (21, 635, 6),       # 9 folds, remaining 0                                     push G = 16
    (21, 370, 14),      # 16 folds, remaining 1                                    push G = 16
    (21, 326, 13),      # 17 folds, remaining stride - 1, odd overlap              push G = 32
    (32, 250, 25),      # 32 folds, stride one hop                                 push G = 32
    (21, 141, 33),      # 33 folds, remaining 0, odd overlap                       wide grid W2
    (21, 50, 41),       # 64 folds, remaining 1, odd overlap                       W2
    (21, 32, 56),       # 65 folds, remaining stride - 1, target < overlap         W4
    (21, 30, 15),       # 128 folds, remaining 0                                   W4
    (23, 45, 4),        # 129 folds, remaining 0                                   W4x2, utterance G = 1
    (27, 27, 2),        # 256 folds, overlap 2 (one-point linspace), rem. stride-1  W4x2, utterance G = 2
    (30, 5, 27),        # 257 folds (a second 256-row tile), target < overlap      W4x2, utterance G = 2
    (24, 1, 21),        # 300 folds, remaining 1, target < overlap                 W4x2, utterance G = 4
    (21, 1, 2),         # 1 925 folds (L = 5, 2 048 padded rows), remaining 1     W4x2, utterance G = 8
]
# the shipped checkpoint on one geometry of each step kernel's fold path
CKPT_CASES = [(21, 713, 8), (21, 141, 33), (30, 5, 27), (21, 1, 2)]
# also checked with mu_law=False
LINEAR_CASES = [(21, 2883, 3), (27, 27, 2), (21, 1, 2)]


def geometry(T, target, overlap):
    """(n_folds, L, stride, remaining) of fold_with_overlap (fatchord_version.py:319-330) for a T-frame utterance."""
    S, stride = T * HOP, target + overlap
    n = (S - overlap) // stride
    remaining = S - (n * stride + overlap)
    return n + (remaining != 0), target + 2 * overlap, stride, remaining


def grid_kernel_for(n_folds):
    """The step kernel kernel='grid' (and 'auto') runs for n_folds folds."""
    return PUSH if n_folds <= 32 else GRID


def reference_wave(labels, T, target, overlap, mu_law=True):
    """xfade_and_unfold of the decoded labels, truncated to (T - 1) hops with the 20-hop fade-out (fatchord_version.py:243-258)."""
    y = wo.label_to_float(np.asarray(labels), NC).astype(np.float64)
    if mu_law:
        y = wo.decode_mu_law(y, NC)
    w = wo.xfade_and_unfold(y, target, overlap)[:(T - 1) * HOP].copy()
    w[-20 * HOP:] *= np.linspace(1, 0, 20 * HOP)
    return w


_ref = {}


def _teacher_forced_reference(model, T, target, overlap):
    """(mel, teacher labels, oracle logits [L][n_folds][NC]) of one case; only the latest case is kept."""
    key = (model, T, target, overlap)
    if key not in _ref:
        _ref.clear()
        _, p = engine_for(model)
        nf, L, _, _ = geometry(T, target, overlap)
        mel = synth.synth_mels(T * 1000 + overlap, 1, T)
        teacher = np.random.RandomState(target + overlap).randint(0, NC, size=(nf, L)).astype(np.int16)
        r = wo.generate_batched(p, mel, target, overlap, teacher=teacher, keep_logits=range(L))
        _ref[key] = (mel, teacher, np.stack([r['logits'][s] for s in range(L)]))
    return _ref[key]


SWEEP = ([('synth5', g, k) for g in FOLD_CASES for k in ('utterance', 'grid')]
         + [('ckpt', g, k) for g in CKPT_CASES for k in ('utterance', 'grid')])


@pytest.mark.parametrize('model,geom,kernel', SWEEP, ids=[f'{m}-T{g[0]}-t{g[1]}-o{g[2]}-{k}' for m, g, k in SWEEP])
def test_fold_teacher_forced_logits_and_wave(torch_cuda, model, geom, kernel):
    """Logits of every (step, fold, class) to the bar of the other parity tests, 5e-6 * max|logit| + 1e-4, and the wave as the
    oracle's cross-fade of the GPU's own labels (so it does not depend on sampling)."""
    T, target, overlap = geom
    eng, _ = engine_for(model)
    nf, L, _, _ = geometry(T, target, overlap)
    assert eng.fold_geometry(T, target, overlap) == (nf, L)
    mel, teacher, want = _teacher_forced_reference(model, T, target, overlap)
    assert want.shape == (L, nf, NC)
    out = eng.generate(mel, seed=nf, teacher=teacher, return_logits=True, kernel=kernel, fold=(target, overlap))
    eng.check()
    assert eng.last_kernel() == (UTT if kernel == 'utterance' else grid_kernel_for(nf))
    err = np.abs(out['logits'].cpu().numpy() - want)
    tol = 5e-6 * max(1.0, float(np.abs(want).max())) + 1e-4
    worst = np.unravel_index(int(err.argmax()), err.shape)
    lab = out['labels'].cpu().numpy()
    assert lab.shape == (nf, L)
    wave_err = np.abs(out['wave'].cpu().numpy()[0] - reference_wave(lab, T, target, overlap)).max()
    print(f'\n{nf} folds of {L} on {eng.last_kernel()}: logit error {err.max():.3e} (bar {tol:.3e}), wave error {wave_err:.1e}')
    assert err.max() <= tol, f'logit error {err.max():.3e} > {tol:.3e} at (step, fold, class) = {worst}'
    assert wave_err <= 1e-12
    if geom in LINEAR_CASES:
        out = eng.generate(mel, seed=nf, teacher=teacher, kernel=kernel, fold=(target, overlap), mu_law=False)
        eng.check()
        lab = out['labels'].cpu().numpy()
        np.testing.assert_allclose(out['wave'].cpu().numpy()[0], reference_wave(lab, T, target, overlap, mu_law=False),
                                   rtol=0, atol=1e-12)


@pytest.mark.parametrize('model', ['synth5', 'ckpt'])
@pytest.mark.parametrize('T,kernel', [(402, PUSH), (1347, GRID)])
def test_fold_production_geometry_free_running(torch_cuda, model, T, kernel):
    """wavernn_gen.py --batched defaults (target 11 000, overlap 550): 402 frames (5 s, 10 folds, push G = 16) and 1 347 frames
    (33 folds, the wide grid).  Philox noise, replayed per fold; folds 0, 1, the middle, the second-to-last and the last are
    compared over all L = 12 100 steps, and a first mismatch is accepted only as a sampling near-tie."""
    eng, p = engine_for(model)
    target, overlap, seed = 11000, 550, 7000 + T
    nf, L, _, _ = geometry(T, target, overlap)
    mel = synth.synth_mels(T, 1, T)
    out = eng.generate(mel, seed=seed, fold=(target, overlap))
    eng.check()
    assert eng.last_kernel() == kernel
    lab = out['labels'].cpu().numpy()
    assert lab.shape == (nf, L)
    rows = sorted({0, 1, nf // 2, nf - 2, nf - 1})
    q = np.concatenate([eng.philox_exponential(seed, u, 1, 0, L).cpu().numpy() for u in rows], axis=1)
    up, aux = wo.upsample(p, _padded(mel))
    sub = tuple(np.ascontiguousarray(wo.fold_with_overlap(a, target, overlap)[rows]) for a in (up, aux))
    del up, aux
    stub = np.zeros((len(rows), 80, 21), np.float32)      # generate() takes the row count and wave length from the mels
    ref = wo.generate(p, stub, q=q, cond=sub)
    for i, u in enumerate(rows):
        mism = np.nonzero(lab[u] != ref['labels'][i])[0]
        if mism.size:
            t = int(mism[0])
            rr = wo.generate(p, stub, q=q[:t + 1], teacher=ref['labels'], keep_logits=[t], max_steps=t + 1, cond=sub)
            key = rr['logits'][t][i].astype(np.float64) - np.log(q[t, i].astype(np.float64))
            top = np.sort(key)[-2:]
            print(f'\n{model}, fold {u} of {nf}: first mismatch at step {t}, race gap {top[1] - top[0]:.3e}')
            assert (top[1] - top[0]) < 1e-3 * max(1.0, abs(top[1])), \
                f'fold {u} diverged from the oracle at step {t} without a sampling near-tie (gap {top[1] - top[0]:.3e})'
    np.testing.assert_allclose(out['wave'].cpu().numpy()[0], reference_wave(lab, T, target, overlap), rtol=0, atol=1e-12)


@pytest.mark.parametrize('geom', [(23, 45, 4), (30, 5, 27), (21, 1, 2)])
def test_auto_keeps_folds_off_the_tensor_cores(torch_cuda, geom):
    """129 or more folds are rows the tensor-core kernel could take, but it refuses folding: kernel='auto' runs the wide grid, with
    labels and wave bit-identical to kernel='grid'."""
    T, target, overlap = geom
    eng, _ = engine_for('synth5')
    mel = synth.synth_mels(5, 1, T)
    a = eng.generate(mel, seed=3, fold=(target, overlap))
    assert eng.last_kernel() == GRID
    b = eng.generate(mel, seed=3, fold=(target, overlap), kernel='grid')
    assert eng.last_kernel() == GRID
    assert np.array_equal(a['labels'].cpu().numpy(), b['labels'].cpu().numpy())
    np.testing.assert_array_equal(a['wave'].cpu().numpy(), b['wave'].cpu().numpy())


def _library_generate(eng, B, T, target, overlap, utterance_ids=False):
    """b200tts_wavernn_generate called directly, past the engine's own argument checks; labels and wave stay in the context."""
    import torch
    from tacotronv2_wavernn_chinese_b200 import _lib
    mel = eng._mel(synth.synth_mels(2, B, T))
    ids = torch.arange(B, dtype=torch.int64, device=mel.device)
    rng = _lib.Rng()
    rng.mode = _lib.RNG_PHILOX
    if utterance_ids:
        rng.d_utterance_ids = ids.data_ptr()
    opts = _lib.GenOpts()
    opts.kernel, opts.mu_law = _lib.KERNELS['auto'], 1
    opts.fold_target, opts.fold_overlap = target, overlap
    _lib.check(eng.lib.b200tts_wavernn_generate(eng._h, ctypes.c_void_p(mel.data_ptr()), B, T, ctypes.byref(rng),
                                                ctypes.byref(opts), None, None, eng._stream()))
    torch.cuda.synchronize()


def test_fold_refusals_launch_nothing(torch_cuda):
    """What fold-with-overlap cannot serve is refused before anything is launched."""
    from tacotronv2_wavernn_chinese_b200._lib import B200TTSError
    eng, _ = engine_for('synth5')
    mel = synth.synth_mels(1, 1, 21)

    def refused(call, text, err=B200TTSError):
        n = eng.launch_count
        with pytest.raises(err) as e:
            call()
        assert text in str(e.value), str(e.value)
        if err is B200TTSError:
            assert e.value.code == -1, str(e.value)                                   # B200TTS_EINVAL
        assert eng.launch_count == n, f'a refused call launched work: {e.value}'

    refused(lambda: eng.generate(mel, seed=1, fold=(100, 20), kernel='tc'), 'kernel=tc needs')
    refused(lambda: eng.generate(mel, seed=1, fold=(100, 20), max_steps=10), 'max_steps is not supported together with folding')
    refused(lambda: eng.generate(synth.synth_mels(1, 2, 21), seed=1, fold=(100, 20)), 'exactly one utterance', ValueError)
    refused(lambda: eng.generate(mel, seed=1, fold=(100, 20), utterance_ids=[0]), 'cannot be combined with fold', ValueError)
    refused(lambda: eng.generate(mel, seed=1, fold=(100, 1)), 'fold target/overlap out of range')
    refused(lambda: eng.generate(mel, seed=1, fold=(100, 5775)), 'shorter than the fold overlap')
    # 715 frames at target 1, overlap 2: 65 541 folds, past the 65 535 a launch grid can index
    assert geometry(715, 1, 2)[0] == 65541
    refused(lambda: eng.generate(synth.synth_mels(1, 1, 715), seed=1, fold=(1, 2)), 'fold count out of range')
    # the same checks in the library, past the engine's
    refused(lambda: _library_generate(eng, 2, 21, 100, 20), 'exactly one utterance')
    refused(lambda: _library_generate(eng, 1, 21, 100, 20, utterance_ids=True), 'd_utterance_ids cannot be combined')
    refused(lambda: _library_generate(eng, 1, 21, 100, 1), 'fold target/overlap out of range')
    refused(lambda: _library_generate(eng, 1, 21, -1, 20), 'fold target/overlap out of range')          # 0 turns folding off
    refused(lambda: _library_generate(eng, 1, 21, 100, 5775), 'shorter than the fold overlap')
    refused(lambda: _library_generate(eng, 1, 21, 2 ** 31 - 1000, 550), 'longer than 2^31 - 1 samples')
    # the context still generates afterwards
    n = eng.launch_count
    eng.generate(mel, seed=1, fold=(100, 20))
    eng.check()
    assert eng.launch_count > n
