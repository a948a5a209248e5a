"""Parity of the sm_90a WaveRNN path against the oracle and the reference-generated goldens.
Everything here calls the CUDA kernels through the C ABI (engine.WaveRNNEngine -> libb200tts.so)."""
import os

import numpy as np
import pytest

from conftest import GOLDEN, load_ckpt_state_dict
from oracle import wavernn_oracle as wo
from tacotronv2_wavernn_chinese_b200 import synth

pytestmark = pytest.mark.gpu

KERNELS = ['utterance', 'grid']
# plain batches also run on the tensor-core pipeline (kernel='tc' refuses folding and packed rows)
PLAIN_KERNELS = KERNELS + ['tc']


@pytest.fixture(scope='module')
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.fail('GPU tests need a CUDA device (and there is no CPU fallback to hide behind)')
    return torch


_engines = {}


def engine_for(case):
    """case: 'synth<seed>' or 'ckpt'."""
    from tacotronv2_wavernn_chinese_b200.engine import WaveRNNEngine
    if case not in _engines:
        if case == 'ckpt':
            sd = load_ckpt_state_dict()
            if sd is None:
                pytest.skip('shipped checkpoint not available on this box')
        else:
            sd = synth.synth_state_dict(int(case[5:]))
        _engines[case] = (WaveRNNEngine(sd, synth.DEFAULT_DIMS), wo.as_params(sd))
    return _engines[case]


def _padded(mels):
    B, F, T = mels.shape
    mp = np.zeros((B, F, T + 4), dtype=np.float32)
    mp[:, :, 2:-2] = mels
    return mp


def _golden(name):
    return np.load(os.path.join(GOLDEN, name + '.npz'))


def _case_of(name):
    return 'ckpt' if 'ckpt' in name else 'synth11'


# ------------------------------------------------------------------------------------------------
# conditioning network
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ['wavernn_synth_T24', 'wavernn_ckpt_T24'])
def test_upsample_vs_reference_golden(torch_cuda, name):
    g = _golden(name)
    eng, p = engine_for(_case_of(name))
    mels = synth.synth_mels(int(g['mel_seed']), int(g['B']), int(g['T']))
    up, aux = eng.upsample(mels, full_aux=True)
    up, aux = up.cpu().numpy(), aux.cpu().numpy()
    st = int(g['up_stride'])
    # fp32 re-association only (composite polyphase FIR instead of three staged convolutions; BN folded to scale/shift)
    np.testing.assert_allclose(up[:, ::st], g['mels_up_sub'], rtol=0, atol=5e-6)
    np.testing.assert_allclose(aux[:, ::275], g['aux_frames'], rtol=0, atol=2e-4)
    assert np.array_equal(aux, np.repeat(aux[:, ::275], 275, axis=1))


# T on both sides of melresnet_kernel's 8-frame tile, and the long mel_fir_kernel grids of the fold tests' utterances
@pytest.mark.parametrize('B,T', [(1, 21), (3, 37), (2, 5), (1, 1), (4, 7), (2, 8), (3, 9), (4, 16), (1, 17), (2, 255), (4, 256),
                                 (3, 257)])
def test_upsample_vs_oracle_shapes(torch_cuda, B, T):
    eng, p = engine_for('synth5')
    mels = synth.synth_mels(77 + T, B, T)
    up, auxf = eng.upsample(mels, full_aux=False)
    ref_up, ref_aux = wo.upsample(p, _padded(mels))
    np.testing.assert_allclose(up.cpu().numpy(), ref_up, rtol=0, atol=5e-6)
    np.testing.assert_allclose(auxf.cpu().numpy(), ref_aux[:, ::275], rtol=0, atol=2e-4)


# ------------------------------------------------------------------------------------------------
# generation: teacher-forced logits, free-running labels, wave
# ------------------------------------------------------------------------------------------------
def _explain_divergence(p, mels, q, ref_labels, t, b):
    """True when the first mismatch at (b, t) is a near-tie of the sampling race (l - log q top-2 gap tiny)."""
    r = wo.generate(p, mels, q=q[:t + 1], teacher=ref_labels, keep_logits=[t], max_steps=t + 1)
    key = r['logits'][t][b].astype(np.float64) - np.log(q[t, b].astype(np.float64))
    top = np.sort(key)[-2:]
    return (top[1] - top[0]) < 1e-3 * max(1.0, abs(top[1]))


@pytest.mark.parametrize('kernel', PLAIN_KERNELS)
@pytest.mark.parametrize('name', ['wavernn_synth_T24', 'wavernn_ckpt_T24'])
def test_generate_vs_reference_golden(torch_cuda, name, kernel):
    g = _golden(name)
    eng, p = engine_for(_case_of(name))
    B, T = int(g['B']), int(g['T'])
    S = T * 275
    mels = synth.synth_mels(int(g['mel_seed']), B, T)
    q = synth.synth_exponential_noise(int(g['noise_seed']), S, B)
    steps = [int(s) for s in g['logit_steps']]
    # (a) teacher-forced on the reference's label sequence: logits of every recorded step
    out = eng.generate(mels, q=q, teacher=g['labels'], return_logits=True, kernel=kernel)
    lg = out['logits'].cpu().numpy()
    scale = max(1.0, float(np.abs(g['gen_logits']).max()))
    # tolerance: the reference's own nn.GRU-vs-nn.GRUCell floor is 1e-3 abs at |logit|~450 (SURVEY section 4) = 2e-6*scale
    tol = 5e-6 * scale + 1e-4
    err = max(np.abs(lg[s] - g['gen_logits'][i]).max() for i, s in enumerate(steps))
    assert err <= tol, f'teacher-forced logit error {err:.3e} > {tol:.3e}'
    lab_tf = out['labels'].cpu().numpy()
    assert (lab_tf != g['labels']).sum() <= 2, 'sampling from near-identical logits with identical noise must agree'
    # (b) free running, shared noise: identical labels, or a first mismatch that is a genuine near-tie
    out = eng.generate(mels, q=q, kernel=kernel)
    lab = out['labels'].cpu().numpy()
    for b in range(B):
        mism = np.nonzero(lab[b] != g['labels'][b])[0]
        if mism.size:
            t = int(mism[0])
            assert t > S // 4 and _explain_divergence(p, mels, q, g['labels'], t, b), \
                f'utterance {b} diverged from the reference at step {t} without a sampling near-tie'
    if np.array_equal(lab[0], g['labels'][0]):
        np.testing.assert_allclose(out['wave'].cpu().numpy()[0], g['wave0'], rtol=0, atol=1e-12)


@pytest.mark.parametrize('kernel', PLAIN_KERNELS)
def test_generate_config1_shape_vs_reference(torch_cuda, kernel):
    """BASELINE config 1 shape (80 frames, 22 000 steps) on the shipped checkpoint vs the reference's own labels."""
    g = _golden('wavernn_ckpt_T80')
    eng, p = engine_for('ckpt')
    mels = synth.synth_mels(int(g['mel_seed']), 1, 80)
    q = synth.synth_exponential_noise(int(g['noise_seed']), 80 * 275, 1)
    out = eng.generate(mels, q=q, kernel=kernel)
    lab = out['labels'].cpu().numpy()
    mism = np.nonzero(lab[0] != g['labels'][0])[0]
    if mism.size:
        t = int(mism[0])
        assert t > 2000 and _explain_divergence(p, mels, q, g['labels'], t, 0), f'diverged at step {t}'
    else:
        np.testing.assert_allclose(out['wave'].cpu().numpy()[0], g['wave0'], rtol=0, atol=1e-12)
    # teacher-forced logits at the recorded steps over the full length
    out = eng.generate(mels, q=q, teacher=g['labels'], return_logits=True, kernel=kernel)
    lg = out['logits'].cpu().numpy()
    scale = float(np.abs(g['gen_logits']).max())
    for i, s in enumerate(int(s) for s in g['logit_steps']):
        assert np.abs(lg[s] - g['gen_logits'][i]).max() <= 5e-6 * scale + 1e-4


@pytest.mark.parametrize('kernel', PLAIN_KERNELS)
def test_philox_stream_matches_oracle(torch_cuda, kernel):
    """Production RNG: dump the Philox Exp(1) stream the kernel draws and replay it through the oracle."""
    eng, p = engine_for('synth5')
    B, T, seed, off = 2, 21, 0xC0FFEE, 7
    S = T * 275
    mels = synth.synth_mels(31, B, T)
    q = eng.philox_exponential(seed, off, B, 0, S).cpu().numpy()
    assert q.min() > 0 and abs(q.mean() - 1.0) < 0.01 and abs(q.var() - 1.0) < 0.02
    out = eng.generate(mels, seed=seed, utterance_offset=off, kernel=kernel)
    ref = wo.generate(p, mels, q=q)
    lab = out['labels'].cpu().numpy()
    for b in range(B):
        mism = np.nonzero(lab[b] != ref['labels'][b])[0]
        assert mism.size == 0 or (mism[0] > S // 4 and _explain_divergence(p, mels, q, ref['labels'], int(mism[0]), b))
    if np.array_equal(lab, ref['labels']):
        np.testing.assert_allclose(out['wave'].cpu().numpy(), ref['wave'], rtol=0, atol=1e-12)


@pytest.mark.parametrize('kernel', PLAIN_KERNELS)
def test_batch_composition_invariance(torch_cuda, kernel):
    """Philox is keyed by the GLOBAL utterance index, so a row's output cannot depend on what it is batched with
    (this is what makes multi-GPU sharding reproduce the single-GPU result).  Covers the G=1,2,4,8 row-group variants, and for the
    tensor-core kernel a row that sits at another position than alone."""
    eng, _ = engine_for('synth5')
    T, seed = 21, 99
    for B in (3, 9):
        mels = synth.synth_mels(500 + B, B, T)
        full = eng.generate(mels, seed=seed, kernel=kernel, max_steps=1500)['labels'].cpu().numpy()
        for b in (0, B - 1):
            solo = eng.generate(mels[b:b + 1], seed=seed, utterance_offset=b, kernel=kernel, max_steps=1500)
            assert np.array_equal(solo['labels'].cpu().numpy()[0, :1500], full[b, :1500])


@pytest.mark.parametrize('B', [33, 129, 300, 520])
def test_grid_tiles_and_padding(torch_cuda, B):
    """Batches that do not fill a tile / need several tiles per group: the grid kernel must give every row exactly what
    it gives that row alone (Philox keyed by the global row), incl. the last row of a partially filled tile."""
    eng, _ = engine_for('synth5')
    mels = synth.synth_mels(900 + B, B, 21)
    full = eng.generate(mels, seed=17, kernel='grid', max_steps=400)['labels'].cpu().numpy()
    for b in (0, B // 2, B - 1):
        solo = eng.generate(mels[b:b + 1], seed=17, utterance_offset=b, kernel='grid', max_steps=400)['labels'].cpu().numpy()
        assert np.array_equal(solo[0, :400], full[b, :400]), f'row {b} of {B}'


def test_kernels_agree_full_size(torch_cuda):
    """Both kernels, BASELINE-shaped batch (80-frame mels), free running with Philox: identical label streams for
    the first 3000 steps (beyond that fp32 re-association differences may flip a sampling near-tie)."""
    eng, _ = engine_for('synth5')
    mels = synth.synth_mels(4242, 16, 80)
    a = eng.generate(mels, seed=5, kernel='utterance', max_steps=3000)['labels'].cpu().numpy()
    b = eng.generate(mels, seed=5, kernel='grid', max_steps=3000)['labels'].cpu().numpy()
    agree = (a[:, :3000] == b[:, :3000]).all(axis=1)
    assert agree.mean() >= 0.8, f'only {agree.mean():.2f} of utterances agree between kernels'


@pytest.mark.parametrize('kernel', KERNELS)
@pytest.mark.parametrize('name', ['wavernn_synth_batched_T30', 'wavernn_ckpt_batched_T30'])
def test_fold_with_overlap_vs_reference_golden(torch_cuda, name, kernel):
    """--batched mode (fold_with_overlap + xfade_and_unfold, fatchord_version.py:293-405) against the reference's own
    generate(batched=True) under shared noise; the ckpt case uses target/overlap that are NOT hop aligned."""
    g = _golden(name)
    eng, p = engine_for(_case_of(name))
    T, target, overlap = int(g['T']), int(g['target']), int(g['overlap'])
    mel = synth.synth_mels(int(g['mel_seed']), 1, T)
    nf, L = g['labels'].shape
    assert eng.fold_geometry(T, target, overlap) == (nf, L)
    q = synth.synth_exponential_noise(int(g['noise_seed']), L, nf)
    out = eng.generate(mel, q=q, kernel=kernel, fold=(target, overlap))
    lab = out['labels'].cpu().numpy()
    assert lab.shape == (nf, L)
    for b in range(nf):
        mism = np.nonzero(lab[b] != g['labels'][b])[0]
        if mism.size:     # accepted only when the race (l - log q) has a genuine near-tie at that step (teacher-forced oracle)
            t = int(mism[0])
            r = wo.generate_batched(p, mel, target, overlap, q=q, teacher=g['labels'], keep_logits=(t,), max_steps=t + 1)
            key = r['logits'][t][b].astype(np.float64) - np.log(q[t, b].astype(np.float64))
            top = np.sort(key)[-2:]
            assert t > L // 4 and (top[1] - top[0]) < 1e-3 * max(1.0, abs(top[1])), \
                f'fold {b} diverged from the reference at step {t} without a sampling near-tie (gap {top[1] - top[0]:.3e})'
    if np.array_equal(lab, g['labels']):
        np.testing.assert_allclose(out['wave'].cpu().numpy()[0], g['wave'], rtol=0, atol=1e-12)
    # the unfold/cross-fade epilogue on the reference's own labels (independent of sampling)
    ref = wo.xfade_and_unfold(wo.decode_mu_law(wo.label_to_float(lab, 1024).astype(np.float64), 1024), target, overlap)
    wl = (T - 1) * 275
    ref = ref[:wl].copy()
    ref[-20 * 275:] *= np.linspace(1, 0, 20 * 275)
    np.testing.assert_allclose(out['wave'].cpu().numpy()[0], ref, rtol=0, atol=1e-12)


def test_host_entry_point_equals_device_path(torch_cuda):
    eng, _ = engine_for('synth5')
    mels = synth.synth_mels(9, 2, 22)
    dev = eng.generate(mels, seed=42)
    host = eng.generate_host(mels, seed=42)
    assert np.array_equal(host['labels'], dev['labels'].cpu().numpy())
    np.testing.assert_array_equal(host['wave'], dev['wave'].cpu().numpy())
    assert host['wave'].dtype == np.float64 and host['wave'].shape == (2, 21 * 275)
    assert np.all(host['wave'][:, -1] == 0.0) and np.abs(host['wave']).max() <= 1.0


def test_wave_epilogue_matches_oracle(torch_cuda):
    eng, _ = engine_for('synth5')
    mels = synth.synth_mels(10, 3, 25)
    out = eng.generate(mels, seed=1)
    lab = out['labels'].cpu().numpy()
    np.testing.assert_allclose(out['wave'].cpu().numpy(), wo.finish_wave(lab, 1024, 24 * 275, 275), rtol=0, atol=1e-12)
    out2 = eng.generate(mels, seed=1, mu_law=False)
    np.testing.assert_allclose(out2['wave'].cpu().numpy(), wo.finish_wave(lab, 1024, 24 * 275, 275, mu_law=False),
                               rtol=0, atol=1e-12)


def test_error_behaviour(torch_cuda):
    from tacotronv2_wavernn_chinese_b200._lib import B200TTSError
    from tacotronv2_wavernn_chinese_b200.engine import WaveRNNEngine
    eng, _ = engine_for('synth5')
    with pytest.raises(B200TTSError) as e:
        eng.generate(synth.synth_mels(1, 1, 20), seed=1)          # T < 21: the reference's fade-out cannot run either
    assert 'T must be >= 21' in str(e.value)
    with pytest.raises(ValueError):
        eng.generate(np.zeros((1, 79, 30), np.float32))
    sd = synth.synth_state_dict(1)
    bad = dict(sd)
    del bad['fc3.bias']
    with pytest.raises(B200TTSError) as e:
        WaveRNNEngine(bad, synth.DEFAULT_DIMS)
    assert e.value.code == -4 and 'fc3.bias' in str(e.value)
    bad = dict(sd)
    bad['rnn1.weight_hh_l0'] = np.zeros((1536, 511), np.float32)
    with pytest.raises(B200TTSError) as e:
        WaveRNNEngine(bad, synth.DEFAULT_DIMS)
    assert e.value.code == -5


def test_dropin_model_generate(torch_cuda, tmp_path):
    """The reference-facing class: same constructor, state_dict keys, generate() signature and return type."""
    torch = torch_cuda
    from scipy.io import wavfile
    from tacotronv2_wavernn_chinese_b200.wavernn.models.fatchord_version import WaveRNN
    m = WaveRNN(512, 512, 10, 2, (5, 5, 11), 80, 128, 128, 10, 275, 22050, 'RAW')
    sd = synth.synth_state_dict(5)
    m.load_state_dict({k: torch.as_tensor(v) for k, v in sd.items()})
    mel = torch.as_tensor(synth.synth_mels(3, 1, 23))
    path = tmp_path / 'o.wav'
    torch.manual_seed(7)
    w1 = m.generate(mel, str(path), False, 11000, 550, True)
    assert isinstance(w1, np.ndarray) and w1.dtype == np.float64 and w1.shape == (22 * 275,)
    assert m.training          # generate() leaves the module in train() mode like the reference (:262)
    sr, y = wavfile.read(path)
    assert sr == 22050 and np.array_equal(y, w1.astype(np.float32))
    eng, p = engine_for('synth5')
    lab = m.last_labels.cpu().numpy()
    np.testing.assert_allclose(w1, wo.finish_wave(lab, 1024, 22 * 275, 275)[0], rtol=0, atol=1e-12)
    wb = m.generate(torch.as_tensor(synth.synth_mels(4, 1, 40)), None, True, 2750, 550, True)     # --batched
    assert wb.shape == (39 * 275,) and np.isfinite(wb).all() and np.all(wb[:275] == 0.0)            # fade-in starts silent
    up, aux = m.upsample(torch.as_tensor(_padded(mel.numpy())))
    assert tuple(up.shape) == (1, 23 * 275, 80) and tuple(aux.shape) == (1, 23 * 275, 128)


# ------------------------------------------------------------------------------------------------
# every batch mapping the product dispatches, DIRECTLY against the oracle on the shipped checkpoint
# (VERDICT r1 weak #1: the benchmarked instantiations were only compared with themselves at B=1)
# ------------------------------------------------------------------------------------------------
# B -> mapping launch_grid picks: 256/300 two-group wide <4,1,2> (300 = partially filled second tile of each group),
# 128/100 <4,1,1>, 64 <2,1,1>, 32/20/7 <1,1,1>, 3 narrow <0,4,1>; with the push kernel (round 2) B <= 32 runs
# wavernn_push_kernel<G> with G = 4/8/16/32.
MAPPING_BATCHES = [256, 300, 128, 100, 64, 32, 20, 12, 7, 3]


def _distinct_cond(p, B, T, seed, distinct=16):
    """Oracle conditioning for `distinct` different utterances, tiled to B rows (the numpy conditioning network costs
    ~0.1 s per utterance; rows are made different by their teacher labels / noise instead)."""
    n = min(B, distinct)
    mels = synth.synth_mels(seed, n, T)
    up, aux = wo.upsample(p, _padded(mels))
    reps = (B + n - 1) // n
    tile = lambda a: np.ascontiguousarray(np.tile(a, (reps,) + (1,) * (a.ndim - 1))[:B])
    return tile(mels), (tile(up), tile(aux))


# the tensor-core pipeline (wavernn_tc.cuh, kernel='tc'): two full groups, a partial second group (255, 200, and 129 with one live
# row in group 1), one full group, partial single groups (127, 100, 40, 33) and a single row
TC_BATCHES = [256, 255, 200, 129, 128, 127, 100, 40, 33, 1]


@pytest.mark.parametrize('B', TC_BATCHES)
def test_tc_teacher_forced_logits_vs_oracle(torch_cuda, B):
    """The split-fp16 wgmma kernel to the SAME bar as the fp32 CUDA-core mappings: all rows, 300 steps, shipped checkpoint."""
    test_mapping_teacher_forced_logits_vs_oracle(torch_cuda, B, kernel='tc')


@pytest.mark.parametrize('B', TC_BATCHES)
def test_tc_free_running_labels_vs_oracle(torch_cuda, B):
    test_mapping_free_running_labels_vs_oracle(torch_cuda, B, kernel='tc')


@pytest.mark.parametrize('B', MAPPING_BATCHES)
def test_mapping_teacher_forced_logits_vs_oracle(torch_cuda, B, kernel='grid'):
    """Teacher-forced logits of ALL rows for 300 steps, shipped checkpoint, every mapping, against oracle.generate.
    Same bar as the golden tests: 5e-6 * max|logit| + 1e-4."""
    eng, p = engine_for('ckpt')
    T, steps = 21, 300
    S = T * 275
    mels, cond = _distinct_cond(p, B, T, 4000 + B)
    teacher = np.random.RandomState(B).randint(0, 1024, size=(B, S)).astype(np.int16)
    ref = wo.generate(p, mels, teacher=teacher, keep_logits='all', max_steps=steps, cond=cond)
    out = eng.generate(mels, seed=B, teacher=teacher, return_logits=True, max_steps=steps, kernel=kernel)
    lg = out['logits'].cpu().numpy()
    want = np.stack([ref['logits'][s] for s in range(steps)])
    scale = max(1.0, float(np.abs(want).max()))
    err = np.abs(lg - want)
    tol = 5e-6 * scale + 1e-4
    worst = np.unravel_index(int(err.argmax()), err.shape)
    assert err.max() <= tol, f'B={B}: logit error {err.max():.3e} > {tol:.3e} at (step, row, class) = {worst}'


@pytest.mark.parametrize('B', MAPPING_BATCHES)
def test_mapping_free_running_labels_vs_oracle(torch_cuda, B, kernel='grid'):
    """Free-running labels for 2000 steps under the production Philox noise, shipped checkpoint: >= 16 rows spread over
    both utterance groups and every tile position must reproduce the oracle's sequence (the Philox stream of each row is
    dumped and replayed through the oracle); a first mismatch is accepted only as a sampling near-tie."""
    eng, p = engine_for('ckpt')
    T, steps, seed = 21, 2000, 1000 + B
    mels, cond = _distinct_cond(p, B, T, 5000 + B)
    rows = sorted(set([0, B - 1, B // 2, max(0, B // 2 - 1)] + [int(r) for r in np.linspace(0, B - 1, 16)]
                      + [r for r in (31, 32, 127, 128, 129, 255, 256, 299) if r < B]))
    out = eng.generate(mels, seed=seed, max_steps=steps, kernel=kernel)
    lab = out['labels'].cpu().numpy()[:, :steps]
    q = np.concatenate([eng.philox_exponential(seed, r, 1, 0, steps).cpu().numpy() for r in rows], axis=1)
    sub = (cond[0][rows], cond[1][rows])
    ref = wo.generate(p, mels[rows], q=q, max_steps=steps, cond=sub)
    for i, r in enumerate(rows):
        mism = np.nonzero(lab[r] != ref['labels'][i])[0]
        if mism.size:
            t = int(mism[0])
            rr = wo.generate(p, mels[rows], q=q[:t + 1], teacher=ref['labels'], keep_logits=[t], max_steps=t + 1, cond=sub)
            key = rr['logits'][t][i].astype(np.float64) - np.log(q[t, i].astype(np.float64))
            top = np.sort(key)[-2:]
            assert (top[1] - top[0]) < 1e-3 * max(1.0, abs(top[1])), \
                f'B={B} row {r} diverged from the oracle at step {t} without a sampling near-tie (gap {top[1] - top[0]:.3e})'


def test_config2_single_utterance_5s_vs_oracle(torch_cuda):
    """BASELINE config 2: ONE utterance, 402 frames = 5.0 s of audio (110 550 steps), shipped checkpoint, Philox noise.
    The oracle is run ONCE over the full length, teacher-forced on the GPU's labels with the replayed noise: its own
    draw at every step must equal the GPU's label (a handful of sampling near-ties allowed), the logits at fixed
    early / middle / last steps must agree to the usual bar, and the wave must be the oracle's epilogue of those labels."""
    torch = torch_cuda
    eng, p = engine_for('ckpt')
    T, seed = 402, 1235
    S = T * 275
    mels = synth.synth_mels(1235, 1, T)
    out = eng.generate(mels, seed=seed)
    lab = out['labels'].cpu().numpy()
    probe = [0, 1, 999, S // 2, S - 2, S - 1]
    tf = eng.generate(mels, seed=seed, teacher=lab, return_logits=True, want_wave=False)
    lg = tf['logits'][probe].cpu().numpy()
    del tf
    q = torch.cat([eng.philox_exponential(seed, 0, 1, s0, min(20000, S - s0)) for s0 in range(0, S, 20000)]).cpu().numpy()
    from threadpoolctl import threadpool_limits
    with threadpool_limits(limits=min(16, os.cpu_count() or 1)):      # 110 550 sequential matvec steps: ~25 s on the GPU box's host
        ref = wo.generate(p, mels, q=q, teacher=lab, keep_logits=probe)
    mism = int((ref['labels'] != lab).sum())
    assert mism <= 5, f'{mism} of {S} oracle draws differ from the GPU labels'
    scale = max(1.0, max(float(np.abs(ref['logits'][s]).max()) for s in probe))
    for i, s in enumerate(probe):
        assert np.abs(lg[i] - ref['logits'][s]).max() <= 5e-6 * scale + 1e-4, f'step {s}'
    np.testing.assert_allclose(out['wave'].cpu().numpy(), wo.finish_wave(lab, 1024, (T - 1) * 275, 275), rtol=0, atol=1e-12)


def test_push_kernel_result_is_independent_of_batch_size(torch_cuda):
    """The push kernel (B <= 32) sums the 128 block products of every output in one fixed order for all its row-count variants
    (G = 4, 8, 16, 32), so a row's labels are BIT-IDENTICAL whatever batch it is generated in -- the property that makes an
    N-rank sharded run reproduce the single-rank run exactly.  Full length (5775 steps), shipped checkpoint, Philox noise."""
    eng, _ = engine_for('ckpt')
    mels = synth.synth_mels(777, 20, 21)
    full = eng.generate(mels, seed=5, kernel='grid')['labels'].cpu().numpy()              # 20 rows -> G = 32
    for B in (1, 3, 7, 12):                                                                # G = 4, 4, 8, 16
        part = eng.generate(mels[:B], seed=5, kernel='grid')['labels'].cpu().numpy()
        assert np.array_equal(part, full[:B]), f'rows generated {B} at a time differ from the same rows in a batch of 20'
    tail = eng.generate(mels[8:20], seed=5, utterance_offset=8, kernel='grid')['labels'].cpu().numpy()   # a "second rank's" shard
    assert np.array_equal(tail, full[8:20])


def test_large_request_is_cut_into_row_ranges(torch_cuda):
    """A batch whose sample-rate conditioning buffer would exceed the memory budget (wide mapping: S x 80 x rows floats; 22.5 GB
    at 256 rows x 1000 frames) is run as several launches over row ranges.  The noise is keyed by the global row, so the labels
    are those of the same row ranges generated by hand.  Budget forced down through B200TTS_MAX_COND_BYTES (read per call)."""
    eng, _ = engine_for('synth5')
    mels = synth.synth_mels(321, 100, 21)
    os.environ['B200TTS_MAX_COND_BYTES'] = '100e6'          # 1.85 MB per row -> 54 rows fit -> ranges of 32 rows
    try:
        cut = eng.generate(mels, seed=4)
    finally:
        del os.environ['B200TTS_MAX_COND_BYTES']
    lab, wave = cut['labels'].cpu().numpy(), cut['wave'].cpu().numpy()
    for lo in range(0, 100, 32):
        hi = min(lo + 32, 100)
        part = eng.generate(mels[lo:hi], seed=4, utterance_offset=lo)
        assert np.array_equal(part['labels'].cpu().numpy(), lab[lo:hi]), f'rows {lo}:{hi}'
        np.testing.assert_array_equal(part['wave'].cpu().numpy(), wave[lo:hi])


def test_auto_dispatch_and_slicing_through_the_tensor_core_kernel(torch_cuda):
    """kernel='auto': 129-256 rows run wavernn_tc_kernel; more than 256 rows are cut into launches of 256 rows (tensor-core pipeline)
    plus a tail on the CUDA-core kernels.  The noise is keyed by the global row, so every range equals the same rows generated by
    hand; a row's arithmetic in the tensor-core kernel does not depend on its batch (bit-equal against a 200-row launch)."""
    eng, _ = engine_for('ckpt')
    mels = synth.synth_mels(77, 300, 21)
    steps = 500
    a = eng.generate(mels[:256], seed=9, max_steps=steps, want_wave=False)
    assert eng.last_kernel() == 'wavernn_tc_kernel'
    la = a['labels'].cpu().numpy()[:, :steps]
    b = eng.generate(mels[:200], seed=9, max_steps=steps, want_wave=False, kernel='tc')['labels'].cpu().numpy()[:, :steps]
    assert np.array_equal(la[:200], b)
    small = eng.generate(mels[:100], seed=9, max_steps=steps, want_wave=False)
    assert eng.last_kernel() == 'wavernn_grid_kernel'
    full = eng.generate(mels, seed=9, max_steps=steps, want_wave=False)['labels'].cpu().numpy()[:, :steps]
    assert np.array_equal(full[:256], la)
    tail = eng.generate(mels[256:], seed=9, utterance_offset=256, max_steps=steps, want_wave=False)['labels'].cpu().numpy()[:, :steps]
    assert np.array_equal(full[256:], tail)
    # the CUDA-core and the tensor-core kernel draw the same labels up to sampling near-ties (which then diverge the row)
    same = (small['labels'].cpu().numpy()[:, :50] == la[:100, :50]).all(axis=1).mean()
    assert same >= 0.9, f'only {same:.2f} of the rows agree between the wide and the tensor-core kernel over 50 steps'


def test_packed_rows_equal_standalone_utterances(torch_cuda):
    """Packed generation of a ragged set (gen_opts.d_pack_*): 2 / 8 kernel rows each run a queue of utterances back to back and
    restart from the zero state at every utterance start.  Every utterance must come out BIT FOR BIT as from a stand-alone run
    (same noise key, same arithmetic) -- labels over its full length and the truncated / faded wave.  Shipped checkpoint."""
    from tacotronv2_wavernn_chinese_b200 import pipeline as pl
    eng, _ = engine_for('ckpt')
    frames = [60, 25, 40, 21, 33, 52, 30, 47, 22, 36, 28]
    T = max(frames)
    ids = [100 + 3 * i for i in range(len(frames))]                     # arbitrary global utterance indices
    full = synth.synth_mels(808, len(frames), T)
    batch = np.zeros_like(full)
    for i, f in enumerate(frames):
        batch[i, :, :f] = full[i, :, :f]                                # zero frames past each utterance's end
    solo = [eng.generate(batch[i:i + 1, :, :f], seed=21, utterance_ids=[ids[i]]) for i, f in enumerate(frames)]
    for rows in (2, 8):
        sch = pl.pack_schedule(frames, rows)
        assert sch['steps'] < sum(frames) * 275                         # really several utterances per row
        out = eng.generate(batch, seed=21, utterance_ids=ids, utt_frames=np.array(frames, np.int32), pack=sch)
        eng.check()
        lab, wave = out['labels'].cpu().numpy(), out['wave'].cpu().numpy()
        for i, f in enumerate(frames):
            assert np.array_equal(lab[i, :f * 275], solo[i]['labels'].cpu().numpy()[0]), f'rows={rows}: utterance {i} ({f} frames)'
            np.testing.assert_array_equal(wave[i, :(f - 1) * 275], solo[i]['wave'].cpu().numpy()[0])
            assert np.all(wave[i, (f - 1) * 275:] == 0.0)
