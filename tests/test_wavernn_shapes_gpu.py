"""WaveRNN generation at every model shape the library accepts, on each step kernel that runs it, against the oracle.

`SHAPES` holds models that move several hparams at once away from the shipped one (R = F = 512, 10 bits, feat 80, aux 32,
compute 128, 10 blocks, pad 2, factors (5, 5, 11)).  For each, `kernels_for` restates which step kernels csrc/ gives it
(pack_grid_model, pack_push_model, pack_tc_images, choose_kernel), and every one of them runs the model at row counts that reach
its tiles: push 1 and 32, grid 4 (or 33) and 129, tensor cores 129 and 256, utterance 1, 133 and 529.

Checks, all against oracle/wavernn_oracle.py (RAW) or oracle/wavernn_mol_oracle.py (MOL), which read every dimension from the
weights' shapes: the conditioning network at T = 1, 8, 9 and 21; teacher-forced logits of every row over two frame boundaries
within the bar 5e-6 * max|logit| + 1e-4; Philox free runs replayed through the oracle (a divergence only at a sampling near-tie);
the wave epilogue with mu-law on and off; fold-with-overlap at hop 200; sessions at hop 200 and hop 7 bit-equal to the one-shot
run.  Rows repeat a pattern of `NPAT` distinct (mel, teacher) inputs, so the oracle runs NPAT rows per shape and every GPU row is
compared with the oracle row of its pattern."""
import numpy as np
import pytest

from oracle import wavernn_mol_oracle as mo
from oracle import wavernn_oracle as wo
from tacotronv2_wavernn_chinese_b200 import synth
from test_wavernn_gpu import torch_cuda  # noqa: F401  (torch_cuda is a fixture)

pytestmark = pytest.mark.gpu

UTT, GRID, PUSH, TC = 'wavernn_utt_kernel', 'wavernn_grid_kernel', 'wavernn_push_kernel', 'wavernn_tc_kernel'
NPAT = 13          # distinct inputs per shape; prime, so no tile of 4 .. 256 rows holds two rows of one pattern at a fixed offset
T_TF = 3           # frames of the teacher-forced and free runs (more for hop < 22, so two frame boundaries are crossed)

# name -> hparams over the shipped ones (hop_length follows the factors).  Comments: the edge each shape reaches.
SHAPES = {
    # hop % 8 == 0 (no remainder conditioning block); feat 4, aux 4, compute 32, 1 block, pad 1
    'hop256_feat4_aux4': dict(upsample_factors=(4, 4, 16), feat_dims=4, res_out_dims=16, compute_dims=32, res_blocks=1, pad=1),
    # 4 stages; feat 128, aux 128 (R + aux = 640 exactly), compute 100, no residual block, pad 4
    'hop256_4stages_aux128': dict(upsample_factors=(4, 4, 4, 4), feat_dims=128, res_out_dims=512, compute_dims=100,
                                  res_blocks=0, pad=4),
    # hop 200: folds and sessions; compute 1024 (melresnet_kernel with 1024 threads)
    'hop200_compute1024': dict(upsample_factors=(5, 5, 8), compute_dims=1024, res_blocks=2),
    # hop 8: exactly one conditioning block per frame; the shipped 10 residual blocks
    'hop8': dict(upsample_factors=(2, 2, 2)),
    # hop < 8, one stage, 3 taps; pad 3, aux 16; sessions
    'hop7_pad3': dict(upsample_factors=(7,), pad=3, res_out_dims=64, res_blocks=1),
    # hop 1
    'hop1_pad1': dict(upsample_factors=(1,), pad=1, res_blocks=1),
    # 7 taps: the kMaxTaps limit
    'taps7': dict(upsample_factors=(1, 1, 2), res_blocks=1),
    # hop x taps = 8190 floats: the largest FIR that fits the tensor-core kernel's slot
    'fir8190': dict(upsample_factors=(2730,), feat_dims=4, compute_dims=32, res_blocks=0),
    # 8193 floats: kernel='tc' refused, auto gives 129 rows to the grid kernel
    'fir8193': dict(upsample_factors=(2731,), feat_dims=8, compute_dims=32, res_blocks=0),
    # hop 1800 x 5 taps: push and grid, not the tensor cores
    'fir_8x15x15': dict(upsample_factors=(8, 15, 15), feat_dims=8, compute_dims=32, res_blocks=1),
    # grid kernel on 32 CTAs; pad 1 at hop 275, where the composite reach (341) exceeds the trimmed indent (275)
    'R128_bits8_pad1': dict(rnn_dims=128, fc_dims=128, bits=8, feat_dims=20, res_out_dims=64, res_blocks=1, pad=1),
    # grid kernel on 64 CTAs
    'R256_bits9': dict(rnn_dims=256, fc_dims=256, bits=9, upsample_factors=(4, 4, 16), res_blocks=1),
    # utterance kernel only: R = F = 1024 with 4096 classes, 4 rows per CTA at 529 rows (8 do not fit its shared memory)
    'R1024_bits12': dict(rnn_dims=1024, fc_dims=1024, bits=12, upsample_factors=(7,), compute_dims=64, res_blocks=1),
    # utterance kernel only: F != R, feat % 4 != 0, 2048 classes
    'F256_feat13_bits11': dict(fc_dims=256, feat_dims=13, bits=11, upsample_factors=(2, 2, 2), res_blocks=1),
    # utterance kernel only: 4 classes (fewer than a warp's lanes), aux 132 (R + aux > 640)
    'bits2_aux132': dict(bits=2, res_out_dims=528, upsample_factors=(3,), res_blocks=1),
    # utterance kernel only: 32768 classes
    'bits15': dict(bits=15, upsample_factors=(2,), compute_dims=32, res_blocks=1),
    # MOL: grid on 96 CTAs; grid on 64 CTAs; push at hop 200
    'mol_R384': dict(mode='MOL', rnn_dims=384, fc_dims=384, res_blocks=1),
    'mol_R256': dict(mode='MOL', rnn_dims=256, fc_dims=256, upsample_factors=(4, 4, 16), res_blocks=1),
    'mol_hop200': dict(mode='MOL', upsample_factors=(5, 5, 8), res_blocks=1),
}


def dims_of(name):
    d = dict(synth.DEFAULT_DIMS, **SHAPES[name])
    d['hop_length'] = int(np.prod(d['upsample_factors']))
    return d


def fir_taps(factors):
    """NT of composite_fir (csrc/wavernn.cu): frames on each side within the composite reach, both sides and the frame."""
    hop, rate, reach = int(np.prod(factors)), int(np.prod(factors)), 0
    for s in factors:
        rate //= s
        reach += s * rate
    return 2 * (-(-reach // hop)) + 1


def kernels_for(d):
    """The fast step kernels csrc/ builds for model `d` on an H100 (132 SMs): a subset of {'grid', 'push', 'tc'}."""
    R, F, hop = d['rnn_dims'], d['fc_dims'], d['hop_length']
    mol = d.get('mode') == 'MOL'
    aux, feat = d['res_out_dims'] // 4, d['feat_dims']
    nc = 2 * R if mol else 1 << d['bits']                 # MOL: fc3's 30 rows spread to 2R classes, 8 per CTA
    out = set()
    if R == F and nc == 2 * R and R <= 512 and feat % 4 == 0 and R + aux <= 640 and feat + aux <= 640:
        out.add('grid')
        # every FIR table of SHAPES fits the push kernel's shared memory (at most 1800 x 5 = 9000 floats)
        if R == 512:
            out.add('push')
            if not mol and nc == 1024 and hop * fir_taps(d['upsample_factors']) <= 8192:
                out.add('tc')
    return out


def runs_for(d):
    """(kernel argument, rows, step kernel that must run) of every run of model `d`."""
    k = kernels_for(d)
    out = [('utterance', r, UTT) for r in (1, 133, 529)]
    if 'push' in k:
        out += [('grid', 1, PUSH), ('grid', 32, PUSH), ('grid', 33, GRID), ('grid', 129, GRID)]
    elif 'grid' in k:
        out += [('grid', 4, GRID), ('grid', 33, GRID), ('grid', 129, GRID)]
    if 'tc' in k:
        out += [('tc', 129, TC), ('tc', 256, TC)]
    return out


def test_shape_table_reaches_every_edge():
    """The table holds the edges it claims, and each fast kernel family runs the ones that concern it."""
    D = {n: dims_of(n) for n in SHAPES}
    fast = {n: kernels_for(d) for n, d in D.items()}
    hops = {n: d['hop_length'] for n, d in D.items() if 'tc' in fast[n]}
    assert {256, 200, 8, 7, 1, 2, 2730} <= set(hops.values())
    assert {fir_taps(D[n]['upsample_factors']) for n in hops} >= {3, 5, 7}
    assert 2730 * fir_taps((2730,)) == 8190 and 2731 * fir_taps((2731,)) == 8193 and 'tc' not in fast['fir8193']
    assert fast['fir_8x15x15'] == {'grid', 'push'}
    assert {D[n]['rnn_dims'] for n in D if 'grid' in fast[n]} == {128, 256, 384, 512}
    assert {D[n]['feat_dims'] for n in D if fast[n]} >= {4, 128} and not fast['F256_feat13_bits11']
    assert {D[n]['res_out_dims'] for n in D if fast[n]} >= {16, 512} and not fast['bits2_aux132']
    assert {D[n]['compute_dims'] for n in D if fast[n]} >= {32, 100, 1024}
    assert {D[n]['res_blocks'] for n in D if fast[n]} >= {0, 1, 10} and {D[n]['pad'] for n in D if fast[n]} >= {1, 2, 4}
    assert {D[n]['bits'] for n in D if D[n].get('mode') != 'MOL'} >= {2, 8, 9, 10, 11, 12, 15}


# ------------------------------------------------------------------------------------------------
# engines, inputs and the oracle, once per shape
# ------------------------------------------------------------------------------------------------
_cache = {}


@pytest.fixture(scope='module')
def shapes(torch_cuda):
    yield _cache
    for v in _cache.values():
        if 'eng' in v:
            v['eng'].close()
    _cache.clear()


def model(cache, name):
    from tacotronv2_wavernn_chinese_b200.engine import WaveRNNEngine
    if name not in cache:
        d = dims_of(name)
        sd = synth.synth_state_dict(7, d, mode=d.get('mode', 'RAW'))
        cache[name] = dict(d=d, sd=sd, p=wo.as_params(sd), eng=WaveRNNEngine(sd, d))
    return cache[name]


def padded(mels, pad):
    B, F, T = mels.shape
    mp = np.zeros((B, F, T + 2 * pad), dtype=np.float32)
    mp[:, :, pad:pad + T] = mels
    return mp


def steps_of(d):
    """Steps of the teacher-forced and free runs: past the second frame boundary."""
    return max(2 * d['hop_length'] + 3, 40)


def frames_of(d):
    return max(T_TF, steps_of(d) // d['hop_length'] + 1)


def pattern(m):
    """The NPAT distinct rows of a shape: mels [NPAT, feat, T], oracle conditioning, teacher labels or samples [NPAT, S],
    and the oracle's teacher-forced logits [steps, NPAT, NC]."""
    if 'pat' not in m:
        d, p = m['d'], m['p']
        T, steps = frames_of(d), steps_of(d)
        S = T * d['hop_length']
        mels = synth.synth_mels(300 + d['hop_length'], NPAT, T, d['feat_dims'])
        rs = np.random.RandomState(d['hop_length'] + d['bits'])
        if d.get('mode') == 'MOL':
            teacher = np.clip(rs.normal(0, 0.3, (NPAT, S)), -1, 1).astype(np.float32)
            u = synth.synth_mol_uniform(5, steps, NPAT)
            ref = mo.generate(m['sd'], mels, u, teacher=teacher, keep_logits='all', max_steps=steps)
            cond = None
        else:
            teacher = rs.randint(0, 1 << d['bits'], size=(NPAT, S)).astype(np.int16)
            cond = wo.upsample(p, padded(mels, d['pad']))
            ref = wo.generate(p, mels, teacher=teacher, keep_logits='all', max_steps=steps, cond=cond)
        m['pat'] = dict(T=T, steps=steps, mels=mels, cond=cond, teacher=teacher,
                        logits=np.stack([ref['logits'][s] for s in range(steps)]))
    return m['pat']


def tile(a, rows, axis=0):
    idx = np.arange(rows) % NPAT
    return np.ascontiguousarray(np.take(a, idx, axis=axis))


def logit_bar(ref):
    return 5e-6 * max(1.0, float(np.abs(ref).max())) + 1e-4


def logit_error(lg, ref):
    """max |lg - ref[row % NPAT]| over steps, rows and classes, computed on the device (lg [steps, B, NC] cuda)."""
    import torch
    r = torch.as_tensor(ref, device=lg.device)
    err = 0.0
    for k in range(min(NPAT, lg.shape[1])):
        err = max(err, float((lg[:, k::NPAT] - r[:, k:k + 1]).abs().max()))
    return err


RUNS = [(n, k, r, sk) for n in SHAPES for k, r, sk in runs_for(dims_of(n))]


# ------------------------------------------------------------------------------------------------
# conditioning network
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', list(SHAPES))
def test_upsample_vs_oracle(shapes, name):
    """eng.upsample against the oracle's staged network at T = 1, 8, 9 and 21 (1 and 2 for the 2730-sample hops, whose staged
    numpy convolution alone takes seconds per frame)."""
    m = model(shapes, name)
    d, p, eng = m['d'], m['p'], m['eng']
    Ts = (1, 2) if d['hop_length'] > 2000 else (1, 8, 9, 21)
    for T in Ts:
        mels = synth.synth_mels(50 + T, 2, T, d['feat_dims'])
        up, auxf = eng.upsample(mels, full_aux=False)
        ref_up, ref_aux = wo.upsample(p, padded(mels, d['pad']))
        err_up = float(np.abs(up.cpu().numpy() - ref_up).max())
        err_aux = float(np.abs(auxf.cpu().numpy() - ref_aux[:, ::d['hop_length']]).max())
        assert err_up <= 5e-6 and err_aux <= 2e-4, f'{name} T={T}: upsample {err_up:.2e}, aux {err_aux:.2e}'
        print(f'{name} T={T}: upsample err {err_up:.2e}, aux err {err_aux:.2e}')


# ------------------------------------------------------------------------------------------------
# teacher-forced logits and Philox free runs, every kernel, every tile
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name,kernel,rows,step_kernel', RUNS, ids=[f'{n}-{k}-{r}' for n, k, r, _ in RUNS])
def test_teacher_forced_logits(shapes, name, kernel, rows, step_kernel):
    m = model(shapes, name)
    eng, pat = m['eng'], pattern(m)
    mol = m['d'].get('mode') == 'MOL'
    mels, teacher = tile(pat['mels'], rows), tile(pat['teacher'], rows)
    kw = dict(u=tile(synth.synth_mol_uniform(5, pat['steps'], NPAT), rows, axis=1)) if mol else dict(seed=3)
    out = eng.generate(mels, teacher=teacher, return_logits=True, max_steps=pat['steps'], kernel=kernel, **kw)
    eng.check()
    assert eng.last_kernel() == step_kernel
    err, bar = logit_error(out['logits'], pat['logits']), logit_bar(pat['logits'])
    print(f'{name} {step_kernel} rows={rows}: logit err {err:.2e} (bar {bar:.2e}, max|logit| {np.abs(pat["logits"]).max():.1f})')
    assert err <= bar, f'{name} {kernel} {rows} rows: teacher-forced logit error {err:.3e} > {bar:.3e}'


def _near_tie(p, mels, q, labels, t, i, cond):
    r = wo.generate(p, mels, q=q[:t + 1], teacher=labels, keep_logits=[t], max_steps=t + 1, cond=cond)
    key = r['logits'][t][i].astype(np.float64) - np.log(q[t, i].astype(np.float64))
    top = np.sort(key)[-2:]
    return (top[1] - top[0]) < 1e-3 * max(1.0, abs(top[1]))


# one free run per shape and step kernel, at its largest row count
FREE = [(n, k, r, sk) for n, k, r, sk in RUNS if r == max(rr for nn, _, rr, s in RUNS if nn == n and s == sk)]


@pytest.mark.parametrize('name,kernel,rows,step_kernel', FREE, ids=[f'{n}-{k}-{r}' for n, k, r, _ in FREE])
def test_philox_free_run(shapes, name, kernel, rows, step_kernel):
    """Philox noise, free running: the first, middle and last rows replayed through the oracle with the kernel's own noise."""
    from test_wavernn_mol_gpu import check_replay
    m = model(shapes, name)
    d, p, eng, pat = m['d'], m['p'], m['eng'], pattern(m)
    steps, seed = pat['steps'], 40 + rows
    mels = tile(pat['mels'], rows)
    out = eng.generate(mels, seed=seed, max_steps=steps, kernel=kernel, return_logits=d.get('mode') == 'MOL')
    eng.check()
    assert eng.last_kernel() == step_kernel
    sel = sorted({0, rows // 2, rows - 1})
    if d.get('mode') == 'MOL':
        u = np.concatenate([eng.philox_mol_uniform(seed, r, 1, 0, steps).cpu().numpy() for r in sel], axis=1)
        check_replay(m['sd'], mels[sel], u, out['samples'].cpu().numpy()[sel, :steps], out['logits'].cpu().numpy()[:, sel], steps=steps)
        return
    lab = out['labels'].cpu().numpy()[sel, :steps]
    q = np.concatenate([eng.philox_exponential(seed, r, 1, 0, steps).cpu().numpy() for r in sel], axis=1)
    cond = tuple(tile(c, rows)[sel] for c in pat['cond'])
    ref = wo.generate(p, mels[sel], q=q, max_steps=steps, cond=cond)
    for i, r in enumerate(sel):
        mism = np.nonzero(lab[i] != ref['labels'][i])[0]
        if mism.size:
            t = int(mism[0])
            assert _near_tie(p, mels[sel], q, ref['labels'], t, i, cond), \
                f'{name} {kernel} row {r} diverged from the oracle at step {t} without a sampling near-tie'


# ------------------------------------------------------------------------------------------------
# the wave, fold-with-overlap and sessions
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', list(SHAPES))
def test_wave_epilogue(shapes, name):
    """One full 21-frame wave per shape (kernel=auto) against the oracle's epilogue of the GPU's own labels or samples."""
    m = model(shapes, name)
    d, eng = m['d'], m['eng']
    T, hop = 21, d['hop_length']
    mels = synth.synth_mels(9, 2, T, d['feat_dims'])
    if d.get('mode') == 'MOL':
        out = eng.generate(mels, seed=2)
        eng.check()
        ref = mo.finish_wave(out['samples'].cpu().numpy(), (T - 1) * hop, hop)
        np.testing.assert_allclose(out['wave'].cpu().numpy(), ref, rtol=0, atol=1e-12)
        return
    for mu_law in (True, False):
        out = eng.generate(mels, seed=2, mu_law=mu_law)
        eng.check()
        ref = wo.finish_wave(out['labels'].cpu().numpy(), 1 << d['bits'], (T - 1) * hop, hop, mu_law=mu_law)
        np.testing.assert_allclose(out['wave'].cpu().numpy(), ref, rtol=0, atol=1e-12)


@pytest.mark.parametrize('kernel,fold,step_kernel', [('grid', (550, 50), PUSH), ('grid', (100, 20), GRID),
                                                     ('utterance', (550, 50), UTT)])
def test_fold_with_overlap_hop200(shapes, kernel, fold, step_kernel):
    """Folds of one 21-frame utterance at hop 200: teacher-forced logits of every fold against the oracle's folded run, and the
    cross-faded wave against the oracle's unfold of the GPU's labels."""
    m = model(shapes, 'hop200_compute1024')
    d, p, eng = m['d'], m['p'], m['eng']
    T, hop = 21, d['hop_length']
    target, overlap = fold
    mel = synth.synth_mels(61, 1, T, d['feat_dims'])
    nf, L = eng.fold_geometry(T, target, overlap)
    teacher = np.random.RandomState(nf).randint(0, 1024, size=(nf, L)).astype(np.int16)
    out = eng.generate(mel, seed=1, teacher=teacher, return_logits=True, kernel=kernel, fold=fold, want_wave=False)
    eng.check()
    assert eng.last_kernel() == step_kernel
    ref = wo.generate_batched(p, mel, target, overlap, teacher=teacher, keep_logits=tuple(range(L)), q=np.ones((L, nf, 1024), np.float32))
    want = np.stack([ref['logits'][s] for s in range(L)])
    err, bar = float(np.abs(out['logits'].cpu().numpy() - want).max()), logit_bar(want)
    assert err <= bar, f'{nf} folds: logit error {err:.3e} > {bar:.3e}'
    free = eng.generate(mel, seed=1, kernel=kernel, fold=fold)
    eng.check()
    lab = free['labels'].cpu().numpy()
    wave = wo.xfade_and_unfold(wo.decode_mu_law(wo.label_to_float(lab, 1024).astype(np.float64), 1024), target, overlap)
    wave = wave[:(T - 1) * hop].copy()
    wave[-20 * hop:] *= np.linspace(1, 0, 20 * hop)
    np.testing.assert_allclose(free['wave'].cpu().numpy()[0], wave, rtol=0, atol=1e-12)


@pytest.mark.parametrize('name', ['hop200_compute1024', 'hop7_pad3'])
@pytest.mark.parametrize('kernel', ['auto', 'tc'])
def test_sessions_equal_the_one_shot_run(shapes, name, kernel):
    """Two sessions of 21 frames generated in pieces of 3 hops (a multiple of hop, as tensor-core sessions need), bit-equal to the
    one-shot run on the same kernel: the push kernel for 'auto', the tensor cores for 'tc'."""
    m = model(shapes, name)
    d, eng = m['d'], m['eng']
    T, hop = 21, d['hop_length']
    mels = synth.synth_mels(71, 2, T, d['feat_dims'])
    sess = [eng.open_session(mels[i], seed=6, utterance_id=10 + i, kernel=kernel) for i in range(2)]
    labs, waves = [[], []], [[], []]
    while not all(s.done for s in sess):
        for i, (lab, wave) in enumerate(eng.advance(sess, 3 * hop)):
            labs[i].append(lab.cpu().numpy())
            waves[i].append(wave.cpu().numpy())
        eng.check()
    assert eng.last_kernel() == ('wavernn_tc_session_kernel' if kernel == 'tc' else 'wavernn_push_session_kernel')
    for s in sess:
        s.close()
    one = eng.generate(mels, seed=6, utterance_ids=[10, 11], kernel='grid' if kernel == 'auto' else 'tc')
    eng.check()
    assert eng.last_kernel() == (TC if kernel == 'tc' else PUSH)
    for i in range(2):
        assert np.array_equal(np.concatenate(labs[i]), one['labels'][i].cpu().numpy())
        assert np.array_equal(np.concatenate(waves[i]), one['wave'][i].cpu().numpy())


# ------------------------------------------------------------------------------------------------
# dispatch at the edges, and the utterance kernel's shared memory
# ------------------------------------------------------------------------------------------------
def _refused(eng, call, text):
    from tacotronv2_wavernn_chinese_b200._lib import B200TTSError
    n = eng.launch_count
    with pytest.raises(B200TTSError) as e:
        call()
    assert e.value.code == -1 and text in str(e.value), str(e.value)
    assert eng.launch_count == n, f'a refused call launched work: {e.value}'


def test_fir_past_the_tensor_core_slot_falls_back(shapes):
    eng = model(shapes, 'fir8193')['eng']
    mels = synth.synth_mels(3, 129, 3, 8)
    eng.generate(mels, seed=1, max_steps=8, want_wave=False)
    assert eng.last_kernel() == GRID
    _refused(eng, lambda: eng.generate(mels, seed=1, max_steps=8, want_wave=False, kernel='tc'), 'kernel=tc needs')
    eng8190 = model(shapes, 'fir8190')['eng']
    eng8190.generate(synth.synth_mels(3, 129, 3, 4), seed=1, max_steps=8, want_wave=False)
    assert eng8190.last_kernel() == TC


def test_aux_past_the_grid_kernel_falls_back_with_a_warning(shapes, capfd):
    """aux 132: kernel=auto runs the utterance kernel and says so once per engine (a fresh one here); kernel=grid is refused."""
    from tacotronv2_wavernn_chinese_b200.engine import WaveRNNEngine
    m = model(shapes, 'bits2_aux132')
    eng = WaveRNNEngine(m['sd'], m['d'])
    try:
        capfd.readouterr()
        eng.generate(synth.synth_mels(3, 40, 21), seed=1, max_steps=8, want_wave=False)
        eng.check()
        assert eng.last_kernel() == UTT
        assert 'falls back to the L2-streaming utterance kernel' in capfd.readouterr().err
        _refused(eng, lambda: eng.generate(synth.synth_mels(3, 4, 21), seed=1, max_steps=8, kernel='grid'), 'kernel=grid was requested')
    finally:
        eng.close()


def test_model_too_large_for_the_utterance_kernel_is_refused_before_any_launch(torch_cuda):
    """bits 15 with R = F = 2816: one row of the utterance kernel's activations and logits needs 228 KB of shared memory.  The
    call is refused before its conditioning runs, under a memory budget too."""
    import os
    from tacotronv2_wavernn_chinese_b200.engine import WaveRNNEngine
    d = dict(synth.DEFAULT_DIMS, rnn_dims=2816, fc_dims=2816, bits=15, upsample_factors=(2,), hop_length=2, compute_dims=32,
             res_blocks=0)
    sd = {k: np.zeros(v.shape, np.float32) for k, v in synth.synth_state_dict(0, dict(d, rnn_dims=128, fc_dims=128, bits=2)).items()
          if v.dtype.kind == 'f'}
    R, F, A, nc = 2816, 2816, 32, 1 << 15
    for k, shape in {'I.weight': (R, 1 + 80 + A), 'I.bias': (R,), 'rnn1.weight_ih_l0': (3 * R, R), 'rnn1.weight_hh_l0': (3 * R, R),
                     'rnn1.bias_ih_l0': (3 * R,), 'rnn1.bias_hh_l0': (3 * R,), 'rnn2.weight_ih_l0': (3 * R, R + A),
                     'rnn2.weight_hh_l0': (3 * R, R), 'rnn2.bias_ih_l0': (3 * R,), 'rnn2.bias_hh_l0': (3 * R,),
                     'fc1.weight': (F, R + A), 'fc1.bias': (F,), 'fc2.weight': (F, F + A), 'fc2.bias': (F,),
                     'fc3.weight': (nc, F), 'fc3.bias': (nc,)}.items():
        sd[k] = np.zeros(shape, np.float32)
    eng = WaveRNNEngine(sd, d)
    try:
        mels = synth.synth_mels(1, 2, 21)
        _refused(eng, lambda: eng.generate(mels, seed=1, max_steps=4), "model too large for the utterance kernel's shared memory")
        os.environ['B200TTS_MAX_COND_BYTES'] = '1000'
        try:
            _refused(eng, lambda: eng.generate(mels, seed=1), "model too large for the utterance kernel's shared memory")
        finally:
            del os.environ['B200TTS_MAX_COND_BYTES']
    finally:
        eng.close()
