"""The WaveRNN oracle at model shapes other than the shipped one, without a GPU: pinned to the reference's own runs
(tests/golden/wavernn_shapes_from_reference.npz, oracle/make_golden_wavernn_shapes.py), the create-time refusals of hparams the
reference cannot run, and proof that the GPU tests' bars catch the mistakes a kernel could make at these shapes."""
import ctypes
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import wavernn_mol_oracle as mo
from oracle import wavernn_oracle as wo
from tacotronv2_wavernn_chinese_b200 import synth

F32 = np.float32
_Z = dict(np.load(os.path.join(GOLDEN, 'wavernn_shapes_from_reference.npz')))
CASES = sorted({k.split('__')[0] for k in _Z})
RAW_CASES = [c for c in CASES if json.loads(str(_Z[c + '__dims'])).get('mode') != 'MOL']

# the GPU tests' bars (tests/test_wavernn_gpu.py, tests/test_wavernn_shapes_gpu.py)
GPU_UP, GPU_AUX, GPU_WAVE = 5e-6, 2e-4, 1e-12


def gpu_logit_bar(ref):
    return 5e-6 * max(1.0, float(np.abs(ref).max())) + 1e-4


def case(name):
    z = {k.split('__', 1)[1]: v for k, v in _Z.items() if k.startswith(name + '__')}
    d = json.loads(str(z['dims']))
    d['upsample_factors'] = tuple(d['upsample_factors'])
    wseed, mseed, nseed = (int(s) for s in z['seeds'])
    sd = synth.synth_state_dict(wseed, d, mode=d.get('mode', 'RAW'))
    B, T = int(z['B']), int(z['T'])
    mels = synth.synth_mels(mseed, B, T, d['feat_dims'])
    S = T * d['hop_length']
    if d.get('mode') == 'MOL':
        noise = synth.synth_mol_uniform(nseed, S, B)
    else:
        noise = synth.synth_exponential_noise(nseed, S, B, 1 << d['bits'])
    return z, d, wo.as_params(sd), mels, noise


def padded(mels, pad):
    B, F, T = mels.shape
    mp = np.zeros((B, F, T + 2 * pad), dtype=F32)
    mp[:, :, pad:pad + T] = mels
    return mp


def test_fixture_covers_every_dimension_the_oracle_reads():
    seen = {k: set() for k in ('rnn', 'aux', 'feat', 'ncls', 'scales', 'pad', 'hop', 'nblocks')}
    for c in CASES:
        _, _, p, _, _ = case(c)
        for k, v in wo._dims(p).items():
            seen[k].add(v)
    default = wo._dims(wo.as_params(synth.synth_state_dict(0)))
    for k, vals in seen.items():
        assert vals - {default[k]}, f'no fixture case moves {k} away from the shipped {default[k]}'
    assert 'MOL' in {json.loads(str(_Z[c + '__dims'])).get('mode') for c in CASES}
    assert os.path.getsize(os.path.join(GOLDEN, 'wavernn_shapes_from_reference.npz')) < 1_000_000


@pytest.mark.parametrize('name', CASES)
def test_upsample_matches_reference(name):
    z, d, p, mels, _ = case(name)
    up, aux = wo.upsample(p, padded(mels, d['pad']))
    st = int(z['up_stride'])
    np.testing.assert_allclose(up[:, ::st], z['mels_up_sub'], rtol=0, atol=2e-6)
    np.testing.assert_allclose(aux[:, ::d['hop_length']], z['aux_frames'], rtol=0, atol=5e-5)


def _tie(logits, q, t, i):
    key = logits[i].astype(np.float64) - np.log(q[t, i].astype(np.float64))
    top = np.sort(key)[-2:]
    return (top[1] - top[0]) < 1e-3 * max(1.0, abs(top[1]))


@pytest.mark.parametrize('name', RAW_CASES)
def test_raw_generate_matches_reference(name):
    """Teacher-forced on the reference's labels, the oracle's logits at every probe step; free running under the same noise,
    the reference's labels (or a first divergence at a sampling near-tie); the wave with mu-law on and off."""
    z, d, p, mels, q = case(name)
    steps = [int(s) for s in z['logit_steps']]
    ncls, hop = 1 << d['bits'], d['hop_length']
    r = wo.generate(p, mels, q=q, teacher=z['labels'], keep_logits=steps)
    got = np.stack([r['logits'][s] for s in steps])
    assert np.abs(got - z['logits']).max() <= 5e-6 * max(1.0, float(np.abs(z['logits']).max())) + 1e-5
    free = wo.generate(p, mels, q=q, keep_logits=None)['labels']
    for b in range(free.shape[0]):
        mism = np.nonzero(free[b] != z['labels'][b])[0]
        if mism.size:
            t = int(mism[0])
            rr = wo.generate(p, mels, q=q[:t + 1], teacher=z['labels'], keep_logits=[t], max_steps=t + 1)
            assert _tie(rr['logits'][t], q, t, b), f'{name}: utterance {b} diverged from the reference at step {t}'
    wave_len = (int(z['T']) - 1) * hop
    np.testing.assert_allclose(wo.finish_wave(z['labels'], ncls, wave_len, hop)[0], z['wave0_mu_law'], rtol=0, atol=1e-12)
    np.testing.assert_allclose(wo.finish_wave(z['labels'], ncls, wave_len, hop, mu_law=False)[0], z['wave0_linear'],
                               rtol=0, atol=1e-12)


@pytest.mark.parametrize('name', [c for c in CASES if c not in RAW_CASES])
def test_mol_generate_matches_reference(name):
    """Teacher-forced on the reference's samples: its fc3 outputs at every probe step, every sample within the bar they imply,
    and its wave."""
    z, d, p, mels, u = case(name)
    ref = z['samples']
    B = ref.shape[0]
    teacher = np.concatenate([ref, np.zeros((B, 1), F32)], axis=1)
    out = mo.generate(p, mels, u, teacher=teacher, keep_logits='all')
    bar = 5e-6 * float(np.abs(z['logits']).max()) + 1e-4
    for n, s in enumerate(z['logit_steps']):
        np.testing.assert_allclose(out['logits'][int(s)], z['logits'][n], rtol=0, atol=bar)
    for i in range(ref.shape[1]):
        k = mo.mixture_index(out['logits'][i], u[i])
        assert np.array_equal(out['mix'][:, i], k)
        d_ = np.abs(out['samples'][:, i].astype(np.float64) - ref[:, i])
        assert (d_ <= mo.sample_bar(out['logits'][i], u[i], k, bar)).all(), i
    hop = d['hop_length']
    np.testing.assert_array_equal(mo.finish_wave(teacher[:1], (int(z['T']) - 1) * hop, hop)[0], z['wave0'])


# ------------------------------------------------------------------------------------------------
# the GPU bars catch the mistakes a kernel could make at these shapes
# ------------------------------------------------------------------------------------------------
def _chain(name, mistake=None):
    """The oracle's chain on a RAW fixture case with one deliberate mistake: (upsample error, aux error, logit error, wave error)
    against the reference, each divided by its GPU bar (> 1: the GPU test would fail)."""
    z, d, p, mels, q = case(name)
    hop, pad, ncls = d['hop_length'], d['pad'], 1 << d['bits']
    A = d['res_out_dims'] // 4
    up, aux = wo.upsample(p, padded(mels, pad))
    auxf = aux[:, ::hop]
    if mistake == 'fir_phase':                      # the composite FIR read one sample late
        up = np.roll(up, 1, axis=1)
    elif mistake == 'pad':                          # mels padded with pad + 1 frames, trimmed as for pad: one frame off
        T, m_pad = mels.shape[2], padded(mels, pad + 1)
        up = wo.stretch_conv(p, m_pad, d['upsample_factors'])[:, :, pad * hop:pad * hop + T * hop]
        up = np.ascontiguousarray(up.transpose(0, 2, 1))
        auxf = wo.aux_frames(p, m_pad)[:, :T]
        aux = np.repeat(auxf, hop, axis=1)
    elif mistake == 'aux_swap':                     # a2 and a3 exchanged
        aux = aux.copy()
        aux[:, :, A:2 * A], aux[:, :, 2 * A:3 * A] = aux[:, :, 2 * A:3 * A].copy(), aux[:, :, A:2 * A].copy()
    steps = [int(s) for s in z['logit_steps'] if s <= 2 * hop + 1]
    teacher = z['labels'].astype(np.int64)
    if mistake == 'class_index':                    # the label fed back one class off (the top class one down)
        teacher = np.where(teacher < ncls - 1, teacher + 1, teacher - 1)
    r = wo.generate(p, mels, q=q, teacher=teacher, keep_logits=steps, max_steps=steps[-1] + 1, cond=(up, aux))
    got = np.stack([r['logits'][s] for s in steps])
    want = z['logits'][:len(steps)]
    st = int(z['up_stride'])
    wave_len = (int(z['T']) - 1) * hop
    mu = 1024 if mistake == 'mu_1023' else ncls                            # decode_mu_law's mu - 1 = 1023 whatever the bits
    y = wo.label_to_float(z['labels'][:1], ncls).astype(np.float64)
    wave = wo.decode_mu_law(y, mu)[:, :wave_len].copy()
    wave[:, -20 * hop:] *= np.linspace(1, 0, 20 * hop)
    return (float(np.abs(up[:, ::st] - z['mels_up_sub']).max()) / GPU_UP,
            float(np.abs(auxf - z['aux_frames']).max()) / GPU_AUX,
            float(np.abs(got - want).max()) / gpu_logit_bar(want),
            float(np.abs(wave[0] - z['wave0_mu_law']).max()) / GPU_WAVE)


def test_unperturbed_chain_passes_the_gpu_bars():
    for name in RAW_CASES:
        assert max(_chain(name)) <= 1.0, name


@pytest.mark.parametrize('mistake', ['fir_phase', 'pad', 'aux_swap', 'class_index', 'mu_1023'])
def test_each_mistake_fails_a_gpu_bar(mistake):
    worst = {name: max(_chain(name, mistake)) for name in RAW_CASES}
    assert max(worst.values()) > 1.0, f'{mistake}: within every GPU bar on every fixture shape: {worst}'


# ------------------------------------------------------------------------------------------------
# hparams the reference cannot run are refused at create time, before any CUDA call
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('field,value,text', [('pad', 0, 'pad must be >= 1'), ('pad', -1, 'pad must be >= 1'),
                                              ('feat_dims', 0, 'feat_dims must be >= 1'),
                                              ('compute_dims', 0, 'compute_dims must be >= 1'),
                                              ('res_blocks', -1, 'res_blocks must be >= 0')])
def test_create_refuses_hparams_without_a_device(field, value, text):
    from tacotronv2_wavernn_chinese_b200 import _lib as L
    from tacotronv2_wavernn_chinese_b200.engine import _cfg_from_dims
    lib = L.load()
    sd = synth.synth_state_dict(0)
    arr, keep = L.make_tensor_array({k: np.asarray(v, dtype=F32) for k, v in sd.items() if np.asarray(v).dtype.kind == 'f'})
    cfg = _cfg_from_dims(dict(synth.DEFAULT_DIMS, **{field: value}))
    h = ctypes.c_void_p()
    for create in (lib.b200tts_wavernn_create, lib.b200tts_wavernn_create_mol):
        assert create(ctypes.byref(h), 0, ctypes.byref(cfg), arr, len(arr)) == -1 and not h.value      # B200TTS_EINVAL
        assert text in lib.b200tts_last_error().decode()
    del keep
