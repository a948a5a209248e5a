"""Mixture-of-logistics WaveRNN (voc_mode = 'MOL') without a GPU: the oracle pinned to the reference's own MOL runs, the
sampler against the reference's sample_from_discretized_mix_logistic, the uniform-injecting harness, the C-ABI refusals and
the model mirror."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import ref_harness as rh
from oracle import wavernn_mol_oracle as mo
from tacotronv2_wavernn_chinese_b200 import synth

GOLDEN = os.path.join(ROOT, 'tests', 'golden')
F32 = np.float32


def logit_bar(ref):
    """The fc3 bar of the RAW parity tests."""
    return 5e-6 * float(np.abs(ref).max()) + 1e-4


def _fixture(name):
    z = dict(np.load(os.path.join(GOLDEN, name)))
    p = synth.synth_state_dict(int(z['weight_seed']), mode='MOL')
    return z, p


@pytest.mark.parametrize('batched', [False, True], ids=['T24', 'batched_T30'])
def test_oracle_pinned_to_reference(batched):
    """Teacher-forced on the reference's samples, the oracle gives its fc3 outputs, the same mixture at every step, every
    sample within the bar the fc3 bar implies, and the reference's wave."""
    if batched:
        z, p = _fixture('wavernn_mol_synth_batched_T30.npz')
        T, target, overlap = int(z['T']), int(z['target']), int(z['overlap'])
        ref = z['samples']
        nf, L = ref.shape[0], ref.shape[1] + 1
        u = synth.synth_mol_uniform(int(z['u_seed']), L, nf)
        teacher = np.concatenate([ref, np.zeros((nf, 1), F32)], axis=1)
        out = mo.generate_batched(p, synth.synth_mels(int(z['mel_seed']), 1, T), target, overlap, u, teacher=teacher,
                                  keep_logits='all')
    else:
        z, p = _fixture('wavernn_mol_synth_T24.npz')
        B, T = int(z['B']), int(z['T'])
        ref = z['samples']
        u = synth.synth_mol_uniform(int(z['u_seed']), T * 275, B)
        teacher = np.concatenate([ref, np.zeros((B, 1), F32)], axis=1)
        out = mo.generate(p, synth.synth_mels(int(z['mel_seed']), B, T), u, teacher=teacher, keep_logits='all')
    S = ref.shape[1]
    for n, s in enumerate(z['probe']):
        np.testing.assert_allclose(out['logits'][int(s)], z['logits'][n], rtol=0, atol=logit_bar(z['logits'][n]))
    err = logit_bar(z['logits'])
    worst = 0.0
    for i in range(S):
        pi = out['logits'][i]
        k_ref = mo.mixture_index(pi, u[i])         # the reference's choice under the same u, up to fc3 rounding
        assert np.array_equal(out['mix'][:, i], k_ref)
        bar = mo.sample_bar(pi, u[i], k_ref, err)
        d = np.abs(out['samples'][:, i].astype(np.float64) - ref[:, i])
        assert (d <= bar).all(), (i, d.max(), bar.max())
        worst = max(worst, float((d / bar).max()))
    # the wave is the samples in float64, faded: bit for bit from the reference's own samples (the last sample of a fold or
    # utterance is never heard: it falls past wave_len or on a zero of the fold's fade-out)
    if batched:
        np.testing.assert_array_equal(mo.unfold_wave(teacher, target, overlap, (T - 1) * 275, 275), z['wave'])
    else:
        np.testing.assert_array_equal(mo.finish_wave(teacher[:1], (T - 1) * 275, 275)[0], z['wave0'])
    assert worst <= 1.0


needs_ref = pytest.mark.skipif(not rh.available(), reason='the reference is only present in the build container')


def _ref_sampler():
    rh.import_reference()
    sys.path.insert(0, rh.REF_ROOT)
    try:
        from wavernn.utils.distribution import sample_from_discretized_mix_logistic
    finally:
        sys.path.remove(rh.REF_ROOT)
    return sample_from_discretized_mix_logistic


@needs_ref
def test_sampler_matches_reference_on_crafted_parameters():
    """sample_mol == the reference's sample_from_discretized_mix_logistic, fed the same uniforms, on parameters that reach
    every branch: means beyond +-1, log-scales below log(1e-14), tied mixture logits, uniforms at both ends of the range."""
    from oracle.ref_harness_mol import _UniformFeeder
    sample = _ref_sampler()
    rs = np.random.RandomState(5)
    B = 512
    p = rs.uniform(-3, 3, (B, 30)).astype(F32)
    p[:, 10:20] = rs.uniform(-2.5, 2.5, (B, 10))
    p[::3, 20:30] = rs.uniform(-60, -20, (B // 3 + 1, 10))
    p[1::4, :10] = 0.75                                             # all ten mixture logits tied
    u = rs.uniform(1e-5, 1 - 1e-5, (1, B, 11)).astype(F32)
    u[0, ::7, 10] = F32(1e-5)
    u[0, 3::7, 10] = F32(1 - 1e-5)
    u[0, 1::4, :10] = 0.5                                           # tied logits and tied noise: the first mixture wins
    feeder = _UniformFeeder(u)
    orig = torch.Tensor.uniform_
    torch.Tensor.uniform_ = lambda t, a=0.0, b=1.0, **kw: feeder(t, a, b)
    try:
        ref = sample(torch.as_tensor(p).T.unsqueeze(0)).numpy().reshape(-1)
    finally:
        torch.Tensor.uniform_ = orig
    x, k = mo.sample_mol(p, u[0])
    assert (k[1::4] == 0).all()
    assert (np.abs(ref) == 1).sum() > 50 and (np.maximum(p[np.arange(B), 20 + k], -100) < mo.LOG_SCALE_MIN).sum() > 50
    # torch's vectorised log / exp may round differently from numpy's by an ulp: compare within the sampler's rounding bar
    bar = mo.sample_bar(p, u[0], k, 0.0)
    assert (np.abs(x.astype(np.float64) - ref) <= bar).all()


@needs_ref
def test_harness_feeds_exactly_the_injected_uniforms():
    """Two uniform_ calls per step, all served from u; other uniforms give other samples."""
    from oracle import ref_harness_mol as rhm
    model = rhm.build_model_mol(synth.synth_state_dict(21, mode='MOL'))
    mels = synth.synth_mels(7, 1, 21)
    S = 21 * 275
    u1 = synth.synth_mol_uniform(1, S, 1)
    r1 = rhm.reference_generate_mol(model, mels, u1)
    assert r1['uniform_calls'] == 2 * S and r1['steps'] == S
    r1b = rhm.reference_generate_mol(model, mels, u1)
    np.testing.assert_array_equal(r1['inputs'], r1b['inputs'])
    r2 = rhm.reference_generate_mol(model, mels, synth.synth_mol_uniform(2, S, 1))
    assert not np.array_equal(r1['inputs'], r2['inputs'])
    # and the oracle, on the same u and teacher-forced on the reference's own samples, reproduces that run within the sampler's bar
    out = mo.generate(synth.synth_state_dict(21, mode='MOL'), mels, u1, teacher=np.concatenate(
        [r1['inputs'], np.zeros((1, 1), F32)], axis=1), max_steps=S - 1)
    assert np.abs(out['samples'] - r1['inputs']).max() < 1e-3


def _lib():
    from tacotronv2_wavernn_chinese_b200 import build, _lib
    build.build_lib()
    return _lib.load(), _lib


def test_abi_refusals_before_any_cuda_call():
    lib, L = _lib()
    assert lib.b200tts_abi_version() == 3
    for name in ('b200tts_wavernn_create_mol', 'b200tts_wavernn_generate_mol', 'b200tts_philox_mol_uniform'):
        assert hasattr(lib, name) and name in L.SIGNATURES
    assert ctypes.sizeof(L.Rng) == 40 and ctypes.sizeof(L.GenOpts) == 80 and ctypes.sizeof(L.WaveRNNCfg) == 56
    rng, opts = L.Rng(), L.GenOpts()
    buf = (ctypes.c_float * 16)()
    assert lib.b200tts_wavernn_generate_mol(None, buf, 1, 21, ctypes.byref(rng), ctypes.byref(opts), None, buf, None, None) == -1
    assert lib.b200tts_philox_mol_uniform(0, 1, 0, 0, 0, 1, buf, None) == -1
    assert lib.b200tts_philox_mol_uniform(0, 1, 0, 1, 0, 1, None, None) == -1
    assert lib.b200tts_wavernn_create_mol(None, 0, None, None, 0) == -1


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the behaviour without a device')
def test_create_mol_fails_loudly_without_a_device():
    lib, L = _lib()
    from tacotronv2_wavernn_chinese_b200.engine import _cfg_from_dims
    sd = synth.synth_state_dict(0, mode='MOL')
    arr, keep = L.make_tensor_array({k: v for k, v in sd.items() if v.dtype == np.float32})
    cfg = _cfg_from_dims(synth.DEFAULT_DIMS)
    h = ctypes.c_void_p()
    assert lib.b200tts_wavernn_create_mol(ctypes.byref(h), 0, ctypes.byref(cfg), arr, len(arr)) == -2
    assert not h.value


def test_mirror_builds_a_mol_model(tmp_path):
    code = f'''
import sys
sys.path.insert(0, {ROOT!r})
import wavernn_gen
from tacotronv2_wavernn_chinese_b200.wavernn.utils import hparams as hp
hp.configure({str(tmp_path / "mol_hparams.py")!r})
m = wavernn_gen.build_model()
assert m.mode == "MOL" and m.n_classes == 30 and m._dims["mode"] == "MOL", (m.mode, m.n_classes)
assert tuple(m.fc3.weight.shape) == (30, 512)
from tacotronv2_wavernn_chinese_b200 import synth
missing = m.load_state_dict({{k: __import__("torch").as_tensor(v) for k, v in synth.synth_state_dict(0, mode="MOL").items()}},
                            strict=False)
assert not missing.missing_keys
print("OK")
'''
    src = open(os.path.join(ROOT, 'wavernn_hparams.py')).read().replace("voc_mode = 'RAW'", "voc_mode = 'MOL'")
    assert "voc_mode = 'MOL'" in src
    (tmp_path / 'mol_hparams.py').write_text(src)
    r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0 and 'OK' in r.stdout, r.stdout + r.stderr
