"""The library's noise on the device against an independent statement of it (tests/philox_ref.py), and what the step kernels
draw from it against the float64 distributions the sampling contract (DESIGN section 4) states.

- The four noise dumps (WaveRNN Exp(1) noise and MOL uniforms, Griffin-Lim phase uniforms, Tacotron keep flags) equal the
  restatement at the edges of their keys: 64-bit seeds, utterance ids across 2^32 and up to 2^64 - 1, the last step a dump
  accepts.  Flags and uniforms bit for bit; Exp(1) noise within 1 ulp of float64 -log(u), the CUDA bound for logf.
- Streams keyed by the same (seed, utterance id) are independent: one bit of each agrees with one bit of any other half the time.
- The RAW step kernels draw labels from softmax(logits) and the MOL kernels samples from the clamped logistic mixture, tested
  by chi-square and Kolmogorov-Smirnov tests on fixed seeds (deterministic) at p > 1e-6.
"""
import math

import numpy as np
import pytest
from scipy import stats

import philox_ref as pr
from tacotronv2_wavernn_chinese_b200 import synth

pytestmark = pytest.mark.gpu

P_MIN = 1e-6
SEEDS = [0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 63, 2 ** 64 - 1, -12345]
# (utterance_offset, B): plain, ids across 2^32, ids ending at 2^64 - 1
OFFSETS = [(7, 3), (2 ** 32 - 2, 4), (2 ** 64 - 4, 4)]
LAST_STEP = 2 ** 31 - 1          # largest step0 + n_steps the WaveRNN dumps accept


@pytest.fixture(scope='module')
def engines():
    import torch
    if not torch.cuda.is_available():
        pytest.fail('GPU tests need a CUDA device')
    from tacotron_hparams import hparams
    from taco_common import synth_taco_weights
    from tacotronv2_wavernn_chinese_b200.engine import WaveRNNEngine
    from tacotronv2_wavernn_chinese_b200.tacotron.engine import TacoDecoderEngine
    from tacotronv2_wavernn_chinese_b200.tacotron.griffin_lim import GriffinLimEngine
    e = dict(raw=WaveRNNEngine(synth.synth_state_dict(5), synth.DEFAULT_DIMS, device=0),
             mol=WaveRNNEngine(synth.synth_state_dict(21, mode='MOL'), dict(synth.DEFAULT_DIMS, mode='MOL'), device=0),
             gl=GriffinLimEngine(hparams, device=0), taco=TacoDecoderEngine(synth_taco_weights(7), device=0))
    yield e
    for v in e.values():
        v.close()


# ------------------------------------------------------------------------------------------------
# the dumps against the restatement
# ------------------------------------------------------------------------------------------------
def _check_exponential(q, seed, ids, step0):
    n_steps, _, nc = q.shape
    u, q_ref = pr.raw_exponential(seed, ids, step0, n_steps, nc)
    assert np.array_equal(u.astype(np.float32).astype(np.float64), u)         # u is exact in fp32, as the kernel forms it
    ulp = np.spacing(np.abs(q_ref).astype(np.float32)).astype(np.float64)
    err = np.abs(q.astype(np.float64) - q_ref) / ulp
    w = np.unravel_index(int(err.argmax()), err.shape)
    assert err.max() <= 1.0, f'q {q[w]!r} vs -log(u) = {q_ref[w]!r} (u = {u[w]!r}): {err.max():.3f} ulp at (step, row, class) {w}'


@pytest.mark.parametrize('offset,B', OFFSETS)
@pytest.mark.parametrize('seed', SEEDS)
def test_dumps_equal_the_restatement(engines, seed, offset, B):
    ids = pr.ids_of(offset, B)
    q = engines['raw'].philox_exponential(seed, offset, B, 3, 40).cpu().numpy()
    _check_exponential(q, seed, ids, 3)
    u = engines['mol'].philox_mol_uniform(seed, offset, B, 3, 40).cpu().numpy()
    assert np.array_equal(u, pr.mol_uniform(seed, ids, 3, 40))
    g = engines['gl'].philox_uniform(seed, offset, B, 12).cpu().numpy()
    assert g.shape[2] == 1025 and np.array_equal(g, pr.gl_uniform(seed, ids, 12, 1025))
    m = engines['taco'].philox_masks(seed, offset, B, 48).cpu().numpy()
    assert np.array_equal(m, pr.taco_keep(seed, ids, 48, 256))


@pytest.mark.parametrize('seed', [0, 2 ** 64 - 1])
def test_wavernn_dumps_at_the_last_step(engines, seed):
    """Steps up to 2^31 - 2, the last a dump accepts; one more is refused."""
    from tacotronv2_wavernn_chinese_b200._lib import B200TTSError
    n, off, B = 24, 2 ** 32 - 2, 4
    ids = pr.ids_of(off, B)
    q = engines['raw'].philox_exponential(seed, off, B, LAST_STEP - n, n).cpu().numpy()
    _check_exponential(q, seed, ids, LAST_STEP - n)
    u = engines['mol'].philox_mol_uniform(seed, off, B, LAST_STEP - n, n).cpu().numpy()
    assert np.array_equal(u, pr.mol_uniform(seed, ids, LAST_STEP - n, n))
    with pytest.raises(B200TTSError):
        engines['raw'].philox_exponential(seed, off, B, LAST_STEP - n + 1, n)
    with pytest.raises(B200TTSError):
        engines['mol'].philox_mol_uniform(seed, off, B, LAST_STEP - n + 1, n)


# ------------------------------------------------------------------------------------------------
# streams keyed by the same (seed, id) are independent
# ------------------------------------------------------------------------------------------------
def test_streams_with_one_key_are_independent(engines):
    """Tacotron keep flags, WaveRNN RAW noise and MOL uniforms and Griffin-Lim uniforms drawn with one seed and one set of ids
    (the pipeline keys both models so).  A keep flag is the top bit of its word; `q < ln 2` and `u >= 0.5` are the top bits of
    theirs.  Were two streams to read the same counters, those bits would agree always; independent, half the time (+- 6 sigma)."""
    seed, off, B, steps, P = 2024, 2 ** 32 - 5, 8, 400, 256
    keep = engines['taco'].philox_masks(seed, off, B, steps).cpu().numpy().astype(bool)          # [B, steps, 2, P]
    q = engines['raw'].philox_exponential(seed, off, B, 0, steps).cpu().numpy()                 # [steps, B, 1024]
    u_mol = engines['mol'].philox_mol_uniform(seed, off, B, 0, steps).cpu().numpy()            # [steps, B, 11]
    u_gl = engines['gl'].philox_uniform(seed, off, B, steps).cpu().numpy()                     # [B, steps, 1025]
    flags = keep.reshape(B, steps, 2 * P)                                                      # class / bin index L * P + j
    pairs = {
        'keep / RAW q < ln 2': (flags, np.transpose(q, (1, 0, 2))[:, :, :2 * P] < np.float32(math.log(2.0))),
        'keep / MOL u >= 0.5': (flags[:, :, :11], np.transpose(u_mol, (1, 0, 2)) >= 0.5),
        'keep / GL u >= 0.5': (flags, u_gl[:, :, :2 * P] >= 0.5),
        'RAW q < ln 2 / GL u >= 0.5': (np.transpose(q, (1, 0, 2))[:, :, :1024] < np.float32(math.log(2.0)), u_gl[:, :, :1024] >= 0.5),
        'MOL u / GL u >= 0.5': (np.transpose(u_mol, (1, 0, 2)) >= 0.5, u_gl[:, :, :11] >= 0.5),
    }
    for name, (a, b) in pairs.items():
        agree = float((a == b).mean())
        six = 6 * 0.5 / math.sqrt(a.size)
        print(f'{name}: agreement {agree:.5f} over {a.size} pairs (bar 0.5 +- {six:.5f})')
        assert abs(agree - 0.5) <= six, f'{name}: agreement {agree:.5f} over {a.size} pairs'


# ------------------------------------------------------------------------------------------------
# what the step kernels sample
# ------------------------------------------------------------------------------------------------
DRAWS = 1_000_000
MAX_FRAMES = 402                 # the longest utterance the suite generates (BASELINE config 2)
# every row-group variant test_wavernn_gpu.py's mapping tests run: push kernel G = 4/8/16/32 up to 32 rows, wide grid above;
# the tensor-core kernel with a second group of one row and with two full groups; the utterance kernel
RAW_VARIANTS = [('grid', B) for B in (256, 300, 128, 100, 64, 32, 20, 12, 7, 3)] + [('tc', 129), ('tc', 256), ('utterance', 64)]


def _raw_logits():
    """fc3 biases with a wide spread: a run of exactly equal logits, and a tail of classes too rare to test one by one."""
    rs = np.random.RandomState(1)
    b = rs.normal(0.0, 1.5, 1024)
    b[100:110] = b[100]
    b[500:520] = 0.0
    b[900:] = np.linspace(-4.0, -9.0, 124)
    return b.astype(np.float32)


def _step_kernel(kernel, B):
    if kernel == 'grid':
        return 'wavernn_push_kernel' if B <= 32 else 'wavernn_grid_kernel'
    return {'tc': 'wavernn_tc_kernel', 'utterance': 'wavernn_utt_kernel'}[kernel]


def _runs(B):
    """(frames, steps, calls) that give >= DRAWS draws on B rows in utterances no longer than MAX_FRAMES."""
    steps = min(MAX_FRAMES * 275, max(21 * 275, -(-DRAWS // B)))
    return -(-steps // 275), steps, -(-DRAWS // (B * steps))


def _free_run(eng, kernel, B, seed0, step_kernel):
    """Free-running outputs [calls][B, steps] (labels or MOL samples), each call on fresh mels and its own seed."""
    T, steps, calls = _runs(B)
    outs = []
    for c in range(calls):
        out = eng.generate(synth.synth_mels(seed0 + c, B, T), seed=seed0 + c, kernel=kernel, max_steps=steps, want_wave=False)
        assert eng.last_kernel() == step_kernel
        outs.append((out['samples'] if eng.mode == 'MOL' else out['labels'])[:, :steps].cpu().numpy())
    return outs


@pytest.fixture(scope='module')
def raw_engine():
    from tacotronv2_wavernn_chinese_b200.engine import WaveRNNEngine
    sd = synth.synth_state_dict(3)
    sd['fc3.weight'] = np.zeros_like(sd['fc3.weight'])
    sd['fc3.bias'] = _raw_logits()
    e = WaveRNNEngine(sd, synth.DEFAULT_DIMS, device=0)
    yield e
    e.close()


def _equal_pair_bound(p, n):
    """Mean and 6 sigma of the rate of equal labels over n overlapping pairs (x_t, x_t+1) of an iid sequence; non-overlapping
    pairs have the same mean and a smaller variance."""
    s2, s3 = float((p ** 2).sum()), float((p ** 3).sum())
    var = (s2 - s2 * s2) / n + 2.0 * max(s3 - s2 * s2, 0.0) / n
    return s2, 6.0 * math.sqrt(var)


@pytest.mark.parametrize('kernel,B', RAW_VARIANTS)
def test_raw_labels_follow_the_softmax(raw_engine, kernel, B):
    """fc3.weight = 0 makes every step's logits exactly the fc3 bias b, whatever the input, so the labels are iid draws from
    softmax(b).  Chi-square of the label histogram against float64 softmax(b) (classes expected fewer than 20 times pooled into
    one bin), and the rate of equal labels at steps (t, t+1) of a row and in rows (r, r+1) of a step against sum(p^2)."""
    b = _raw_logits().astype(np.float64)
    p = np.exp(b - b.max())
    p /= p.sum()
    outs = _free_run(raw_engine, kernel, B, 7000 + B, _step_kernel(kernel, B))
    lab = np.concatenate([o.ravel() for o in outs]).astype(np.int64)
    n = lab.size
    assert n >= DRAWS and lab.min() >= 0 and lab.max() < 1024
    obs, want = np.bincount(lab, minlength=1024).astype(np.float64), n * p
    rare = want < 20
    o = np.append(obs[~rare], obs[rare].sum())
    e = np.append(want[~rare], want[rare].sum())
    chi = float(((o - e) ** 2 / e).sum())
    pv = float(stats.chi2.sf(chi, o.size - 1))
    print(f'{kernel} B={B}: {n} labels, chi2 {chi:.1f} on {o.size - 1} dof, p = {pv:.3g}')
    assert pv > P_MIN, f'{kernel} B={B}: label histogram is not softmax(b): chi2 {chi:.1f} on {o.size - 1} dof, p = {pv:.3g}'
    for axis, name in ((1, 'steps (t, t+1)'), (0, 'rows (r, r+1)')):
        eq = [np.diff(run, axis=axis) == 0 for run in outs]
        m = sum(int(x.sum()) for x in eq)
        cnt = sum(x.size for x in eq)
        mean, six = _equal_pair_bound(p, cnt)
        print(f'{kernel} B={B}: equal labels at {name}: {m / cnt:.6f} over {cnt} pairs, sum p^2 = {mean:.6f} +- {six:.6f}')
        assert abs(m / cnt - mean) <= six, f'{kernel} B={B}: equal labels at {name}: {m / cnt:.6f} vs {mean:.6f} +- {six:.6f}'


MOL_LOG_SCALE_MIN = float(np.float32(np.log(1e-14)))
MOL_VARIANTS = [('auto', 16, 'wavernn_push_kernel'), ('auto', 40, 'wavernn_grid_kernel'), ('utterance', 40, 'wavernn_utt_kernel')]


def _mol_bias():
    """fc3 biases of the MOL head: 10 mixture logits, 10 means, 10 log-scales.  Component 0 has log-scale -40, below the
    sampler's floor log(1e-14), and mean 0.3: every sample it gives rounds to float32(0.3) exactly.  Component 1 reaches past
    +1 and component 2 past -1, so both clamp atoms have mass."""
    logits = [0.4, 0.0, -0.2, 0.3, -0.6, 0.1, 0.2, -0.1, 0.5, -0.3]
    means = [0.3, 0.9, -0.95, -0.5, 0.1, 0.55, -0.2, 0.7, -0.7, 0.0]
    scales = [-40.0, -1.5, -2.0, -3.0, -2.5, -3.5, -2.2, -4.0, -2.8, -3.2]
    return np.array(logits + means + scales, dtype=np.float32)


class _Mixture:
    """The float64 law of the MOL sample: a logistic mixture clamped to [-1, 1] (atoms at -1 and +1), whose floor-scale component
    is an atom at its mean."""

    def __init__(self, bias):
        b = bias.astype(np.float64)
        w = np.exp(b[:10] - b[:10].max())
        self.pi = w / w.sum()
        self.mu = b[10:20]
        self.s = np.exp(np.maximum(b[20:30], MOL_LOG_SCALE_MIN))
        self.atom = self.s < 1e-9                     # components that are an atom at their mean in fp32

    def cont(self, x, left=False):
        """Unclamped mixture CDF at x (left: the limit from the left)."""
        x = np.asarray(x, dtype=np.float64)[..., None]
        z = (x - self.mu) / np.where(self.atom, 1.0, self.s)
        logistic = 0.5 * (1.0 + np.tanh(0.5 * z))
        step = (x > self.mu) if left else (x >= self.mu)
        return (np.where(self.atom, step, logistic) * self.pi).sum(-1)

    def cdf(self, x, left=False):
        x = np.asarray(x, dtype=np.float64)
        f = self.cont(x, left)
        if left:
            return np.where(x > 1.0, 1.0, np.where(x <= -1.0, 0.0, f))
        return np.where(x >= 1.0, 1.0, np.where(x < -1.0, 0.0, f))


def _ks_with_atoms(x, law):
    """Kolmogorov-Smirnov distance between the sample x and a CDF with atoms: both sides of every distinct sample value."""
    v, cnt = np.unique(x.astype(np.float64), return_counts=True)
    n = x.size
    hi = np.cumsum(cnt) / n
    lo = hi - cnt / n
    return float(max(np.abs(hi - law.cdf(v)).max(), np.abs(lo - law.cdf(v, left=True)).max()))


@pytest.fixture(scope='module')
def mol_engine():
    from tacotronv2_wavernn_chinese_b200.engine import WaveRNNEngine
    sd = synth.synth_state_dict(4, mode='MOL')
    sd['fc3.weight'] = np.zeros_like(sd['fc3.weight'])
    sd['fc3.bias'] = _mol_bias()
    e = WaveRNNEngine(sd, dict(synth.DEFAULT_DIMS, mode='MOL'), device=0)
    yield e
    e.close()


@pytest.mark.parametrize('kernel,B,name', MOL_VARIANTS)
def test_mol_samples_follow_the_mixture(mol_engine, kernel, B, name):
    """fc3.weight = 0: every step's mixture parameters are exactly the fc3 bias, so the samples are iid draws from the clamped
    mixture.  A Kolmogorov-Smirnov test against its float64 CDF, atoms included (conservative where the law has atoms), and the
    frequency of float32(0.3), the atom of the floor-scale component, against that component's weight: the mixture choice
    itself, within 6 sigma.  The sampler truncates its uniforms to [1e-5, 1 - 1e-5]; that moves the law by O(1e-5), under the
    test's resolution (about 3e-3 at 1 M samples)."""
    law = _Mixture(_mol_bias())
    outs = _free_run(mol_engine, kernel, B, 8000 + B, name)
    x = np.concatenate([o.ravel() for o in outs])
    n = x.size
    assert n >= DRAWS and np.isfinite(x).all() and x.min() >= -1.0 and x.max() <= 1.0
    d = _ks_with_atoms(x, law)
    pv = float(stats.kstwo.sf(d, n))
    atoms = {'-1': (x == -1.0).mean(), '+1': (x == 1.0).mean(), '0.3': (x == np.float32(0.3)).mean()}
    want = {'-1': law.cont(-1.0, left=True), '+1': 1.0 - law.cont(1.0), '0.3': law.pi[0]}
    print(f'{kernel} B={B}: {n} samples, KS D {d:.2e}, p = {pv:.3g}; atoms ' +
          ', '.join(f'{k}: {atoms[k]:.5f} (law {float(want[k]):.5f})' for k in atoms))
    assert pv > P_MIN, f'{kernel} B={B}: samples do not follow the mixture: KS D {d:.3e}, p = {pv:.3g}'
    for k in atoms:
        w = float(want[k])
        assert w > 0.005 and abs(atoms[k] - w) <= 6 * math.sqrt(w * (1 - w) / n), (k, atoms[k], w)
