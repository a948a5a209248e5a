"""Import and drive the UNMODIFIED reference WaveRNN from /root/reference -- container-only test tooling.

Used by oracle/make_golden_wavernn.py (golden fixtures) and by tests that are
skipped when /root/reference is absent (it does not exist on the GPU box).
Nothing here is copied from the reference: the reference package is imported
in-process with three shims (SURVEY.md Appendix A): stub `matplotlib` and
`librosa` (absent here, unused on this path), and `np.cumproduct` (removed in
numpy 2, used at wavernn/models/fatchord_version.py:68).
"""
from __future__ import annotations

import os
import sys
import types
import contextlib

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# /root/reference exists only in the build container.  __graft_entry__.build() makes a git-ignored TRAVEL COPY of the
# reference's own `wavernn/` package + `wavernn_hparams.py` + checkpoint under oracle/_ref/ (never committed) so that
# bench.py's CPU arm can run the UNMODIFIED reference on the GPU box's host cores.
TRAVEL_ZIP = os.path.join(_HERE, '_ref', 'reference_src.zip')
TRAVEL_CKPT = os.path.join(_HERE, '_ref', 'latest_weights.pyt')
_unpacked = None


def _travel_root():
    """Unpacks the travel archive into a fresh temp dir (removed at interpreter exit) and returns it, or None."""
    global _unpacked
    if _unpacked is None and os.path.isfile(TRAVEL_ZIP):
        import atexit
        import shutil
        import tempfile
        import zipfile
        d = tempfile.mkdtemp(prefix='b200tts_ref_')
        with zipfile.ZipFile(TRAVEL_ZIP) as z:
            z.extractall(d)
        atexit.register(shutil.rmtree, d, True)
        _unpacked = d
    return _unpacked


def _pick_root():
    env = os.environ.get('B200TTS_REFERENCE')
    for cand in (env, '/root/reference'):
        if cand and os.path.isfile(os.path.join(cand, 'wavernn/models/fatchord_version.py')):
            return cand
    return _travel_root() or env or '/root/reference'


REF_ROOT = _pick_root()
REF_CKPT = os.path.join(REF_ROOT, 'logs_wavernn/checkpoints/latest_weights.pyt')
if not os.path.isfile(REF_CKPT) and os.path.isfile(TRAVEL_CKPT):
    REF_CKPT = TRAVEL_CKPT


def available() -> bool:
    return os.path.isfile(os.path.join(REF_ROOT, 'wavernn/models/fatchord_version.py'))


_fv = None


def import_reference():
    """Returns the reference module `wavernn.models.fatchord_version` (imported once)."""
    global _fv
    if _fv is not None:
        return _fv
    if not available():
        raise RuntimeError(f'reference not found under {REF_ROOT}')
    mpl = types.ModuleType('matplotlib')
    mpl.use = lambda *a, **k: None
    mpl.interactive = lambda *a, **k: None
    plt = types.ModuleType('matplotlib.pyplot')
    mpl.pyplot = plt
    for name, mod in (('matplotlib', mpl), ('matplotlib.pyplot', plt), ('librosa', types.ModuleType('librosa'))):
        sys.modules.setdefault(name, mod)
    if not hasattr(np, 'cumproduct'):
        np.cumproduct = np.cumprod
    # our own drop-in package is also called `wavernn` at some call sites; make sure the reference wins here
    for k in [k for k in sys.modules if k == 'wavernn' or k.startswith('wavernn.')]:
        del sys.modules[k]
    sys.path.insert(0, REF_ROOT)
    try:
        from wavernn.utils import hparams as hp
        if not hp.is_configured():
            hp.configure(os.path.join(REF_ROOT, 'wavernn_hparams.py'))
        from wavernn.models import fatchord_version as fv
    finally:
        sys.path.remove(REF_ROOT)
    fv.save_wav = lambda x, p: None          # librosa.output.write_wav no longer exists (dsp.py:23)
    fv.stream = lambda *a, **k: None         # silence the \r progress line (display.py:17)
    fv._hp = hp
    _fv = fv
    return fv


def build_model(state_dict=None, dims=None, mode=None):
    """Reference WaveRNN with the shipped hparams, or with `dims` (keys of synth.DEFAULT_DIMS) and voc_mode `mode` when given;
    loads `state_dict` (numpy/torch) or the shipped checkpoint."""
    fv = import_reference()
    hp = fv._hp
    if dims is None:
        args = (hp.voc_rnn_dims, hp.voc_fc_dims, hp.bits, hp.voc_pad, hp.voc_upsample_factors, hp.num_mels, hp.voc_compute_dims,
                hp.voc_res_out_dims, hp.voc_res_blocks, hp.hop_length, hp.sample_rate)
    else:
        args = tuple(dims[k] for k in ('rnn_dims', 'fc_dims', 'bits', 'pad', 'upsample_factors', 'feat_dims', 'compute_dims',
                                       'res_out_dims', 'res_blocks', 'hop_length', 'sample_rate'))
    with contextlib.redirect_stdout(open(os.devnull, 'w')):
        m = fv.WaveRNN(*args, mode if mode is not None else hp.voc_mode)
    if state_dict is None:
        m.load(REF_CKPT)
    else:
        sd = {k: torch.as_tensor(np.asarray(v)) for k, v in state_dict.items()}
        missing = m.load_state_dict(sd, strict=False)
        assert not missing.missing_keys, missing
    return m


class _RaceCategorical:
    """Stand-in for torch.distributions.Categorical whose sample() is `argmax(p / q_step)` with injected q.

    torch.multinomial(p, 1, replacement=True) on CPU is exactly `argmax(p / Exp(1))`
    (SURVEY.md 7.3-2); feeding q from a tensor lets the reference, the oracle and the
    CUDA kernels share the noise.
    """
    q = None          # torch [S, B, ncls]
    step = 0
    labels = None     # list of [B] tensors

    def __init__(self, probs):
        self.p = probs

    def sample(self):
        cls = type(self)
        lab = (self.p / cls.q[cls.step]).argmax(-1)
        cls.step += 1
        cls.labels.append(lab.clone())
        return lab


def reference_generate(model, mels, q, capture_logits_at=(), batched=False, target=None, overlap=None, mu_law=None):
    """Runs the reference `generate` (fatchord_version.py:169) unbatched with injected noise (mu_law None: the hparams' value).

    Returns dict(wave0 float64 [wave_len] (utterance 0 only -- :253), labels [B,S] int16, logits {step: [B,ncls]}).
    """
    fv = import_reference()
    want = set(int(s) for s in capture_logits_at)
    kept = {}
    counter = {'i': 0}

    def hook(_mod, _inp, out):
        if counter['i'] in want:
            kept[counter['i']] = out.detach().numpy().copy()
        counter['i'] += 1

    h = model.fc3.register_forward_hook(hook)
    _RaceCategorical.q = torch.as_tensor(q)
    _RaceCategorical.step = 0
    _RaceCategorical.labels = []
    orig = torch.distributions.Categorical
    torch.distributions.Categorical = _RaceCategorical
    try:
        hp = fv._hp
        wave = model.generate(torch.as_tensor(mels), '/dev/null', bool(batched), target if target is not None else hp.voc_target,
                              overlap if overlap is not None else hp.voc_overlap, hp.mu_law if mu_law is None else mu_law)
    finally:
        torch.distributions.Categorical = orig
        h.remove()
    labels = torch.stack(_RaceCategorical.labels, 1).numpy().astype(np.int16)
    return dict(wave0=wave, labels=labels, logits=kept)


def reference_upsample(model, mels):
    """pad_tensor + UpsampleNetwork.forward exactly as generate() calls them (fatchord_version.py:185-186)."""
    model.eval()
    with torch.no_grad():
        m = torch.as_tensor(mels)
        mp = model.pad_tensor(m.transpose(1, 2), pad=model.pad, side='both')
        up, aux = model.upsample(mp.transpose(1, 2))
    return up.numpy(), aux.numpy()


def reference_forward_logits(model, x, mels_padded):
    """Teacher-forced `WaveRNN.forward` (fatchord_version.py:131-167); restores the `step` side effect (:139)."""
    model.eval()
    step = model.step.clone()
    with torch.no_grad():
        out = model(torch.as_tensor(x), torch.as_tensor(mels_padded)).numpy()
    model.step.copy_(step)
    return out


def memoize_upsample(model):
    """bench.py's repeated bounded samples call `generate` on the SAME mel batch; the reference's conditioning network
    (UpsampleNetwork.forward, fatchord_version.py:82-89, ~20 s for 256 x 21 frames on 8 cores) is outside the timed loop, so
    its output -- computed by the reference's own module on first use -- is kept and handed back on later calls with an
    identical input.  The timed sampling loop is untouched."""
    up = model.upsample
    if getattr(up, '_b200_memo', None) is not None:
        return
    orig = up.forward
    memo = {}

    def forward(m):
        key = (tuple(m.shape), float(m.double().sum()), float(m.double().abs().max()))
        if key not in memo:
            memo.clear()
            memo[key] = orig(m)
        return memo[key]

    up.forward = forward
    up._b200_memo = memo


class _StopSample(Exception):
    """Raised by the step-counting hook of `timed_generate_sample` to leave the reference's loop after the sample."""


def timed_generate_sample(model, mels, max_seconds=None, max_steps=None):
    """Times the reference's OWN `WaveRNN.generate` loop (fatchord_version.py:201-241) on `mels` [B, 80, T] without
    touching its code: a forward-pre-hook on `model.I` (first op of a loop step, :208) starts the clock at step 0, a
    forward hook on `model.fc3` (last layer of a step, :223) counts completed steps and, once `max_steps` steps or
    `max_seconds` have passed, raises to leave the loop (a bounded sample; `None` for both = the whole utterance).
    The one-shot conditioning network (:186) runs before the clock starts and is reported separately.
    Returns dict(steps, loop_seconds, upsample_seconds, batch)."""
    import time
    fv = import_reference()
    hp = fv._hp
    st = {'t0': None, 'n': 0, 't_end': None, 't_call': None}

    def pre(_m, _inp):
        if st['t0'] is None:
            st['t0'] = time.perf_counter()

    def post(_m, _inp, _out):
        st['n'] += 1
        if (max_steps is not None and st['n'] >= max_steps) or \
                (max_seconds is not None and st['n'] % 8 == 0 and time.perf_counter() - st['t0'] >= max_seconds):
            st['t_end'] = time.perf_counter()
            raise _StopSample()

    h1 = model.I.register_forward_pre_hook(pre)
    h2 = model.fc3.register_forward_hook(post)
    st['t_call'] = time.perf_counter()
    try:
        model.generate(torch.as_tensor(mels), '/dev/null', False, hp.voc_target, hp.voc_overlap, hp.mu_law)
        st['t_end'] = time.perf_counter()          # ran to the end: includes the (negligible) numpy epilogue
    except _StopSample:
        pass
    finally:
        h1.remove()
        h2.remove()
        model.train()
    return dict(steps=st['n'], loop_seconds=st['t_end'] - st['t0'], upsample_seconds=st['t0'] - st['t_call'],
                batch=int(mels.shape[0]))
