"""CPU oracle for WaveRNN generation in mixture-of-logistics mode (voc_mode = 'MOL') -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A numpy (float32) restatement of the reference's MOL branch: `sample_from_discretized_mix_logistic`
(wavernn/utils/distribution.py:87-123) called from WaveRNN.generate (wavernn/models/fatchord_version.py:225-229), with the
float sample fed back as the next input and no mu-law (:174).  The network up to fc3 is the RAW oracle's
(oracle/wavernn_oracle.py); only fc3's width (30) and the sampler differ.

Parity pin: tests/golden/wavernn_mol_*.npz were produced by running the reference itself in MOL mode
(oracle/make_golden_wavernn_mol.py) and tests/test_wavernn_mol_cpu.py checks this restatement against them.
"""
from __future__ import annotations

import numpy as np

from oracle import wavernn_oracle as wo

F32 = np.float32
NR_MIX = 10
LOG_SCALE_MIN = F32(np.log(1e-14))        # the reference's float(np.log(1e-14)), as torch.clamp rounds it to fp32


def mixture_index(p, u):
    """k = argmax_j (p[j] - log(-log(u[j]))), first maximum (torch .max), distribution.py:105-108.  p [B, 30], u [B, >=10]."""
    p = np.asarray(p, dtype=F32)
    u = np.asarray(u, dtype=F32)
    g = (p[:, :NR_MIX] - np.log(-np.log(u[:, :NR_MIX]))).astype(F32)
    return np.argmax(g, axis=1)


def sample_mol(p, u):
    """sample_from_discretized_mix_logistic for a batch of rows: p [B, 30] fc3 outputs, u [B, 11] uniforms (u[:, :10] choose
    the mixture, u[:, 10] drives the logistic).  Returns (x [B] float32 in [-1, 1], k [B])."""
    p = np.asarray(p, dtype=F32)
    u = np.asarray(u, dtype=F32)
    k = mixture_index(p, u)
    rows = np.arange(p.shape[0])
    means = p[rows, NR_MIX + k]
    log_scales = np.maximum(p[rows, 2 * NR_MIX + k], LOG_SCALE_MIN)                      # :116
    v = u[:, NR_MIX]
    x = (means + np.exp(log_scales).astype(F32) * (np.log(v) - np.log(F32(1.0) - v)).astype(F32)).astype(F32)   # :118
    return np.clip(x, F32(-1.0), F32(1.0)).astype(F32), k                                 # :120


def sample_bar(p, u, k, logit_err):
    """How far a sample may move when every fc3 output moves by up to `logit_err` and log / exp are each off by one ulp:
    the sampler formula differentiated, |d mean| + |exp(ls)| * (|d ls| * |l| + ulp terms).  p [B,30], u [B,11], k [B]."""
    p = np.asarray(p, dtype=np.float64)
    rows = np.arange(p.shape[0])
    ls = np.maximum(p[rows, 2 * NR_MIX + k], float(LOG_SCALE_MIN))
    v = np.asarray(u, dtype=np.float64)[:, NR_MIX]
    l = np.log(v) - np.log(1.0 - v)
    e = np.exp(ls)
    eps = float(np.finfo(F32).eps)
    return logit_err + e * (logit_err * np.abs(l) + 4 * eps * (np.abs(l) + np.abs(np.log(v)) + np.abs(np.log(1.0 - v)))) + \
        4 * eps * (np.abs(p[rows, NR_MIX + k]) + e * np.abs(l) + 1.0)


def _loop(pf, m_up, aux, u, teacher, keep, steps):
    d = wo._dims(pf)
    B = m_up.shape[0]
    A = d['aux']
    h1 = np.zeros((B, d['rnn']), dtype=F32)
    h2 = np.zeros((B, d['rnn']), dtype=F32)
    x = np.zeros((B, 1), dtype=F32)
    samples = np.zeros((B, steps), dtype=F32)
    mix = np.zeros((B, steps), dtype=np.int16)
    kept = {}
    for i in range(steps):
        a = aux[:, i, :]
        p, h1, h2 = wo.step_logits(pf, x, m_up[:, i, :], a[:, :A], a[:, A:2 * A], a[:, 2 * A:3 * A], a[:, 3 * A:4 * A], h1, h2)
        if keep is not None and i in keep:
            kept[i] = p.copy()
        s, k = sample_mol(p, u[i])
        samples[:, i] = s
        mix[:, i] = k
        x = (np.asarray(teacher[:, i], dtype=F32) if teacher is not None else s)[:, None]   # :229
    return samples, mix, kept


def generate(p, mels, u, teacher=None, keep_logits=None, max_steps=None):
    """WaveRNN.generate in MOL mode for a batch of independent utterances.  mels [B, feat, T]; u [S, B, 11];
    teacher optional float [B, S] fed back instead of the samples; keep_logits None | 'all' | steps.
    Returns dict(samples float32 [B, S], mix int16 [B, S], wave float64 [B, wave_len] or None, logits {step: [B, 30]})."""
    d = wo._dims(p)
    pf = {k: (v.astype(F32) if v.dtype.kind == 'f' else v) for k, v in p.items()}
    mels = np.asarray(mels, dtype=F32)
    T = mels.shape[2]
    mp = wo.pad_tensor(mels.transpose(0, 2, 1), d['pad'], 'both').transpose(0, 2, 1)
    m_up, aux = wo.upsample(pf, mp)
    S_all = m_up.shape[1]
    S = S_all if max_steps is None else min(max_steps, S_all)
    keep = None if keep_logits is None else (set(range(S)) if keep_logits == 'all' else set(keep_logits))
    samples, mix, kept = _loop(pf, m_up, aux, u, teacher, keep, S)
    wave = finish_wave(samples, (T - 1) * d['hop'], d['hop']) if S == S_all else None
    return dict(samples=samples, mix=mix, wave=wave, logits=kept)


def generate_batched(p, mel, target, overlap, u, teacher=None, keep_logits=None):
    """generate(batched=True) in MOL mode: ONE utterance mel [1, feat, T] folded with overlap; u [L, num_folds, 11].
    Returns dict(samples [num_folds, L], mix, wave [wave_len] float64, logits)."""
    d = wo._dims(p)
    pf = {k: (v.astype(F32) if v.dtype.kind == 'f' else v) for k, v in p.items()}
    mel = np.asarray(mel, dtype=F32)
    T = mel.shape[2]
    mp = wo.pad_tensor(mel.transpose(0, 2, 1), d['pad'], 'both').transpose(0, 2, 1)
    m_up, aux = wo.upsample(pf, mp)
    m_up = wo.fold_with_overlap(m_up, target, overlap)
    aux = wo.fold_with_overlap(aux, target, overlap)
    L = m_up.shape[1]
    keep = None if keep_logits is None else (set(range(L)) if keep_logits == 'all' else set(keep_logits))
    samples, mix, kept = _loop(pf, m_up, aux, u, teacher, keep, L)
    return dict(samples=samples, mix=mix, wave=unfold_wave(samples, target, overlap, (T - 1) * d['hop'], d['hop']), logits=kept)


def finish_wave(samples, wave_len, hop):
    """generate() epilogue for MOL samples (fatchord_version.py:243-258, mu_law off): float64, truncate, 20-hop fade-out."""
    out = np.asarray(samples, dtype=F32).astype(np.float64)[:, :wave_len].copy()
    out[:, -20 * hop:] *= np.linspace(1, 0, 20 * hop)
    return out


def unfold_wave(samples, target, overlap, wave_len, hop):
    """xfade_and_unfold of the folds' samples (fatchord_version.py:250-251), then the same truncation and fade-out."""
    out = wo.xfade_and_unfold(np.asarray(samples, dtype=F32).astype(np.float64), target, overlap)[:wave_len].copy()
    out[-20 * hop:] *= np.linspace(1, 0, 20 * hop)
    return out
