"""Portable synthetic WaveRNN weights, mels and sampling noise.

The shipped checkpoint (`logs_wavernn/checkpoints/latest_weights.pyt`, reference
wavernn/utils/paths.py:12-13) lives under /root/reference and does not exist on the
GPU box, so the bench, `smoke()` and the portable golden fixtures use weights
generated here.  Everything is drawn from numpy's *legacy* `RandomState`
(bit-stable across numpy versions), so the container that generated
`tests/golden/*` and the GPU box that replays them build identical tensors.

Key names/shapes follow the reference state_dict (wavernn/models/fatchord_version.py:93-126;
SURVEY.md section 2 row 4).
"""
from __future__ import annotations

import numpy as np

# hparams of the shipped model (reference wavernn_hparams.py:18-41,50)
DEFAULT_DIMS = dict(rnn_dims=512, fc_dims=512, bits=10, pad=2, upsample_factors=(5, 5, 11),
                    feat_dims=80, compute_dims=128, res_out_dims=128, res_blocks=10,
                    hop_length=275, sample_rate=22050)


def _uniform(rs, shape, bound):
    return rs.uniform(-bound, bound, size=shape).astype(np.float32)


def synth_state_dict(seed: int = 0, dims: dict | None = None, logit_gain: float = 60.0, mode: str = 'RAW',
                     mol_clamp: bool = False) -> dict:
    """Deterministic numpy state_dict with the reference's key names.

    `logit_gain` scales fc3 so the softmax is peaky like the trained model's
    (trained |logit| reaches ~450, SURVEY.md section 4); gain 1 is torch-default init.
    mode='MOL' gives the mixture-of-logistics head (voc_mode = 'MOL'): fc3 has 30 rows (10 mixture logits, 10 means,
    10 log-scales) and its log-scale biases sit near -5, so that samples stay mostly inside [-1, 1].  `mol_clamp` moves
    half the means beyond +-1 and half the log-scales below the sampler's floor log(1e-14), so both clamps fire often.
    Every other tensor is the same as in RAW mode with the same seed.
    """
    d = dict(DEFAULT_DIMS)
    if dims:
        d.update(dims)
    rs = np.random.RandomState(seed)
    R, F, C, O = d['rnn_dims'], d['fc_dims'], d['compute_dims'], d['res_out_dims']
    feat, aux = d['feat_dims'], d['res_out_dims'] // 4
    ncls = 2 ** d['bits']
    k = 2 * d['pad'] + 1
    sd = {}
    sd['step'] = np.array([seed], dtype=np.int64)
    sd['upsample.resnet.conv_in.weight'] = _uniform(rs, (C, feat, k), 1.0 / np.sqrt(feat * k))

    def bn(prefix):
        sd[prefix + '.weight'] = rs.uniform(0.8, 1.2, C).astype(np.float32)
        sd[prefix + '.bias'] = rs.uniform(-0.1, 0.1, C).astype(np.float32)
        sd[prefix + '.running_mean'] = rs.uniform(-0.5, 0.5, C).astype(np.float32)
        sd[prefix + '.running_var'] = rs.uniform(0.5, 2.0, C).astype(np.float32)
        sd[prefix + '.num_batches_tracked'] = np.array(1, dtype=np.int64)

    bn('upsample.resnet.batch_norm')
    for i in range(d['res_blocks']):
        p = f'upsample.resnet.layers.{i}'
        sd[p + '.conv1.weight'] = _uniform(rs, (C, C, 1), 1.0 / np.sqrt(C))
        sd[p + '.conv2.weight'] = _uniform(rs, (C, C, 1), 1.0 / np.sqrt(C))
        bn(p + '.batch_norm1')
        bn(p + '.batch_norm2')
    sd['upsample.resnet.conv_out.weight'] = _uniform(rs, (O, C, 1), 1.0 / np.sqrt(C))
    sd['upsample.resnet.conv_out.bias'] = _uniform(rs, (O,), 1.0 / np.sqrt(C))
    for j, s in enumerate(d['upsample_factors']):
        w = 1.0 / (2 * s + 1)
        sd[f'upsample.up_layers.{2 * j + 1}.weight'] = (
            w * rs.uniform(0.5, 1.5, (1, 1, 1, 2 * s + 1))).astype(np.float32)
    nin = feat + aux + 1
    sd['I.weight'] = _uniform(rs, (R, nin), 1.0 / np.sqrt(nin))
    sd['I.bias'] = _uniform(rs, (R,), 1.0 / np.sqrt(nin))
    for name, nx in (('rnn1', R), ('rnn2', R + aux)):
        b = 1.0 / np.sqrt(R)
        sd[f'{name}.weight_ih_l0'] = _uniform(rs, (3 * R, nx), b)
        sd[f'{name}.weight_hh_l0'] = _uniform(rs, (3 * R, R), b)
        sd[f'{name}.bias_ih_l0'] = _uniform(rs, (3 * R,), b)
        sd[f'{name}.bias_hh_l0'] = _uniform(rs, (3 * R,), b)
    sd['fc1.weight'] = _uniform(rs, (F, R + aux), 1.0 / np.sqrt(R + aux))
    sd['fc1.bias'] = _uniform(rs, (F,), 1.0 / np.sqrt(R + aux))
    sd['fc2.weight'] = _uniform(rs, (F, F + aux), 1.0 / np.sqrt(F + aux))
    sd['fc2.bias'] = _uniform(rs, (F,), 1.0 / np.sqrt(F + aux))
    if mode == 'MOL':
        w = _uniform(rs, (30, F), 1.0 / np.sqrt(F))
        w[:10] *= 4.0                                             # mixture logits: a few units apart
        w[10:20] *= 0.5                                           # means
        b = np.concatenate([_uniform(rs, (10,), 1.0), _uniform(rs, (10,), 0.5), -5.0 + _uniform(rs, (10,), 1.0)])
        if mol_clamp:
            b[10:20:2] += np.float32(1.5) * np.sign(b[10:20:2] + np.float32(1e-3))
            b[21:30:2] = np.float32(-40.0)
        sd['fc3.weight'] = w.astype(np.float32)
        sd['fc3.bias'] = b.astype(np.float32)
        return sd
    if mode != 'RAW':
        raise ValueError(f"unknown voc_mode {mode!r}")
    sd['fc3.weight'] = (logit_gain * _uniform(rs, (ncls, F), 1.0 / np.sqrt(F))).astype(np.float32)
    sd['fc3.bias'] = _uniform(rs, (ncls,), 1.0 / np.sqrt(F))
    return sd


def synth_mol_uniform(seed: int, steps: int, batch: int) -> np.ndarray:
    """The 11 uniforms of every step, u[S, B, 11] in [1e-5, 1 - 1e-5] (the range of the reference's uniform_ calls,
    wavernn/utils/distribution.py:106,117), for the EXT_UNIFORM mode of MOL generation."""
    rs = np.random.RandomState(seed)
    return rs.uniform(1e-5, 1.0 - 1e-5, size=(steps, batch, 11)).astype(np.float32)


def synth_mels(seed: int, batch: int, frames: int, feat_dims: int = 80) -> np.ndarray:
    """Uniform [0,1) float32 mels shaped [B, feat, T] (the layout `WaveRNN.generate` takes)."""
    rs = np.random.RandomState(seed)
    return rs.uniform(0.0, 1.0, size=(batch, feat_dims, frames)).astype(np.float32)


def synth_exponential_noise(seed: int, steps: int, batch: int, n_classes: int = 1024) -> np.ndarray:
    """Exp(1) race noise q[S, B, n_classes] (float32) for the external-noise sampling mode.

    The reference samples `argmax(p / q)`, q ~ Exp(1), inside torch.multinomial
    (reached from fatchord_version.py:233-235); tests feed the same q to the
    reference, the oracle and the CUDA kernels.
    """
    rs = np.random.RandomState(seed)
    q = rs.standard_exponential(size=(steps, batch, n_classes)).astype(np.float32)
    # an exact 0 would make p/q infinite for every class it hits; the reference never draws it
    np.maximum(q, np.float32(1e-30), out=q)
    return q
