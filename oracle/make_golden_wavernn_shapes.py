"""Generate tests/golden/wavernn_shapes_from_reference.npz by running the UNMODIFIED reference at model shapes other than the
shipped one.

Run where the reference checkout exists (it is not present on the GPU box):

    python oracle/make_golden_wavernn_shapes.py

Cases, on synthetic weights (tacotronv2_wavernn_chinese_b200.synth, legacy RandomState, so every input is regenerated from its
seed rather than stored).  Together they move every dimension the oracle reads from the weights' shapes:
  r256   R = F = 256, 9 bits, pad 1, factors (4, 4, 16), compute 64, res_out 64, 3 blocks
  r128   R = F = 128, 8 bits, feat 20, factors (1, 1, 2) (hop 2, 7 taps), no residual block, compute 100
  bits2  R = F = 512, 2 bits, factors (7,), res_out 16 (aux 4), pad 3
  mol384 MOL, R = F = 384, factors (5, 5, 8)

Each case stores, under keys `<case>__<name>`: its hparams (JSON) and seeds; the reference's labels (RAW) or fed-back samples
(MOL) under injected noise; its fc3 outputs at steps on both sides of the first two frame boundaries and at the last step; the
upsampled mels sub-sampled at a stride coprime with hop; the aux frames; and the wave it returned for utterance 0, with mu-law on
and off for RAW.
"""
from __future__ import annotations

import json
import math
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_harness as rh                                   # noqa: E402
from oracle import ref_harness_mol as rhm                              # noqa: E402
from tacotronv2_wavernn_chinese_b200 import synth                      # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden', 'wavernn_shapes_from_reference.npz')

# case -> (hparams over synth.DEFAULT_DIMS, frames, weight / mel / noise seeds)
CASES = {
    'r256': (dict(rnn_dims=256, fc_dims=256, bits=9, pad=1, upsample_factors=(4, 4, 16), compute_dims=64, res_out_dims=64,
                  res_blocks=3), 21, (31, 32, 33)),
    'r128': (dict(rnn_dims=128, fc_dims=128, bits=8, feat_dims=20, upsample_factors=(1, 1, 2), res_blocks=0, compute_dims=100),
             60, (41, 42, 43)),
    'bits2': (dict(bits=2, upsample_factors=(7,), res_out_dims=16, pad=3), 30, (51, 52, 53)),
    'mol384': (dict(mode='MOL', rnn_dims=384, fc_dims=384, upsample_factors=(5, 5, 8)), 21, (61, 62, 63)),
}
B = 2


def dims_of(over):
    d = dict(synth.DEFAULT_DIMS, **over)
    d['hop_length'] = int(np.prod(d['upsample_factors']))
    return d


def probe_steps(hop, S):
    """Steps on both sides of the first two frame boundaries, and the last step."""
    return sorted({s for s in (0, 1, hop - 1, hop, hop + 1, 2 * hop - 1, 2 * hop, 2 * hop + 1, S - 1) if 0 <= s < S})


def up_stride(hop, S, feat):
    """A stride coprime with hop that keeps about 12 000 floats of upsampled mels per utterance."""
    st = max(3, S * feat // 12000)
    while math.gcd(st, hop) != 1:
        st += 1
    return st


def make_case(name, over, T, seeds, out):
    d = dims_of(over)
    mol = d.get('mode') == 'MOL'
    hop, feat = d['hop_length'], d['feat_dims']
    S = T * hop
    wseed, mseed, nseed = seeds
    sd = synth.synth_state_dict(wseed, d, mode='MOL' if mol else 'RAW')
    mels = synth.synth_mels(mseed, B, T, feat)
    steps = probe_steps(hop, S)
    pre = name + '__'
    out[pre + 'dims'] = np.array(json.dumps(d))
    out[pre + 'seeds'] = np.array(seeds, dtype=np.int64)
    out[pre + 'B'], out[pre + 'T'] = B, T
    out[pre + 'logit_steps'] = np.array(steps, dtype=np.int64)
    if mol:
        model = rhm.build_model_mol(sd, d)
        u = synth.synth_mol_uniform(nseed, S, B)
        res = rhm.reference_generate_mol(model, mels, u, capture_logits_at=steps)
        out[pre + 'samples'] = res['inputs'].astype(np.float32)
        out[pre + 'wave0'] = res['wave0']
    else:
        model = rh.build_model(sd, d, 'RAW')
        q = synth.synth_exponential_noise(nseed, S, B, 1 << d['bits'])
        res = rh.reference_generate(model, mels, q, capture_logits_at=steps, mu_law=True)
        lin = rh.reference_generate(model, mels, q, mu_law=False)
        assert np.array_equal(res['labels'], lin['labels'])
        out[pre + 'labels'] = res['labels']
        out[pre + 'wave0_mu_law'] = res['wave0']
        out[pre + 'wave0_linear'] = lin['wave0']
    out[pre + 'logits'] = np.stack([res['logits'][s] for s in steps])
    up, aux = rh.reference_upsample(model, mels)
    st = up_stride(hop, S, feat)
    out[pre + 'up_stride'] = st
    out[pre + 'mels_up_sub'] = up[:, ::st].copy()
    out[pre + 'aux_frames'] = aux[:, ::hop].copy()
    assert np.array_equal(np.repeat(out[pre + 'aux_frames'], hop, axis=1), aux), 'aux not constant within a hop'
    print(f'  {name}: hop {hop}, {S} steps, |logit| <= {np.abs(out[pre + "logits"]).max():.1f}, up stride {st}')


def main():
    torch.set_num_threads(8)
    out = {}
    for name, (over, T, seeds) in CASES.items():
        make_case(name, over, T, seeds, out)
    np.savez_compressed(OUT, **out)
    print(f'{OUT}: {os.path.getsize(OUT) / 1e3:.0f} kB')


if __name__ == '__main__':
    main()
