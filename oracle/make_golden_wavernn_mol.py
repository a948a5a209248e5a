"""Generate tests/golden/wavernn_mol_*.npz by running the UNMODIFIED reference in MOL mode (voc_mode = 'MOL').

Run in the build container (the reference is not present on the GPU box):

    python oracle/make_golden_wavernn_mol.py

Cases, on synthetic MOL weights (tacotronv2_wavernn_chinese_b200.synth, mode='MOL', seed 21) -- fully portable
  wavernn_mol_synth_T24.npz          3 utterances x 24 frames, unbatched
  wavernn_mol_synth_batched_T30.npz  one 30-frame utterance, fold-with-overlap (target 2750, overlap 550)

Each file holds the seeds of the inputs and of the injected uniforms u [S, B, 11] (synth.synth_mol_uniform; legacy
RandomState, so they are regenerated bit for bit rather than stored), the reference's samples (the inputs it fed back,
steps 0 .. S-2), its fc3 outputs at probe steps and the wave it returned.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_harness_mol as rhm                              # noqa: E402
from tacotronv2_wavernn_chinese_b200 import synth                      # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden')
WEIGHT_SEED = 21


def make_case(model, mel_seed, u_seed, B, T, probe):
    mels = synth.synth_mels(mel_seed, B, T)
    u = synth.synth_mol_uniform(u_seed, T * 275, B)
    res = rhm.reference_generate_mol(model, mels, u, capture_logits_at=probe)
    path = os.path.join(OUT, f'wavernn_mol_synth_T{T}.npz')
    np.savez_compressed(path, weight_seed=WEIGHT_SEED, mel_seed=mel_seed, u_seed=u_seed, B=B, T=T,
                        samples=res['inputs'].astype(np.float32), wave0=res['wave0'], probe=np.array(probe, dtype=np.int64),
                        logits=np.stack([res['logits'][s] for s in probe]))
    print(f'  {path}: samples {res["inputs"].shape} -> {os.path.getsize(path) / 1e3:.0f} kB')


def make_batched_case(model, mel_seed, u_seed, T, target, overlap, probe):
    mels = synth.synth_mels(mel_seed, 1, T)
    S = T * 275
    nf = (S - overlap) // (target + overlap)
    if S - (nf * (target + overlap) + overlap) != 0:
        nf += 1
    L = target + 2 * overlap
    u = synth.synth_mol_uniform(u_seed, L, nf)
    res = rhm.reference_generate_mol(model, mels, u, capture_logits_at=probe, batched=True, target=target, overlap=overlap)
    assert res['inputs'].shape == (nf, L - 1), res['inputs'].shape
    path = os.path.join(OUT, f'wavernn_mol_synth_batched_T{T}.npz')
    np.savez_compressed(path, weight_seed=WEIGHT_SEED, mel_seed=mel_seed, u_seed=u_seed, T=T, target=target, overlap=overlap,
                        samples=res['inputs'].astype(np.float32), wave=res['wave0'],
                        probe=np.array(probe, dtype=np.int64), logits=np.stack([res['logits'][s] for s in probe]))
    print(f'  {path}: folds {nf} x {L} -> {os.path.getsize(path) / 1e3:.0f} kB')


def main():
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(8)
    model = rhm.build_model_mol(synth.synth_state_dict(WEIGHT_SEED, mode='MOL'))
    make_case(model, mel_seed=301, u_seed=302, B=3, T=24, probe=[0, 1, 2, 274, 275, 276, 3000, 6599])
    make_batched_case(model, mel_seed=303, u_seed=304, T=30, target=2750, overlap=550, probe=[0, 1, 549, 550, 3849])


if __name__ == '__main__':
    main()
