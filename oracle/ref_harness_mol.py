"""Drive the UNMODIFIED reference WaveRNN in MOL mode (voc_mode = 'MOL') -- build-container test tooling.

The reference is imported through oracle/ref_harness.py.  Its MOL sampler (wavernn/utils/distribution.py:87-123) draws
its noise with two `Tensor.uniform_` calls per step, [1, B, 10] for the mixture and [1, B] for the logistic; for the
duration of a run `torch.Tensor.uniform_` is replaced by a feeder that checks each requested shape and hands out the
injected uniforms instead, so the reference, the oracle and the CUDA kernels share the noise.  A forward hook on fc3
captures the mixture parameters.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import ref_harness as rh


def build_model_mol(state_dict, dims=None):
    """Reference WaveRNN(mode='MOL') with the shipped hparams, or with `dims` (keys of synth.DEFAULT_DIMS), loaded from a
    numpy/torch state_dict."""
    return rh.build_model(state_dict, dims, 'MOL')


class _UniformFeeder:
    """Stand-in for Tensor.uniform_: per step, the first call must ask for [1, B, 10] and gets u[i, :, :10], the second
    [1, B] and gets u[i, :, 10]."""

    def __init__(self, u):
        self.u = torch.as_tensor(np.asarray(u, dtype=np.float32))
        self.calls = 0

    def __call__(self, t, a=0.0, b=1.0):
        step, second = divmod(self.calls, 2)
        B = self.u.shape[1]
        want = (1, B) if second else (1, B, 10)
        assert tuple(t.shape) == want, f'uniform_ call {self.calls}: shape {tuple(t.shape)}, expected {want}'
        src = self.u[step, :, 10] if second else self.u[step, :, :10]
        t.copy_(src.reshape(want))
        self.calls += 1
        return t


def reference_generate_mol(model, mels, u, capture_logits_at=(), batched=False, target=None, overlap=None):
    """Runs the reference `generate` (fatchord_version.py:169) in MOL mode with injected uniforms u [S, B, 11].

    Returns dict(wave0 float64 [wave_len], samples float32 [B, S] (the inputs fed back), logits {step: [B, 30]},
    uniform_calls)."""
    fv = rh.import_reference()
    want = set(int(s) for s in capture_logits_at)
    kept, samples = {}, []
    counter = {'i': 0}

    def hook(_mod, _inp, out):
        if counter['i'] in want:
            kept[counter['i']] = out.detach().numpy().copy()
        counter['i'] += 1

    def i_hook(_mod, inp):
        samples.append(inp[0][:, 0].detach().numpy().copy())       # x of the step = the previous step's sample

    feeder = _UniformFeeder(u)
    h = model.fc3.register_forward_hook(hook)
    hi = model.I.register_forward_pre_hook(i_hook)
    orig = torch.Tensor.uniform_
    # generate() first builds two GRUCells (fatchord_version.py:178-179) whose initialisation also calls uniform_: only the
    # sampler's calls, on (1e-5, 1 - 1e-5), are fed
    torch.Tensor.uniform_ = lambda t, a=0.0, b=1.0, **kw: feeder(t, a, b) if (a, b) == (1e-5, 1.0 - 1e-5) else orig(t, a, b, **kw)
    try:
        hp = fv._hp
        wave = model.generate(torch.as_tensor(mels), '/dev/null', bool(batched), target if target is not None else hp.voc_target,
                              overlap if overlap is not None else hp.voc_overlap, hp.mu_law)
    finally:
        torch.Tensor.uniform_ = orig
        h.remove()
        hi.remove()
    S = counter['i']
    assert feeder.calls == 2 * S, (feeder.calls, S)
    # the sample of step i is the input of step i + 1, so this holds the samples of steps 0 .. S-2; the last sample is never
    # fed back and is not captured (it lies beyond the wave, which ends at (T - 1) * hop)
    x = np.stack(samples[1:], 1) if S > 1 else np.zeros((len(samples[0]), 0), np.float32)
    return dict(wave0=wave, inputs=x, logits=kept, uniform_calls=feeder.calls, steps=S)
