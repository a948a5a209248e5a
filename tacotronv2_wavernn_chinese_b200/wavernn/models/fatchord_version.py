"""`WaveRNN` / `UpsampleNetwork` with the reference's Python surface, computed on the GPU.

Mirrors lturing/tacotronv2_wavernn_chinese `wavernn/models/fatchord_version.py`:
constructor arguments (:93-95), `load` (:414), `save` (:419), `get_step` (:407),
`generate(mels, save_path, batched, target, overlap, mu_law)` (:169) and the state_dict key
names, so the shipped `logs_wavernn/checkpoints/latest_weights.pyt` loads unchanged.

The torch modules below only HOLD parameters (so `load_state_dict` / `.to()` behave as usual);
none of them is ever called.  Every arithmetic step -- conditioning network, per-sample GRU/FC
recurrence, sampling, mu-law decode, fade-out -- runs in csrc/*.cu through the C ABI
(include/b200tts.h) via `WaveRNNEngine`.  There is no CPU fallback: without a CUDA device
`generate` raises.
"""
from __future__ import annotations

import os
import time
from pathlib import Path
from typing import Union

import numpy as np
import torch
import torch.nn as nn

from ...engine import WaveRNNEngine
from ..utils.display import progbar, stream
from ..utils.dsp import save_wav


class _ResBlockParams(nn.Module):
    def __init__(self, dims):
        super().__init__()
        self.conv1 = nn.Conv1d(dims, dims, kernel_size=1, bias=False)
        self.conv2 = nn.Conv1d(dims, dims, kernel_size=1, bias=False)
        self.batch_norm1 = nn.BatchNorm1d(dims)
        self.batch_norm2 = nn.BatchNorm1d(dims)


class MelResNet(nn.Module):
    """Parameter holder for the reference MelResNet (:31-48); evaluated by `melresnet_kernel`."""

    def __init__(self, res_blocks, in_dims, compute_dims, res_out_dims, pad):
        super().__init__()
        self.conv_in = nn.Conv1d(in_dims, compute_dims, kernel_size=2 * pad + 1, bias=False)
        self.batch_norm = nn.BatchNorm1d(compute_dims)
        self.layers = nn.ModuleList(_ResBlockParams(compute_dims) for _ in range(res_blocks))
        self.conv_out = nn.Conv1d(compute_dims, res_out_dims, kernel_size=1)


class UpsampleNetwork(nn.Module):
    """Reference :64-89.  `forward(m)` takes the PADDED mel [B, feat, T + 2*pad] like the reference and returns
    (mels [B, T*hop, feat], aux [B, T*hop, res_out]) computed on the GPU."""

    def __init__(self, feat_dims, upsample_scales, compute_dims, res_blocks, res_out_dims, pad):
        super().__init__()
        self.pad = pad
        self.total_scale = int(np.prod(upsample_scales))
        self.indent = pad * self.total_scale
        self.resnet = MelResNet(res_blocks, feat_dims, compute_dims, res_out_dims, pad)
        layers = []
        for scale in upsample_scales:     # odd indices carry the trained 1 x (2s+1) kernels (keys up_layers.{1,3,5})
            conv = nn.Conv2d(1, 1, kernel_size=(1, 2 * scale + 1), padding=(0, scale), bias=False)
            conv.weight.data.fill_(1. / (2 * scale + 1))
            layers += [nn.Identity(), conv]
        self.up_layers = nn.ModuleList(layers)
        self._owner = None

    def forward(self, m):
        if self._owner is None:
            raise RuntimeError('UpsampleNetwork must belong to a WaveRNN to run')
        owner = self._owner()
        p = self.pad
        m = torch.as_tensor(m)
        if p:
            edge = torch.cat([m[:, :, :p], m[:, :, -p:]], dim=2)
            if float(edge.abs().max()) != 0.0:
                raise ValueError('the GPU conditioning network assumes generate()-style zero padding '
                                 '(fatchord_version.py:185); got non-zero pad frames')
            m = m[:, :, p:-p]
        return owner._engine_for_current_weights().upsample(m, full_aux=True)


class WaveRNN(nn.Module):
    def __init__(self, rnn_dims, fc_dims, bits, pad, upsample_factors,
                 feat_dims, compute_dims, res_out_dims, res_blocks,
                 hop_length, sample_rate, mode='RAW'):
        super().__init__()
        self.mode = mode
        self.pad = pad
        if mode == 'RAW':
            self.n_classes = 2 ** bits
        elif mode == 'MOL':
            self.n_classes = 30
        else:
            raise RuntimeError(f'Unknown model mode value - {mode}')
        self.rnn_dims = rnn_dims
        self.aux_dims = res_out_dims // 4
        self.hop_length = hop_length
        self.sample_rate = sample_rate
        self._dims = dict(rnn_dims=rnn_dims, fc_dims=fc_dims, bits=bits, pad=pad,
                          upsample_factors=tuple(upsample_factors), feat_dims=feat_dims, compute_dims=compute_dims,
                          res_out_dims=res_out_dims, res_blocks=res_blocks, hop_length=hop_length, mode=mode)

        self.upsample = UpsampleNetwork(feat_dims, upsample_factors, compute_dims, res_blocks, res_out_dims, pad)
        self.I = nn.Linear(feat_dims + self.aux_dims + 1, rnn_dims)
        self.rnn1 = nn.GRU(rnn_dims, rnn_dims, batch_first=True)
        self.rnn2 = nn.GRU(rnn_dims + self.aux_dims, rnn_dims, batch_first=True)
        self.fc1 = nn.Linear(rnn_dims + self.aux_dims, fc_dims)
        self.fc2 = nn.Linear(fc_dims + self.aux_dims, fc_dims)
        self.fc3 = nn.Linear(fc_dims, self.n_classes)
        self.register_buffer('step', torch.zeros(1, dtype=torch.long))

        import weakref
        self.upsample._owner = weakref.ref(self)
        self._engine = None
        self._engine_key = None
        self._gen_calls = 0
        self.last_gen_seconds = None
        self.num_params()

    # ---------------------------------------------------------------------------------------------
    def _weights_key(self):
        return tuple((p.data_ptr(), p._version) for p in list(self.parameters()) + list(self.buffers()))

    def _engine_for_current_weights(self, device=None) -> WaveRNNEngine:
        """(Re)packs the weights into a libb200tts context when they changed since the last call."""
        p = next(self.parameters())
        dev = device if device is not None else (p.device.index if p.is_cuda else torch.cuda.current_device()
                                                 if torch.cuda.is_available() else None)
        if dev is None:
            raise RuntimeError('no CUDA device: the WaveRNN path has no CPU fallback')
        key = (dev, self._weights_key())
        if self._engine is None or self._engine_key != key:
            if self._engine is not None:
                self._engine.close()
            self._engine = WaveRNNEngine(self.state_dict(), self._dims, device=dev)
            self._engine_key = key
        return self._engine

    def forward(self, x, mels):
        raise NotImplementedError('WaveRNN.forward is the teacher-forced TRAINING path (fatchord_version.py:131-167), '
                                  'out of scope for the CUDA generation build; use generate()')

    def generate(self, mels, save_path: Union[str, Path, None], batched, target, overlap, mu_law,
                 seed=None, kernel='auto', return_all=False):
        """Drop-in for reference `generate` (:169-264).

        mels [B, feat, T] (tensor / ndarray, any device).  Returns float64 [wave_len] for B == 1 like the
        reference; for B > 1 the reference silently returns only row 0 (:253) -- this returns row 0 too unless
        `return_all=True`, which gives [B, wave_len].  `seed` fixes the Philox sampling stream (default: derived
        from torch.initial_seed() and a per-model call counter, so torch.manual_seed(k) reproduces a run).
        """
        self.eval()
        start = time.time()
        mu_law = mu_law if self.mode == 'RAW' else False
        eng = self._engine_for_current_weights()
        m = torch.as_tensor(mels)
        if m.dim() != 3:
            raise ValueError(f'mels must be [B, n_mels, T], got {tuple(m.shape)}')
        T = m.shape[-1]
        if (T - 1) * self.hop_length < 20 * self.hop_length:
            raise ValueError('mels need at least 21 frames: generate() fades out over 20 hops (fatchord_version.py:256-258)')
        if seed is None:
            seed = (int(torch.initial_seed()) * 1000003 + self._gen_calls) & 0xFFFFFFFFFFFFFFFF
        self._gen_calls += 1
        if batched and m.shape[0] != 1:
            raise ValueError('batched (fold-with-overlap) generation folds ONE utterance (fatchord_version.py:293-340)')
        out = eng.generate(m, seed=seed, mu_law=bool(mu_law), kernel=kernel, fold=(target, overlap) if batched else None)
        wave = out['wave'].cpu().numpy()                       # [B, wave_len] float64 (synchronises)
        eng.check()                                            # a timed-out persistent kernel must not yield audio
        if self.mode == 'MOL':
            self.last_samples = out['samples']
        else:
            self.last_labels = out['labels']
        self.last_gen_seconds = time.time() - start
        b_size, seq_len = m.shape[0], T * self.hop_length
        self.gen_display(seq_len - 1, seq_len, b_size, start)
        result = wave if return_all else wave[0]
        if save_path is not None and str(save_path) not in ('', os.devnull):
            save_wav(wave[0], save_path, self.sample_rate)
        self.train()
        return result

    def gen_display(self, i, seq_len, b_size, start):
        gen_rate = (i + 1) / max(time.time() - start, 1e-9) * b_size / 1000
        stream(f'| {progbar(i, seq_len)} {(i + 1) * b_size}/{seq_len * b_size} | Batch Size: {b_size} | '
               f'Gen Rate: {gen_rate:.1f}kHz | ')

    def get_step(self):
        return self.step.data.item()

    def log(self, path, msg):
        with open(path, 'a') as f:
            print(msg, file=f)

    def load(self, path: Union[str, Path]):
        device = next(self.parameters()).device
        # a checkpoint is a plain state_dict of tensors (reference :411 saves self.state_dict()): never unpickle arbitrary objects
        self.load_state_dict(torch.load(path, map_location=device, weights_only=True), strict=False)
        self._engine_key = None      # force a repack on next use

    def save(self, path: Union[str, Path]):
        torch.save(self.state_dict(), path)

    def num_params(self, print_out=True):
        n = sum(int(np.prod(p.size())) for p in self.parameters() if p.requires_grad) / 1_000_000
        if print_out:
            print('Trainable Parameters: %.3fM' % n)
        return n
