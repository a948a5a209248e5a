"""GriffinLimEngine: torch-facing wrapper of the Griffin-Lim context of libb200tts (one GPU), the engine behind
`audio.inv_mel_spectrogram` (tacotron/datasets/audio.py:122-137 of the reference)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from .. import _lib
from .._lib import GlCfg, GlPhase


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


class GriffinLimEngine:
    """hparams: the Tacotron hparams (tacotron_hparams.py) -- n_fft, hop_size, win_size, num_mels, max_abs_value, the dB levels,
    magnitude_power, power, preemphasize / preemphasis, sample_rate / fmin / fmax (for the filterbank pseudo-inverse)."""

    def __init__(self, hparams, device: int | None = None):
        if not torch.cuda.is_available():
            raise RuntimeError('no CUDA device: Griffin-Lim has no CPU fallback')
        from . import audio
        if not (hparams.signal_normalization and hparams.allow_clipping_in_normalization and hparams.symmetric_mels):
            raise ValueError('only symmetric, clipped mel normalisation is supported (the reference configuration)')
        self.lib = _lib.load()
        self.device = torch.cuda.current_device() if device is None else int(device)
        self.hp = hparams
        self.n_bins = hparams.n_fft // 2 + 1
        c = GlCfg(n_fft=hparams.n_fft, hop_size=hparams.hop_size, win_size=hparams.win_size, num_mels=hparams.num_mels,
                  max_abs_value=hparams.max_abs_value, min_level_db=hparams.min_level_db, ref_level_db=hparams.ref_level_db,
                  magnitude_power=hparams.magnitude_power, power=hparams.power,
                  preemphasis=hparams.preemphasis if hparams.preemphasize else 0.0)
        pinv = np.ascontiguousarray(audio.inv_mel_basis(hparams), dtype=np.float32)
        h = C.c_void_p()
        _lib.check(self.lib.b200tts_gl_create(C.byref(h), self.device, C.byref(c), pinv.ctypes.data))
        self._h = h

    def close(self):
        if getattr(self, '_h', None):
            self.lib.b200tts_gl_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _dev(self):
        return torch.device('cuda', self.device)

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    @property
    def launch_count(self) -> int:
        return int(self.lib.b200tts_gl_launch_count(self._h))

    def run(self, mels, frames=None, *, seed=0, utterance_offset=0, u=None, n_iters=None, want_u=False):
        """mels [B, T_max, num_mels] (frames x mels, symmetric scale), frames: optional true frame counts [B] (each 2..T_max).
        Initial phase: u [B, T_max, n_fft/2 + 1] uniforms (EXT) if given, else Philox(seed) keyed by (utterance_offset + row,
        frame, bin).  Returns dict(wave [B, hop * (T_max - 1)] float32, zero beyond each row's hop * (frames - 1) samples,
        u = phase of the last stft [B, T_max, n_bins] or None) as CUDA tensors."""
        dev = self._dev()
        m = torch.as_tensor(mels).to(device=dev, dtype=torch.float32).contiguous()
        if m.dim() != 3 or m.shape[2] != self.hp.num_mels:
            raise ValueError(f'mels must be [B, T, {self.hp.num_mels}]')
        B, T, _ = m.shape
        if T < 2:
            raise ValueError('a mel needs at least 2 frames')
        n_iters = self.hp.griffin_lim_iters if n_iters is None else int(n_iters)
        fr = None
        if frames is not None:
            fh = np.asarray(frames, dtype=np.int32).reshape(-1)
            if fh.shape != (B,) or fh.min() < 2 or fh.max() > T:
                raise ValueError(f'frames must be [B] with values in [2, {T}]')
            fr = torch.as_tensor(fh).to(dev)
        with torch.cuda.device(self.device):
            wave = torch.empty(B, self.hp.hop_size * (T - 1), device=dev, dtype=torch.float32)
            u_out = torch.empty(B, T, self.n_bins, device=dev, dtype=torch.float32) if want_u else None
            ph = GlPhase(mode=_lib.GL_PHASE_PHILOX, seed=int(seed) & 0xFFFFFFFFFFFFFFFF, utterance_offset=int(utterance_offset))
            ut = None
            if u is not None:
                ut = torch.as_tensor(u).to(device=dev, dtype=torch.float32).contiguous()
                if tuple(ut.shape) != (B, T, self.n_bins):
                    raise ValueError(f'u must be [B, T, {self.n_bins}]')
                ph.mode, ph.d_u = _lib.GL_PHASE_EXT, ut.data_ptr()
            _lib.check(self.lib.b200tts_griffin_lim(self._h, _ptr(m), _ptr(fr), B, T, C.byref(ph), n_iters, _ptr(wave), _ptr(u_out),
                                                    self._stream()))
            for t in (m, fr, ut):
                if t is not None:
                    t.record_stream(torch.cuda.current_stream(self.device))
        return dict(wave=wave, u=u_out)

    def philox_uniform(self, seed, utterance_offset, B, T):
        """The uniforms the PHILOX phase mode draws: [B, T, n_fft/2 + 1]."""
        with torch.cuda.device(self.device):
            u = torch.empty(B, T, self.n_bins, device=self._dev(), dtype=torch.float32)
            _lib.check(self.lib.b200tts_gl_philox_uniform(self.device, int(seed) & 0xFFFFFFFFFFFFFFFF, int(utterance_offset), B, T,
                                                          self.n_bins, _ptr(u), self._stream()))
        return u
