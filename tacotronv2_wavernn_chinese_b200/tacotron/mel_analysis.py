"""MelAnalysisEngine: torch-facing wrapper of the mel-analysis context of libb200tts (one GPU), the engine behind
`audio.melspectrogram` and `audio.preprocess_wav` (tacotron/datasets/audio.py:95-102 and preprocessor.py:52-121 of the
reference)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from .. import _lib
from .._lib import MelCfg

TRIM, PREEMPHASIS, RESCALE = _lib.MEL_TRIM, _lib.MEL_PREEMPHASIS, _lib.MEL_RESCALE


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def preprocess_flags(hparams):
    """The steps `_process_utterance_v1` applies under these hparams (trim_silence, preemphasize, rescale)."""
    return ((TRIM if hparams.trim_silence else 0) | (PREEMPHASIS if hparams.preemphasize else 0)
            | (RESCALE if hparams.rescale else 0))


class MelAnalysisEngine:
    """hparams: the Tacotron hparams (tacotron_hparams.py) -- n_fft, hop_size, win_size, num_mels, sample_rate / fmin / fmax
    (for the filterbank), max_abs_value, the dB levels, magnitude_power, preemphasis, rescaling_max and the trim_* values."""

    def __init__(self, hparams, device: int | None = None):
        if not torch.cuda.is_available():
            raise RuntimeError('no CUDA device: mel analysis has no CPU fallback')
        from . import audio
        if not (hparams.signal_normalization and hparams.allow_clipping_in_normalization and hparams.symmetric_mels):
            raise ValueError('only symmetric, clipped mel normalisation is supported (the reference configuration)')
        self.lib = _lib.load()
        self.device = torch.cuda.current_device() if device is None else int(device)
        self.hp = hparams
        c = MelCfg(n_fft=hparams.n_fft, hop_size=hparams.hop_size, win_size=hparams.win_size, num_mels=hparams.num_mels,
                   max_abs_value=hparams.max_abs_value, min_level_db=hparams.min_level_db, ref_level_db=hparams.ref_level_db,
                   magnitude_power=hparams.magnitude_power, preemphasis=hparams.preemphasis,
                   rescaling_max=hparams.rescaling_max, trim_fft_size=hparams.trim_fft_size,
                   trim_hop_size=hparams.trim_hop_size, trim_top_db=hparams.trim_top_db)
        basis = np.ascontiguousarray(audio.mel_basis(hparams), dtype=np.float32)
        h = C.c_void_p()
        _lib.check(self.lib.b200tts_mel_create(C.byref(h), self.device, C.byref(c), basis.ctypes.data))
        self._h = h

    def close(self):
        if getattr(self, '_h', None):
            self.lib.b200tts_mel_destroy(self._h)
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
        return int(self.lib.b200tts_mel_launch_count(self._h))

    def run(self, wavs, lengths=None, flags=0, want_audio=False):
        """wavs [B, L_max] float32 signals (zero-padded), lengths: optional [B] sample counts (default L_max each), flags: a
        combination of TRIM, PREEMPHASIS and RESCALE (0 = plain melspectrogram).  Returns dict(mel [B, T_max, num_mels]
        (zero beyond each row's frames), frames [B] int32, bounds [B, 2] int32 = [start, end) of the kept samples,
        audio [B, T_max * hop] or None) as CUDA tensors, T_max = 1 + L_max // hop."""
        dev = self._dev()
        w = torch.as_tensor(wavs).to(device=dev, dtype=torch.float32).contiguous()
        if w.dim() != 2 or w.shape[1] < 1:
            raise ValueError('wavs must be [B, L] with L >= 1')
        B, L = w.shape
        ln = np.full(B, L, np.int32) if lengths is None else np.asarray(lengths, dtype=np.int64).reshape(-1)
        if ln.shape != (B,) or ln.min() < 1 or ln.max() > L:
            raise ValueError(f'lengths must be [B] with values in [1, {L}]')
        if flags & TRIM and ln.min() < self.hp.trim_fft_size:
            raise ValueError(f'trimming needs at least trim_fft_size = {self.hp.trim_fft_size} samples per signal, got '
                             f'{int(ln.min())}')
        lt = torch.as_tensor(ln.astype(np.int32)).to(dev)
        T = 1 + L // self.hp.hop_size
        with torch.cuda.device(self.device):
            mel = torch.empty(B, T, self.hp.num_mels, device=dev, dtype=torch.float32)
            frames = torch.empty(B, device=dev, dtype=torch.int32)
            bounds = torch.empty(B, 2, device=dev, dtype=torch.int32)
            audio = torch.empty(B, T * self.hp.hop_size, device=dev, dtype=torch.float32) if want_audio else None
            _lib.check(self.lib.b200tts_mel_analyze(self._h, _ptr(w), _ptr(lt), B, L, int(flags), _ptr(mel), _ptr(frames),
                                                    _ptr(bounds), _ptr(audio), self._stream()))
            for t in (w, lt):
                t.record_stream(torch.cuda.current_stream(self.device))
        return dict(mel=mel, frames=frames, bounds=bounds, audio=audio)
