"""TacoDecoderEngine: torch-facing wrapper of the Tacotron-2 decoder context of libb200tts (one GPU)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from .. import _lib
from .._lib import TacoCfg, TacoDropout

DEFAULT_CFG = dict(num_mels=80, prenet_units=256, lstm_units=256, enc_dim=512, attn_dim=128, attn_filters=32,
                   attn_kernel=31, zoneout=0.1)      # tacotron_hparams.py:99-215 of the reference


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


class TacoDecoderEngine:
    def __init__(self, weights: dict, cfg: dict | None = None, device: int | None = None):
        if not torch.cuda.is_available():
            raise RuntimeError('no CUDA device: the Tacotron decoder has no CPU fallback')
        self.lib = _lib.load()
        self.device = torch.cuda.current_device() if device is None else int(device)
        self.cfg = dict(DEFAULT_CFG)
        if cfg:
            self.cfg.update(cfg)
        host = {k: np.ascontiguousarray(v, dtype=np.float32) for k, v in weights.items()
                if np.asarray(v).dtype.kind == 'f'}
        arr, keep = _lib.make_tensor_array(host)
        c = TacoCfg()
        for k, v in self.cfg.items():
            setattr(c, k, v)
        h = C.c_void_p()
        _lib.check(self.lib.b200tts_taco_create(C.byref(h), self.device, C.byref(c), arr, len(arr)))
        del keep
        self._h = h

    def close(self):
        if getattr(self, '_h', None):
            self.lib.b200tts_taco_destroy(self._h)
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

    def decode(self, memory, lengths=None, *, masks=None, seed=0, utterance_offset=0, max_steps=2000, window=False,
               want_align=True, forced_states=None):
        """memory [B, Tx, enc_dim] (tensor/ndarray); lengths [B] or None (= Tx).  masks: optional uint8 keep flags
        [B, max_steps, 2, prenet_units] (EXT mode) else Philox(seed).  Returns dict(frames [B,max_steps,80], stop
        [B,max_steps], align [B,max_steps,Tx] or None, nsteps [B]) as CUDA tensors (rows beyond nsteps are undefined).
        forced_states: optional [B, max_steps, state_floats(Tx)] teacher-forcing records (see include/b200tts.h,
        b200tts_taco_decode_forced): the whole recurrent state is reloaded before every step and exactly max_steps steps run."""
        dev = self._dev()
        m = torch.as_tensor(memory).to(device=dev, dtype=torch.float32).contiguous()
        if m.dim() != 3 or m.shape[2] != self.cfg['enc_dim']:
            raise ValueError(f'memory must be [B, Tx, {self.cfg["enc_dim"]}]')
        B, Tx, _ = m.shape
        ln = torch.full((B,), Tx, dtype=torch.int32) if lengths is None else torch.as_tensor(lengths, dtype=torch.int32)
        if int(ln.max()) > Tx or int(ln.min()) < 1:
            raise ValueError('lengths must be in [1, Tx]')
        ln = ln.to(dev)
        with torch.cuda.device(self.device):
            frames = torch.zeros(B, max_steps, self.cfg['num_mels'], device=dev, dtype=torch.float32)
            stop = torch.zeros(B, max_steps, device=dev, dtype=torch.float32)
            align = torch.zeros(B, max_steps, Tx, device=dev, dtype=torch.float32) if want_align else None
            nsteps = torch.zeros(B, device=dev, dtype=torch.int32)
            d = TacoDropout()
            d.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
            d.utterance_offset = int(utterance_offset)
            md = None
            if masks is not None:
                md = torch.as_tensor(masks).to(device=dev, dtype=torch.uint8).contiguous()
                if tuple(md.shape) != (B, max_steps, 2, self.cfg['prenet_units']):
                    raise ValueError('masks must be [B, max_steps, 2, prenet_units]')
                d.mode = 1
                d.d_masks = md.data_ptr()
            fs = None
            if forced_states is not None:
                fs = torch.as_tensor(forced_states).to(device=dev, dtype=torch.float32).contiguous()
                if tuple(fs.shape) != (B, max_steps, self.state_floats(Tx)):
                    raise ValueError(f'forced_states must be [B, max_steps, {self.state_floats(Tx)}]')
                _lib.check(self.lib.b200tts_taco_decode_forced(self._h, _ptr(m), _ptr(ln), B, Tx, C.byref(d), int(max_steps),
                                                               1 if window else 0, _ptr(fs), _ptr(frames), _ptr(stop), _ptr(align),
                                                               _ptr(nsteps), self._stream()))
            else:
                _lib.check(self.lib.b200tts_taco_decode(self._h, _ptr(m), _ptr(ln), B, Tx, C.byref(d), int(max_steps),
                                                        1 if window else 0, _ptr(frames), _ptr(stop), _ptr(align), _ptr(nsteps),
                                                        self._stream()))
            for t in (m, ln, md, fs):
                if t is not None:
                    t.record_stream(torch.cuda.current_stream(self.device))
        return dict(frames=frames, stop=stop, align=align, nsteps=nsteps)

    def state_floats(self, Tx: int) -> int:
        return int(self.lib.b200tts_taco_state_floats(self._h, int(Tx)))

    @staticmethod
    def pack_state(x, st, win=None, Tx_max=None):
        """One teacher-forcing record from the oracle's loop state (oracle/tacotron_oracle.decode, capture_states):
        x [1,80], st = dict(c1,h1,c2,h2 [1,U], ctx [1,E], alpha, cum [Tx], mu), win = dict(max_att, pos_rec)."""
        Tx = st['alpha'].shape[0]
        Tx_max = Tx if Tx_max is None else Tx_max
        pad = np.zeros(Tx_max - Tx, dtype=np.float32)
        win = win or {}
        tail = np.array([float(st['mu']), float(win.get('max_att', 0)), float(win.get('pos_rec', 0)), 0.0], dtype=np.float32)
        return np.concatenate([np.asarray(x, np.float32).ravel(), np.asarray(st['ctx'], np.float32).ravel(),
                               np.asarray(st['c1'], np.float32).ravel(), np.asarray(st['h1'], np.float32).ravel(),
                               np.asarray(st['c2'], np.float32).ravel(), np.asarray(st['h2'], np.float32).ravel(), tail,
                               np.asarray(st['cum'], np.float32), pad, np.asarray(st['alpha'], np.float32), pad])

    def encode(self, ids, lengths=None):
        """ids int [B, Tx] (padded with anything beyond lengths) -> memory [B, Tx, enc_dim] (CUDA tensor)."""
        dev = self._dev()
        i = torch.as_tensor(ids).to(device=dev, dtype=torch.int32).contiguous()
        if i.dim() != 2:
            raise ValueError('ids must be [B, Tx]')
        B, Tx = i.shape
        ln = torch.full((B,), Tx, dtype=torch.int32) if lengths is None else torch.as_tensor(lengths, dtype=torch.int32)
        ln = ln.to(dev)
        with torch.cuda.device(self.device):
            mem = torch.zeros(B, Tx, self.cfg['enc_dim'], device=dev, dtype=torch.float32)
            _lib.check(self.lib.b200tts_taco_encode(self._h, _ptr(i), _ptr(ln), B, Tx, _ptr(mem), self._stream()))
            i.record_stream(torch.cuda.current_stream(self.device)); ln.record_stream(torch.cuda.current_stream(self.device))
        return mem

    def postnet(self, frames, nsteps):
        """frames [B, max_steps, num_mels] raw decoder outputs + nsteps [B] -> mel [B, max_steps, num_mels] (clipped)."""
        dev = self._dev()
        f = torch.as_tensor(frames).to(device=dev, dtype=torch.float32).contiguous()
        n = torch.as_tensor(nsteps).to(device=dev, dtype=torch.int32).contiguous()
        B, ms, _ = f.shape
        with torch.cuda.device(self.device):
            mel = torch.zeros_like(f)
            _lib.check(self.lib.b200tts_taco_postnet(self._h, _ptr(f), _ptr(n), B, ms, _ptr(mel), self._stream()))
            f.record_stream(torch.cuda.current_stream(self.device)); n.record_stream(torch.cuda.current_stream(self.device))
        return mel

    def philox_masks(self, seed, utterance_offset, B, steps):
        with torch.cuda.device(self.device):
            m = torch.empty(B, steps, 2, self.cfg['prenet_units'], device=self._dev(), dtype=torch.uint8)
            _lib.check(self.lib.b200tts_taco_philox_masks(self.device, int(seed) & 0xFFFFFFFFFFFFFFFF, int(utterance_offset),
                                                          B, steps, self.cfg['prenet_units'], _ptr(m), self._stream()))
        return m
