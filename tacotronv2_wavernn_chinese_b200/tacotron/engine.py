"""TacoDecoderEngine: torch-facing wrapper of the Tacotron-2 decoder context of libb200tts (one GPU)."""
from __future__ import annotations

import ctypes as C
import weakref

import numpy as np
import torch

from .. import _lib
from .._lib import TacoCfg, TacoDropout

MAX_TOKENS = 512       # kTacoMaxTx: the longest sentence, in symbols, the encoder and decoders take
MAX_DECODE_SESSIONS = 128     # kTacoSessRows: the most decoder sessions one open or slice takes (one wave of the SMs)

DEFAULT_CFG = dict(num_mels=80, prenet_units=256, lstm_units=256, enc_dim=512, attn_dim=128, attn_filters=32,
                   attn_kernel=31, zoneout=0.1)      # tacotron_hparams.py:99-215 of the reference


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def mu_bias_array(mu_bias, B):
    """Speaking-rate biases of a batch of B sentences (b200tts_taco_decode_biased): a scalar or [B] -> float32 [B], or None when
    there is none (None, or every bias 0: the unbiased decoder, bit for bit).  Each must be finite and in [-1, 1]; positive
    biases speak faster.  Raises ValueError otherwise."""
    if mu_bias is None:
        return None
    b = np.asarray(mu_bias, dtype=np.float32)
    if b.ndim == 0:
        b = np.full(B, b, dtype=np.float32)
    if b.shape != (B,):
        raise ValueError(f'mu_bias must be a scalar or [{B}] (one per sentence), got shape {b.shape}')
    if not (np.isfinite(b).all() and (np.abs(b) <= 1).all()):
        raise ValueError('mu_bias must be finite and in [-1, 1]')
    return None if not b.any() else np.ascontiguousarray(b)


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
        self._sessions = weakref.WeakSet()
        emb = host.get('inputs_embedding')
        self.vocab = int(emb.shape[0]) if emb is not None and emb.ndim == 2 else None

    def close(self):
        if getattr(self, '_h', None):
            for s in list(self._sessions):      # the context frees its open sessions
                s._h = None
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

    def _memory(self, memory, rows='B'):
        """An encoder output [rows, Tx, enc_dim] -> contiguous float32 on this engine's device."""
        m = torch.as_tensor(memory).to(device=self._dev(), dtype=torch.float32).contiguous()
        if m.dim() != 3 or m.shape[2] != self.cfg['enc_dim']:
            raise ValueError(f'memory must be [{rows}, Tx, {self.cfg["enc_dim"]}]')
        return m

    @staticmethod
    def _lengths(lengths, B, Tx):
        """Sentence lengths [B] in [1, Tx], or None (= Tx) -> int32 tensor."""
        ln = torch.full((B,), Tx, dtype=torch.int32) if lengths is None else torch.as_tensor(lengths, dtype=torch.int32)
        if tuple(ln.shape) != (B,) or B < 1 or int(ln.max()) > Tx or int(ln.min()) < 1:
            raise ValueError('lengths must be [B] in [1, Tx]')
        return ln

    def _dropout(self, seed, utterance_offset, masks, B, steps):
        """The prenet-dropout descriptor: PHILOX keyed by (seed, utterance_offset + b), or EXT when `masks`, uint8 keep flags
        [B, steps, 2, prenet_units], are given.  Returns (descriptor, the masks on the device or None)."""
        d = TacoDropout()
        d.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
        d.utterance_offset = int(utterance_offset)
        if masks is None:
            return d, None
        md = torch.as_tensor(masks).to(device=self._dev(), dtype=torch.uint8).contiguous()
        if tuple(md.shape) != (B, steps, 2, self.cfg['prenet_units']):
            raise ValueError(f'masks must be [{B}, {steps}, 2, {self.cfg["prenet_units"]}]')
        d.mode = 1
        d.d_masks = md.data_ptr()
        return d, md

    def decode(self, memory, lengths=None, *, masks=None, seed=0, utterance_offset=0, max_steps=2000, window=False,
               want_align=True, forced_states=None, mu_bias=None):
        """memory [B, Tx, enc_dim] (tensor/ndarray); lengths [B] or None (= Tx).  masks: optional uint8 keep flags
        [B, max_steps, 2, prenet_units] (EXT mode) else Philox(seed).  Returns dict(frames [B,max_steps,80], stop
        [B,max_steps], align [B,max_steps,Tx] or None, nsteps [B]) as CUDA tensors (rows beyond nsteps are undefined).
        forced_states: optional [B, max_steps, state_floats(Tx)] teacher-forcing records (see include/b200tts.h,
        b200tts_taco_decode_forced): the whole recurrent state is reloaded before every step and exactly max_steps steps run.
        mu_bias: speaking-rate bias, a scalar or one per sentence, each finite in [-1, 1] (b200tts_taco_decode_biased: the
        forward-attention speed bias of attention.py:163-165; positive is faster).  None or all zeros: the unbiased decoder."""
        dev = self._dev()
        m = self._memory(memory)
        B, Tx, _ = m.shape
        bias = mu_bias_array(mu_bias, B)
        ln = self._lengths(lengths, B, Tx).to(dev)
        with torch.cuda.device(self.device):
            frames = torch.zeros(B, max_steps, self.cfg['num_mels'], device=dev, dtype=torch.float32)
            stop = torch.zeros(B, max_steps, device=dev, dtype=torch.float32)
            align = torch.zeros(B, max_steps, Tx, device=dev, dtype=torch.float32) if want_align else None
            nsteps = torch.zeros(B, device=dev, dtype=torch.int32)
            d, md = self._dropout(seed, utterance_offset, masks, B, max_steps)
            fs = None
            if forced_states is not None:
                fs = torch.as_tensor(forced_states).to(device=dev, dtype=torch.float32).contiguous()
                if tuple(fs.shape) != (B, max_steps, self.state_floats(Tx)):
                    raise ValueError(f'forced_states must be [B, max_steps, {self.state_floats(Tx)}]')
            if bias is not None:
                _lib.check(self.lib.b200tts_taco_decode_biased(self._h, _ptr(m), _ptr(ln), B, Tx, C.byref(d), int(max_steps),
                                                               1 if window else 0, bias.ctypes.data_as(C.POINTER(C.c_float)),
                                                               _ptr(fs), _ptr(frames), _ptr(stop), _ptr(align), _ptr(nsteps),
                                                               self._stream()))
            elif fs is not None:
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

    def decode_gta(self, memory, lengths, targets, target_lengths, *, masks=None, seed=0, utterance_offset=0, want_align=False):
        """Ground-truth-aligned decoding (b200tts_taco_decode_gta): teacher-forced on `targets` [B, Ty_max, num_mels] (used as
        given; the reference clips them to +-4 first), exactly clamp(target_lengths[b], 0, Ty_max) steps per sentence.
        memory [B, Tx, enc_dim]; lengths [B] or None (= Tx); target_lengths [B] or None (= Ty_max).  masks: optional uint8 keep
        flags [B, Ty_max, 2, prenet_units] (EXT mode) else Philox(seed), the stream `decode` draws.  Returns dict(frames
        [B, Ty_max, 80] raw decoder outputs, align [B, Ty_max, Tx] or None, nsteps [B] int32) as CUDA tensors; rows at or
        beyond nsteps are zero."""
        dev = self._dev()
        m = self._memory(memory)
        B, Tx, _ = m.shape
        tg = torch.as_tensor(targets).to(device=dev, dtype=torch.float32).contiguous()
        if tg.dim() != 3 or tg.shape[0] != B or tg.shape[2] != self.cfg['num_mels'] or tg.shape[1] < 1:
            raise ValueError(f'targets must be [{B}, Ty_max >= 1, {self.cfg["num_mels"]}]')
        Ty = tg.shape[1]
        ln = self._lengths(lengths, B, Tx).to(dev)
        tl = torch.full((B,), Ty, dtype=torch.int32) if target_lengths is None else torch.as_tensor(target_lengths, dtype=torch.int32)
        if tuple(tl.shape) != (B,):
            raise ValueError('target_lengths must be [B]')
        tl = tl.clamp(0, Ty).to(dev)
        with torch.cuda.device(self.device):
            frames = torch.zeros(B, Ty, self.cfg['num_mels'], device=dev, dtype=torch.float32)
            align = torch.zeros(B, Ty, Tx, device=dev, dtype=torch.float32) if want_align else None
            d, md = self._dropout(seed, utterance_offset, masks, B, Ty)
            _lib.check(self.lib.b200tts_taco_decode_gta(self._h, _ptr(m), _ptr(ln), B, Tx, C.byref(d), _ptr(tg), _ptr(tl), Ty,
                                                        _ptr(frames), _ptr(align), self._stream()))
            for t in (m, ln, tg, tl, md):
                if t is not None:
                    t.record_stream(torch.cuda.current_stream(self.device))
        return dict(frames=frames, align=align, nsteps=tl)

    def open_decode_sessions(self, memory, lengths, ids, *, seed=0, max_steps=2000, window=False, mu_bias=None) -> list:
        """Free runs to be decoded in slices (b200tts_taco_session_open_batch): memory [n, Tx, enc_dim] (n 1..128), lengths [n]
        in [1, Tx] or None (= Tx), ids: n 64-bit utterance ids keying each row's prenet dropout with `seed`.  mu_bias: a scalar or
        one per row, as in `decode`.  The memory is copied and its keys computed here, on the current stream; every session
        starts at step 0.  However `advance_decodes` cuts them, a session's frames, stop values and step count are bit for bit
        those `decode` gives its row at B >= 2 (one thread block per sentence) with utterance_offset = its id."""
        m = self._memory(memory, 'n')
        n, Tx, _ = m.shape
        ln = np.ascontiguousarray(self._lengths(lengths, n, Tx).cpu().numpy())
        uid = np.ascontiguousarray([int(i) & 0xFFFFFFFFFFFFFFFF for i in ids], dtype=np.uint64)
        if len(uid) != n:
            raise ValueError(f'need one id per row ({n} rows)')
        bias = mu_bias_array(mu_bias, n)
        d, _ = self._dropout(seed, 0, None, n, max_steps)
        handles = (C.c_void_p * max(n, 1))()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.b200tts_taco_session_open_batch(
                self._h, _ptr(m), ln.ctypes.data_as(C.POINTER(C.c_int32)), n, Tx, C.byref(d), uid.ctypes.data_as(C.POINTER(C.c_uint64)),
                int(max_steps), 1 if window else 0, None if bias is None else bias.ctypes.data_as(C.POINTER(C.c_float)), handles,
                self._stream()))
            m.record_stream(torch.cuda.current_stream(self.device))
        out = []
        for h in handles[:n]:
            s = TacoDecodeSession(self, C.c_void_p(h))
            self._sessions.add(s)
            out.append(s)
        return out

    def advance_decodes(self, sessions, n: int):
        """Advances 1..128 distinct open decoder sessions of this engine by up to n steps each in one launch (a finished session
        takes part with 0 steps); a session stops at the step whose stop token exceeds 0.5.  Returns when the slice has finished,
        with every session's `position` and `done` updated."""
        sessions = list(sessions)
        if any(s._h is None for s in sessions):
            raise ValueError('a session is closed')
        handles = (C.c_void_p * max(len(sessions), 1))(*[s._h.value for s in sessions])
        with torch.cuda.device(self.device):
            _lib.check(self.lib.b200tts_taco_session_run(self._h, handles, len(sessions), int(n), self._stream()))

    def decode_outputs(self, sessions):
        """The steps decoded so far by 1..128 sessions, in the layout `decode` returns: dict(frames [n, T, 80], stop [n, T],
        nsteps [n] int32) as CUDA tensors, T the longest position (at least 1), zeros past each session's position."""
        sessions = list(sessions)
        if any(s._h is None for s in sessions):
            raise ValueError('a session is closed')
        T = max([1] + [s.position for s in sessions])
        n = len(sessions)
        dev = self._dev()
        handles = (C.c_void_p * max(n, 1))(*[s._h.value for s in sessions])
        with torch.cuda.device(self.device):
            frames = torch.empty(max(n, 1), T, self.cfg['num_mels'], device=dev, dtype=torch.float32)
            stop = torch.empty(max(n, 1), T, device=dev, dtype=torch.float32)
            nsteps = torch.empty(max(n, 1), device=dev, dtype=torch.int32)
            _lib.check(self.lib.b200tts_taco_session_outputs(handles, n, T, _ptr(frames), _ptr(stop), _ptr(nsteps), self._stream()))
        return dict(frames=frames, stop=stop, nsteps=nsteps)

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
        """ids int [B, Tx] (padded with anything beyond lengths) -> memory [B, Tx, enc_dim] (CUDA tensor); lengths [B] in
        [1, Tx] or None (= Tx).  Every id below its sentence's length must be in [0, vocab): checked before anything launches."""
        dev = self._dev()
        i = torch.as_tensor(ids).to(dtype=torch.int32)
        if i.dim() != 2:
            raise ValueError('ids must be [B, Tx]')
        B, Tx = i.shape
        ln = self._lengths(lengths, B, Tx)
        if self.vocab is not None:                 # (without the encoder variables the library refuses the call itself)
            valid = torch.arange(Tx, device=i.device)[None, :] < ln.to(i.device)[:, None]
            if bool(((i < 0) | (i >= self.vocab))[valid].any()):
                raise ValueError(f'ids below lengths must be in [0, {self.vocab})')
        i = i.to(dev).contiguous()
        ln = ln.to(dev)
        with torch.cuda.device(self.device):
            mem = torch.zeros(B, Tx, self.cfg['enc_dim'], device=dev, dtype=torch.float32)
            _lib.check(self.lib.b200tts_taco_encode(self._h, _ptr(i), _ptr(ln), B, Tx, _ptr(mem), self._stream()))
            i.record_stream(torch.cuda.current_stream(self.device)); ln.record_stream(torch.cuda.current_stream(self.device))
        return mem

    def postnet(self, frames, nsteps):
        """frames [B, max_steps, num_mels] raw decoder outputs + nsteps [B] (<= max_steps; <= 0, e.g. the -1 of a failed decode,
        is an empty row) -> mel [B, max_steps, num_mels] (clipped; rows at or beyond nsteps are zero)."""
        dev = self._dev()
        f = torch.as_tensor(frames).to(device=dev, dtype=torch.float32).contiguous()
        if f.dim() != 3 or f.shape[2] != self.cfg['num_mels']:
            raise ValueError(f'frames must be [B, max_steps, {self.cfg["num_mels"]}]')
        B, ms, _ = f.shape
        n = torch.as_tensor(nsteps).to(device=dev, dtype=torch.int32).contiguous()
        if tuple(n.shape) != (B,) or B < 1 or int(n.max()) > ms:
            raise ValueError('nsteps must be [B] with values <= max_steps')
        with torch.cuda.device(self.device):
            mel = torch.zeros_like(f)
            _lib.check(self.lib.b200tts_taco_postnet(self._h, _ptr(f), _ptr(n), B, ms, _ptr(mel), self._stream()))
            f.record_stream(torch.cuda.current_stream(self.device)); n.record_stream(torch.cuda.current_stream(self.device))
        return mel

    def target_lengths(self, stop, nsteps):
        """The reference's cut of a free run (tacotron_synthesize.py:104-105), on the device: per sentence the first step
        t < nsteps whose np.round(stop) is 1 (stop > 0.5), else nsteps.  stop [B, max_steps] and nsteps [B] as `decode` returns
        them -> int32 [B] CUDA tensor (a negative nsteps, a failed decode, is passed through)."""
        dev = self._dev()
        st = torch.as_tensor(stop).to(device=dev, dtype=torch.float32).contiguous()
        if st.dim() != 2 or st.shape[0] < 1 or st.shape[1] < 1:
            raise ValueError('stop must be [B, max_steps]')
        B, ms = st.shape
        n = torch.as_tensor(nsteps).to(device=dev, dtype=torch.int32).contiguous()
        if tuple(n.shape) != (B,):
            raise ValueError('nsteps must be [B]')
        with torch.cuda.device(self.device):
            out = torch.empty(B, device=dev, dtype=torch.int32)
            _lib.check(self.lib.b200tts_taco_target_lengths(_ptr(st), _ptr(n), B, ms, _ptr(out), self._stream()))
            st.record_stream(torch.cuda.current_stream(self.device)); n.record_stream(torch.cuda.current_stream(self.device))
        return out

    def philox_masks(self, seed, utterance_offset, B, steps):
        with torch.cuda.device(self.device):
            m = torch.empty(B, steps, 2, self.cfg['prenet_units'], device=self._dev(), dtype=torch.uint8)
            _lib.check(self.lib.b200tts_taco_philox_masks(self.device, int(seed) & 0xFFFFFFFFFFFFFFFF, int(utterance_offset),
                                                          B, steps, self.cfg['prenet_units'], _ptr(m), self._stream()))
        return m


class TacoDecodeSession:
    """One free-running Tacotron decode in slices (TacoDecoderEngine.open_decode_sessions / advance_decodes).  A context
    manager; close() frees its device memory once the other sessions of its open are closed too (closing the engine frees it)."""

    def __init__(self, engine: TacoDecoderEngine, handle):
        self.engine = engine
        self._h = handle

    def _info(self):
        if self._h is None:
            raise ValueError('the session is closed')
        pos, done, ms = C.c_int32(), C.c_int32(), C.c_int32()
        _lib.check(self.engine.lib.b200tts_taco_session_info(self._h, C.byref(pos), C.byref(done), C.byref(ms)))
        return pos.value, bool(done.value), ms.value

    @property
    def position(self) -> int:
        """Steps decoded so far."""
        return self._info()[0]

    @property
    def done(self) -> bool:
        """The stop token fired, or the decode reached max_steps."""
        return self._info()[1]

    @property
    def max_steps(self) -> int:
        return self._info()[2]

    def close(self):
        if self._h is not None:
            self.engine.lib.b200tts_taco_session_destroy(self._h)
            self._h = None
            self.engine._sessions.discard(self)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
