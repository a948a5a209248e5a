"""WaveRNNEngine: the torch-facing wrapper of one libb200tts context (one GPU).

PyTorch is only plumbing here (device memory, current stream); all arithmetic runs in
csrc/ through the C ABI.  Tensors in, tensors out.
"""
from __future__ import annotations

import ctypes as C
import weakref

import numpy as np
import torch

from . import _lib
from ._lib import GenOpts, Rng, WaveRNNCfg


def _cfg_from_dims(dims: dict) -> WaveRNNCfg:
    c = WaveRNNCfg()
    c.rnn_dims, c.fc_dims, c.bits, c.pad = dims['rnn_dims'], dims['fc_dims'], dims['bits'], dims['pad']
    c.feat_dims, c.compute_dims = dims['feat_dims'], dims['compute_dims']
    c.res_out_dims, c.res_blocks = dims['res_out_dims'], dims['res_blocks']
    f = tuple(int(x) for x in dims['upsample_factors'])
    if not 1 <= len(f) <= 4:
        raise ValueError('upsample_factors must have 1..4 entries')
    c.n_upsample = len(f)
    for i, s in enumerate(f):
        c.upsample_factors[i] = s
    c.hop_length = dims['hop_length']
    return c


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _rng(mode: int, seed: int, utterance_offset: int) -> Rng:
    """The noise of a call: `mode`, keyed by the 64-bit seed and the utterance id of row 0."""
    rng = Rng()
    rng.mode = mode
    rng.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    rng.utterance_offset = int(utterance_offset) & 0xFFFFFFFFFFFFFFFF
    return rng


MOL_PARAMS, MOL_U = 30, 11          # fc3 outputs and uniforms per step of a mixture-of-logistics model (voc_mode = 'MOL')


class WaveRNNEngine:
    """Owns the packed weights of one model on one device.  `dims['mode']` is the reference's voc_mode: 'RAW' (default)
    or 'MOL'."""

    def __init__(self, state_dict: dict, dims: dict, device: int | None = None):
        if not torch.cuda.is_available():
            raise RuntimeError('no CUDA device: the WaveRNN path has no CPU fallback')
        self.lib = _lib.load()
        self.device = torch.cuda.current_device() if device is None else int(device)
        self.dims = dict(dims)
        self.mode = dims.get('mode', 'RAW')
        if self.mode not in ('RAW', 'MOL'):
            raise ValueError(f"unknown voc_mode {self.mode!r} (expected 'RAW' or 'MOL')")
        self.hop = int(dims['hop_length'])
        self.feat = int(dims['feat_dims'])
        self.res_out = int(dims['res_out_dims'])
        self.n_classes = MOL_PARAMS if self.mode == 'MOL' else 1 << int(dims['bits'])
        host = {}
        for k, v in state_dict.items():
            if hasattr(v, 'detach'):
                v = v.detach().cpu().numpy()
            v = np.asarray(v)
            if v.dtype.kind == 'f':
                host[k] = np.ascontiguousarray(v, dtype=np.float32)
        arr, keep = _lib.make_tensor_array(host)
        cfg = _cfg_from_dims(dims)
        h = C.c_void_p()
        create = self.lib.b200tts_wavernn_create_mol if self.mode == 'MOL' else self.lib.b200tts_wavernn_create
        _lib.check(create(C.byref(h), self.device, C.byref(cfg), arr, len(arr)))
        del keep
        self._h = h
        self._sessions = weakref.WeakSet()

    def close(self):
        if getattr(self, '_h', None):
            for s in list(self._sessions):      # the context frees its open sessions
                s._h = None
            self.lib.b200tts_wavernn_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -------------------------------------------------------------------------------------------
    def _dev(self):
        return torch.device('cuda', self.device)

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _mel(self, mels):
        m = torch.as_tensor(mels)
        if m.dim() != 3 or m.shape[1] != self.feat:
            raise ValueError(f'mels must be [B, {self.feat}, T], got {tuple(m.shape)}')
        return m.to(device=self._dev(), dtype=torch.float32).contiguous()

    def upsample(self, mels, full_aux: bool = True):
        """[B, feat, T] -> (mels_up [B, T*hop, feat], aux [B, T*hop, res_out] or frame-rate [B, T, res_out])."""
        m = self._mel(mels)
        B, _, T = m.shape
        S = T * self.hop
        with torch.cuda.device(self.device):
            up = torch.empty(B, S, self.feat, device=self._dev(), dtype=torch.float32)
            auxf = torch.empty(B, T, self.res_out, device=self._dev(), dtype=torch.float32)
            aux = torch.empty(B, S, self.res_out, device=self._dev(), dtype=torch.float32) if full_aux else None
            _lib.check(self.lib.b200tts_wavernn_upsample(self._h, _ptr(m), B, T, _ptr(up), _ptr(auxf), _ptr(aux),
                                                         self._stream()))
        return up, (aux if full_aux else auxf)

    def generate(self, mels, *, seed: int = 0, utterance_offset: int = 0, utterance_ids=None, q=None, teacher=None,
                 return_logits: bool = False, want_wave: bool = True, mu_law: bool = True, kernel: str = 'auto',
                 max_steps: int = 0, fold=None, utt_frames=None, pack=None, u=None):
        """Runs the generation loop on the device.

        Returns dict(labels int16 [B,S] cuda, wave float64 [B,wave_len] cuda or None, logits [S,B,NC] or None).
        q: optional Exp(1) noise [S,B,NC] (torch/numpy) -> EXT_EXPONENTIAL mode; otherwise PHILOX(seed).
        pack: optional packed-row schedule dict(rows, utt int32 [rows, segs], start int32 [rows, segs+1], steps) from
        pipeline.pack_schedule: `rows` kernel rows run queues of the B utterances back to back (gen_opts.d_pack_*).

        A MOL engine returns dict(samples float32 [B,S] cuda, wave, logits [S,B,30] or None) instead: it takes `u`, the
        uniforms [S,B,11] of every step (EXT_UNIFORM mode), in place of `q`, `teacher` as float samples [B,S], and ignores
        mu_law (the reference turns it off for MOL).  Folding changes [B,S] to [n_folds, fold_len] as for RAW.
        """
        mol = self.mode == 'MOL'
        if mol:
            if q is not None:
                raise ValueError('a MOL engine takes uniforms u [S, B, 11], not the Exp(1) race noise q')
            if pack is not None:
                raise ValueError('packed rows are not built for MOL models: generate the utterances in plain batches')
            noise, noise_name, noise_width, noise_mode = u, 'u', MOL_U, _lib.RNG_EXT_UNIFORM
        else:
            if u is not None:
                raise ValueError('u (uniforms) is the noise of a MOL engine; a RAW engine takes q')
            noise, noise_name, noise_width, noise_mode = q, 'q', self.n_classes, _lib.RNG_EXT_EXPONENTIAL
        m = self._mel(mels)
        B, _, T = m.shape
        S = T * self.hop
        GB, GS = B, S                                     # rows / steps the generation kernels see
        if fold is not None:
            if B != 1:
                raise ValueError('fold-with-overlap generation takes exactly one utterance')
            GB, GS = self.fold_geometry(T, int(fold[0]), int(fold[1]))
        steps = max_steps if max_steps else GS
        dev = self._dev()
        with torch.cuda.device(self.device):
            # labels (RAW) or samples (MOL); a teacher is fed back in their place, so it takes their dtype
            out = torch.zeros(GB, GS, device=dev, dtype=torch.float32 if mol else torch.int16)
            wave = None
            if want_wave and steps == GS:
                wave = torch.empty(B, (T - 1) * self.hop, device=dev, dtype=torch.float64)
            keep = [m]                          # inputs the stream reads after this call returns
            rng = _rng(_lib.RNG_PHILOX if noise is None else noise_mode, seed, utterance_offset)
            if utterance_ids is not None:       # rows that are NOT consecutive utterances (length-sorted chunks): per-row global index
                ids = torch.as_tensor(np.asarray(utterance_ids, dtype=np.int64)).to(dev).contiguous()
                if tuple(ids.shape) != (B,) or fold is not None:
                    raise ValueError('utterance_ids must be [B] (and cannot be combined with fold)')
                rng.d_utterance_ids = ids.data_ptr()
                keep.append(ids)
            if noise is not None:
                nd = torch.as_tensor(noise).to(device=dev, dtype=torch.float32).contiguous()
                if nd.dim() != 3 or tuple(nd.shape[1:]) != (GB, noise_width) or nd.shape[0] < steps:
                    raise ValueError(f'{noise_name} must be [>= {steps}, {GB}, {noise_width}], got {tuple(nd.shape)}')
                rng.d_q = nd.data_ptr()
                keep.append(nd)
            opts = GenOpts()
            opts.kernel = _lib.KERNELS[kernel]
            opts.mu_law = 1 if mu_law and not mol else 0
            opts.max_steps = int(max_steps)
            if fold is not None:
                opts.fold_target, opts.fold_overlap = int(fold[0]), int(fold[1])
            if pack is not None:
                pk_u = torch.as_tensor(np.ascontiguousarray(pack['utt'], dtype=np.int32)).to(dev)
                pk_s = torch.as_tensor(np.ascontiguousarray(pack['start'], dtype=np.int32)).to(dev)
                rows, segs = pk_u.shape
                if tuple(pk_s.shape) != (rows, segs + 1) or rows != int(pack['rows']):
                    raise ValueError('pack: utt must be [rows, segs], start [rows, segs + 1]')
                opts.d_pack_utt, opts.d_pack_start = pk_u.data_ptr(), pk_s.data_ptr()
                opts.pack_rows, opts.pack_segs, opts.pack_steps = rows, segs, int(pack['steps'])
                keep += [pk_u, pk_s]
            if utt_frames is not None:
                uf = torch.as_tensor(utt_frames).to(device=dev, dtype=torch.int32).contiguous()
                if tuple(uf.shape) != (B,):
                    raise ValueError('utt_frames must be [B]')
                opts.d_utt_frames = uf.data_ptr()
                keep.append(uf)
            td = None
            if teacher is not None:
                td = torch.as_tensor(teacher).to(device=dev, dtype=out.dtype).contiguous()
                if tuple(td.shape) != (GB, GS):
                    raise ValueError('teacher must be [B, S] ([n_folds, fold_len] when folding)')
                if not mol:
                    opts.d_teacher = td.data_ptr()
                keep.append(td)
            logits = None
            if return_logits:
                logits = torch.empty(steps, GB, self.n_classes, device=dev, dtype=torch.float32)
                opts.d_logits = logits.data_ptr()
            if mol:
                _lib.check(self.lib.b200tts_wavernn_generate_mol(self._h, _ptr(m), B, T, C.byref(rng), C.byref(opts), _ptr(td),
                                                                 _ptr(out), _ptr(wave), self._stream()))
            else:
                _lib.check(self.lib.b200tts_wavernn_generate(self._h, _ptr(m), B, T, C.byref(rng), C.byref(opts),
                                                             _ptr(out), _ptr(wave), self._stream()))
            for t in keep:
                t.record_stream(torch.cuda.current_stream(self.device))
        return {'samples' if mol else 'labels': out, 'wave': wave, 'logits': logits, 'steps': steps}

    def open_session(self, mel, *, seed: int = 0, utterance_id: int = 0, mu_law: bool = True, kernel: str = 'auto') -> 'WaveRNNSession':
        """A generation session of one RAW utterance: mel [feat, T] (T >= 21) in [0, 1].  Its sample loop then runs in pieces
        (`advance`), and the pieces, concatenated, are bit for bit `generate(mel[None], seed=seed, utterance_ids=[utterance_id])`.
        The conditioning is computed here, once, on the current stream.

        kernel: 'auto' runs the session on the push kernel (up to 32 sessions per run, any cut); 'tc' on the tensor cores (up to
        `max_session_rows` sessions per run, runs of a multiple of hop steps), and its pieces are then bit for bit
        `generate(..., kernel='tc')`.  A session stays on the kernel it was opened for."""
        if kernel not in ('auto', 'tc'):
            raise ValueError(f"kernel must be 'auto' (push) or 'tc', got {kernel!r}")
        m = torch.as_tensor(mel)
        if m.dim() != 2 or m.shape[0] != self.feat:
            raise ValueError(f'mel must be [{self.feat}, T], got {tuple(m.shape)}')
        with torch.cuda.device(self.device):
            m = m.to(device=self._dev(), dtype=torch.float32).contiguous()
            rng = _rng(_lib.RNG_PHILOX, seed, utterance_id)
            h = C.c_void_p()
            _lib.check(self.lib.b200tts_wavernn_session_open_kernel(self._h, _ptr(m), int(m.shape[1]), C.byref(rng), 1 if mu_law else 0,
                                                                    _lib.KERNELS[kernel], C.byref(h), self._stream()))
            m.record_stream(torch.cuda.current_stream(self.device))
        s = WaveRNNSession(self, h)
        self._sessions.add(s)
        return s

    def open_sessions(self, mels, frames, *, seed: int = 0, utterance_ids, mu_law: bool = True, kernel: str = 'auto',
                      layout: str = 'feat_t', max_abs_value: float = 4.0) -> list:
        """n generation sessions opened in three launches, whatever n is (b200tts_wavernn_session_open_batch); device tensors are
        read in place.  Session i is bit for bit `open_session` of row i's first frames[i] frames, zero-padded to 21 frames
        when shorter, with utterance_id utterance_ids[i].

        layout 'feat_t': mels [n, feat, T_max] in [0, 1].  layout 'taco': mels [n, T_max, feat], the Tacotron postnet output,
        mapped on the device like Synthesizer.mels: clip(m, -max_abs_value, max_abs_value), then clip((m + a) / (2a), 0, 1).
        frames: n ints in 1..T_max (host).  n is 1..max_session_rows; kernel 'auto' (push) or 'tc'."""
        if kernel not in ('auto', 'tc'):
            raise ValueError(f"kernel must be 'auto' (push) or 'tc', got {kernel!r}")
        if layout not in _lib.MEL_LAYOUTS:
            raise ValueError(f"layout must be 'feat_t' or 'taco', got {layout!r}")
        m = torch.as_tensor(mels)
        if m.dim() != 3 or m.shape[1 if layout == 'feat_t' else 2] != self.feat:
            want = f'[n, {self.feat}, T_max]' if layout == 'feat_t' else f'[n, T_max, {self.feat}]'
            raise ValueError(f'mels must be {want} for layout {layout!r}, got {tuple(m.shape)}')
        n = int(m.shape[0])
        T_max = int(m.shape[2 if layout == 'feat_t' else 1])
        fr = np.ascontiguousarray(np.asarray(frames).reshape(-1), dtype=np.int32)
        ids = [int(u) & 0xFFFFFFFFFFFFFFFF for u in utterance_ids]
        if len(fr) != n or len(ids) != n:
            raise ValueError(f'need one frame count and one utterance id per row ({n} rows)')
        with torch.cuda.device(self.device):
            m = m.to(device=self._dev(), dtype=torch.float32).contiguous()
            d_ids = torch.tensor(np.array(ids, dtype=np.uint64).view(np.int64), device=self._dev())
            rng = _rng(_lib.RNG_PHILOX, seed, 0)
            rng.d_utterance_ids = d_ids.data_ptr()
            handles = (C.c_void_p * n)()
            _lib.check(self.lib.b200tts_wavernn_session_open_batch(
                self._h, _ptr(m), _lib.MEL_LAYOUTS[layout], float(max_abs_value), fr.ctypes.data_as(C.POINTER(C.c_int32)), n,
                T_max, C.byref(rng), 1 if mu_law else 0, _lib.KERNELS[kernel], handles, self._stream()))
            m.record_stream(torch.cuda.current_stream(self.device))
        out = []
        for h in handles:
            s = WaveRNNSession(self, C.c_void_p(h))
            self._sessions.add(s)
            out.append(s)
        return out

    def advance(self, sessions, max_steps: int):
        """Runs up to `max_steps` more steps of each session in one launch: 1..32 distinct open push sessions of this engine, or
        1..`max_session_rows` tensor-core sessions with `max_steps` a multiple of hop.
        Returns, for each session, (labels int16 [n], wave float64 [w]) cuda tensors: its n = min(max_steps, steps - position)
        labels from its old position, and the w samples of its wave among them (none past wave_len)."""
        sessions = list(sessions)
        if any(s._h is None for s in sessions):
            raise ValueError('a session is closed')
        max_steps = int(max_steps)
        n = len(sessions)
        info = [(s.position, s.steps, s.wave_len) for s in sessions]
        dev = self._dev()
        with torch.cuda.device(self.device):
            rows = max(n, 1)
            labels = torch.empty(rows, max(max_steps, 1), device=dev, dtype=torch.int16)
            wave = torch.empty(rows, max(max_steps, 1), device=dev, dtype=torch.float64)
            handles = (C.c_void_p * rows)(*[s._h.value for s in sessions])
            _lib.check(self.lib.b200tts_wavernn_session_run(self._h, handles, n, max_steps, _ptr(labels), _ptr(wave), self._stream()))
        out = []
        for i, (pos, steps, wave_len) in enumerate(info):
            k = min(max_steps, steps - pos)
            w = max(0, min(pos + k, wave_len) - pos)
            out.append((labels[i, :k], wave[i, :w]))
        return out

    @property
    def max_session_rows(self) -> int:
        """The most sessions one `advance` takes on this engine: 256 where the tensor-core kernel runs, else 32."""
        return int(self.lib.b200tts_wavernn_session_max_rows(self._h))

    def fold_geometry(self, T: int, target: int, overlap: int):
        """(n_folds, fold_len) of fold_with_overlap for a T-frame utterance."""
        nf, fl = C.c_int(), C.c_int()
        _lib.check(self.lib.b200tts_wavernn_fold_geometry(int(T), self.hop, int(target), int(overlap), C.byref(nf), C.byref(fl)))
        return nf.value, fl.value

    def generate_host(self, mels: np.ndarray, *, seed: int = 0, utterance_offset: int = 0, mu_law: bool = True,
                      kernel: str = 'auto', want_labels: bool = True, want_wave: bool = True):
        """HOST buffers in, HOST buffers out, synchronous: the call `wavernn_gen.py` makes end to end."""
        m = np.ascontiguousarray(mels, dtype=np.float32)
        if m.ndim != 3 or m.shape[1] != self.feat:
            raise ValueError(f'mels must be [B, {self.feat}, T], got {m.shape}')
        B, _, T = m.shape
        S = T * self.hop
        labels = np.empty((B, S), dtype=np.int16) if want_labels else None
        wave = np.empty((B, (T - 1) * self.hop), dtype=np.float64) if want_wave else None
        rng = _rng(_lib.RNG_PHILOX, seed, utterance_offset)
        opts = GenOpts()
        opts.kernel = _lib.KERNELS[kernel]
        opts.mu_law = 1 if mu_law else 0
        _lib.check(self.lib.b200tts_wavernn_generate_host(
            self._h, m.ctypes.data_as(C.c_void_p), B, T, C.byref(rng), C.byref(opts),
            labels.ctypes.data_as(C.c_void_p) if labels is not None else C.c_void_p(0),
            wave.ctypes.data_as(C.c_void_p) if wave is not None else C.c_void_p(0)))
        return dict(labels=labels, wave=wave)

    def philox_exponential(self, seed: int, utterance_offset: int, B: int, step0: int, n_steps: int):
        """The Exp(1) noise the PHILOX mode draws, [n_steps, B, NC] on the device (for parity tests)."""
        with torch.cuda.device(self.device):
            q = torch.empty(n_steps, B, self.n_classes, device=self._dev(), dtype=torch.float32)
            _lib.check(self.lib.b200tts_philox_exponential(self.device, int(seed) & 0xFFFFFFFFFFFFFFFF, int(utterance_offset),
                                                           B, step0, n_steps, self.n_classes, _ptr(q), self._stream()))
        return q

    def philox_mol_uniform(self, seed: int, utterance_offset: int, B: int, step0: int, n_steps: int):
        """The uniforms the PHILOX mode of a MOL engine draws, [n_steps, B, 11] on the device (for parity tests)."""
        with torch.cuda.device(self.device):
            u = torch.empty(n_steps, B, MOL_U, device=self._dev(), dtype=torch.float32)
            _lib.check(self.lib.b200tts_philox_mol_uniform(self.device, int(seed) & 0xFFFFFFFFFFFFFFFF, int(utterance_offset),
                                                           B, step0, n_steps, _ptr(u), self._stream()))
        return u

    def debug_phase_cycles(self):
        """[6][2] mean cycles (compute, barrier) per phase of the last grid launch; needs B200TTS_GRID_PROF=1.  After a
        tensor-core launch the 12 values are (exchange wait, GEMM, epilogue) of GRU-2's x1 job, fc1, fc2 and fc3."""
        out = (C.c_double * 12)()
        _lib.check(self.lib.b200tts_wavernn_debug_phase_cycles(self._h, out))
        return np.array(list(out)).reshape(6, 2)

    def check(self):
        """Synchronises and raises if the last generate call's persistent kernel gave up waiting for a peer thread block
        (its wave is NaN-filled in that case).  Call after the point where the caller synchronises anyway."""
        _lib.check(self.lib.b200tts_wavernn_check(self._h))

    def fp32_peak_tflops(self) -> float:
        """Measured fp32 CUDA-core ceiling of this device (register-only FFMA loop), TFLOP/s."""
        v = C.c_double()
        _lib.check(self.lib.b200tts_debug_fp32_peak(self.device, C.byref(v)))
        return float(v.value)

    @property
    def launch_count(self) -> int:
        return int(self.lib.b200tts_wavernn_launch_count(self._h))

    KERNEL_NAMES = {0: None, 1: 'wavernn_utt_kernel', 2: 'wavernn_grid_kernel', 3: 'wavernn_push_kernel', 5: 'wavernn_tc_kernel',
                    6: 'wavernn_push_session_kernel', 7: 'wavernn_tc_session_kernel'}

    def last_kernel(self):
        """Name of the step kernel the last generate call ran."""
        return self.KERNEL_NAMES.get(int(self.lib.b200tts_wavernn_last_kernel(self._h)))

    def last_kernel_ms(self) -> float:
        ms = float(self.lib.b200tts_wavernn_last_kernel_ms(self._h))
        if ms < 0:
            raise _lib.B200TTSError(-1, self.lib.b200tts_last_error().decode())
        return ms


class WaveRNNSession:
    """One RAW utterance whose sample loop runs in pieces (WaveRNNEngine.open_session / advance).  A context manager; close()
    frees its device memory (closing the engine frees it too)."""

    def __init__(self, engine: WaveRNNEngine, handle):
        self.engine = engine
        self._h = handle

    def _info(self):
        if self._h is None:
            raise ValueError('the session is closed')
        pos, steps, wave_len = C.c_int64(), C.c_int64(), C.c_int64()
        _lib.check(self.engine.lib.b200tts_wavernn_session_info(self._h, C.byref(pos), C.byref(steps), C.byref(wave_len)))
        return pos.value, steps.value, wave_len.value

    @property
    def position(self) -> int:
        """Steps generated so far (counted when a run is enqueued)."""
        return self._info()[0]

    @property
    def steps(self) -> int:
        """Steps of the utterance, T * hop."""
        return self._info()[1]

    @property
    def wave_len(self) -> int:
        """Samples of its wave, (T - 1) * hop."""
        return self._info()[2]

    @property
    def done(self) -> bool:
        pos, steps, _ = self._info()
        return pos >= steps

    def close(self):
        if self._h is not None:
            self.engine.lib.b200tts_wavernn_session_destroy(self._h)
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
