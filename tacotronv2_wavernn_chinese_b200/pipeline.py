"""Text -> mel -> audio in one process on the GPU(s) (BASELINE config 5; SURVEY.md 8f rank 2, 8e).

The reference couples its two halves only through a `.npy` file on disk (tacotron_synthesize.py:114-116 ->
wavernn_gen.py:22, float32 (T, 80) = clip((mel + 4) / 8, 0, 1)).  Here the same array goes straight from the Tacotron
postnet to the WaveRNN conditioning network.

Ragged sets are scheduled, not just padded.  A lock-step costs the same whether a row still has samples to produce or not,
and below ~32 rows it barely depends on the row count at all, so
  * the vocoder runs LENGTH-SORTED CHUNKS of at most `max_rows` rows (one launch each, padded only to the longest mel of the
    chunk; every row is truncated / faded at its own length, `gen_opts.d_utt_frames`) -- the padded lock-steps of a 64-sentence
    set drop from (longest - mean) x 64 to the spread inside each chunk;
  * or, when cheaper by the measured step times, PACKED ROWS: one launch whose 8 / 16 / 32 kernel rows each run a queue of
    utterances back to back (longest-processing-time list scheduling, `gen_opts.d_pack_*`), the row restarting from the zero
    state at every utterance start -- no lock-step is spent on padding and a short queue can use a faster, narrower kernel;
  * across ranks the sentences are dealt round-robin in order of decreasing length (SURVEY 8e), so every rank gets the same
    length profile and the makespan is the longest sentence's;
  * the sampling noise and the prenet dropout are keyed by the GLOBAL sentence index (`rng.d_utterance_ids`), so a
    sentence's audio depends neither on the chunking nor on the number of ranks.
For a service, where the time to the first audio matters more than the makespan, StreamingVocoder runs generation SESSIONS
(engine.open_session / advance): every utterance advances by `chunk_steps` samples per launch, its piece of wave is handed out
after each launch, finished utterances leave and queued ones take their rows between launches (continuous batching).  The
pieces of an utterance concatenate to exactly the wave vocode_ragged gives it.
Tacotron itself is replicated on every rank: one thread block decodes one sentence, all sentences of a set decode
concurrently (<= 132 per GPU), so sharding it would not shorten anything -- and it removes the mel exchange.
"""
from __future__ import annotations

import collections

import numpy as np
import torch
import torch.distributed as dist

MIN_FRAMES = 21          # shorter than the 20-hop fade-out cannot be faded (the reference raises, fatchord_version.py:256-258)


def plan_chunks(frames, max_rows=32):
    """Indices of `frames` grouped into launches: sorted by decreasing length, cut every `max_rows`."""
    order = sorted(range(len(frames)), key=lambda i: (-int(frames[i]), i))
    return [order[i:i + max_rows] for i in range(0, len(order), max_rows)]


def deal_round_robin(frames, world):
    """Sentence indices of every rank: the length-sorted list dealt like cards (rank r gets positions r, r+world, ...)."""
    order = sorted(range(len(frames)), key=lambda i: (-int(frames[i]), i))
    return [order[r::world] for r in range(world)]


def padded_lockstep_rows(frames, chunks, hop=275):
    """(row-steps computed, row-steps needed) of a chunk plan: the scheduler's efficiency."""
    done = sum(len(c) * max(max(int(frames[i]) for i in c), MIN_FRAMES) for c in chunks) * hop
    need = sum(max(int(f), MIN_FRAMES) for f in frames) * hop
    return done, need


# us per lock-step of the push kernel by row count (one H100 80GB HBM3 at 700 W, tools/quick_time.py grid 1,8,16,32 3000): the
# scheduler's cost model
STEP_US = {8: 18.0, 16: 34.3, 32: 31.0}


def pack_schedule(frames, rows, hop=275):
    """Longest-processing-time list scheduling of utterances onto `rows` kernel rows: every utterance (longest first) goes to
    the row that frees first.  Returns dict(rows, utt [rows, segs], start [rows, segs + 1], steps) for gen_opts.d_pack_*:
    row r runs utterance utt[r, k] during lock-steps [start[r, k], start[r, k+1]); unused slots: utt = -1, start = 2^31 - 1."""
    order = sorted(range(len(frames)), key=lambda i: (-int(frames[i]), i))
    queue = [[] for _ in range(rows)]
    load = [0] * rows
    for i in order:
        r = min(range(rows), key=lambda j: (load[j], j))
        queue[r].append(i)
        load[r] += max(int(frames[i]), MIN_FRAMES) * hop
    segs = max(1, max(len(q) for q in queue))
    big = 2 ** 31 - 1
    utt = np.full((rows, segs), -1, dtype=np.int32)
    start = np.full((rows, segs + 1), big, dtype=np.int32)
    for r, q in enumerate(queue):
        t = 0
        start[r, 0] = 0
        for k, i in enumerate(q):
            utt[r, k] = i
            t += max(int(frames[i]), MIN_FRAMES) * hop
            start[r, k + 1] = t
    return dict(rows=rows, utt=utt, start=start, steps=int(max(load)), queue=queue)


def plan_ragged(frames, max_rows=32, hop=275):
    """Cheapest of: length-sorted chunks (one utterance per row, padded to the chunk's longest) and packed rows at 8 / 16 / 32
    rows, by the measured step times.  Returns ('chunks', chunk list) or ('pack', schedule)."""
    step = lambda rows: STEP_US[8 if rows <= 8 else (16 if rows <= 16 else 32)]
    chunks = plan_chunks(frames, max_rows)
    best = ('chunks', chunks)
    best_us = sum(max(max(int(frames[i]) for i in c), MIN_FRAMES) * hop * step(len(c)) for c in chunks)
    for rows in (8, 16, 32):
        if rows > max_rows or rows >= 2 * len(frames):
            continue
        sch = pack_schedule(frames, rows, hop)
        us = sch['steps'] * step(rows)
        if us < 0.97 * best_us:
            best, best_us = ('pack', sch), us
    return best


def vocode_ragged(voc, mels, ids, seed=0, max_rows=32, kernel='auto', allow_pack=True):
    """mels: list of float32 [T_b, 80] in [0, 1]; ids: global sentence index of each (keys the sampling noise).
    Returns the list of float64 waves [(max(T_b, 21) - 1) * hop] in the order given."""
    n = len(mels)
    if n == 0:
        return []
    frames = [int(m.shape[0]) for m in mels]
    allow_pack = allow_pack and getattr(voc, 'mode', 'RAW') == 'RAW'      # packed rows are not built for MOL models
    kind, plan = plan_ragged(frames, max_rows, voc.hop) if allow_pack else ('chunks', plan_chunks(frames, max_rows))
    if kind == 'pack':
        # ONE launch: `rows` kernel rows run queues of utterances back to back (state reset at every utterance start)
        T = max(max(frames), MIN_FRAMES)
        feat = mels[0].shape[1]
        batch = np.zeros((n, feat, T), dtype=np.float32)
        uf = np.zeros(n, dtype=np.int32)
        for i, m in enumerate(mels):
            batch[i, :, :frames[i]] = m.T
            uf[i] = max(frames[i], MIN_FRAMES)
        out = voc.generate(torch.as_tensor(batch), seed=seed, utterance_ids=[int(i) for i in ids], kernel=kernel, utt_frames=uf,
                           pack=plan)
        wave = out['wave'].cpu().numpy()
        voc.check()
        return [wave[i, :(uf[i] - 1) * voc.hop].copy() for i in range(n)]
    waves = [None] * n
    feat = mels[0].shape[1]
    for chunk in plan:
        T = max(max(frames[i] for i in chunk), MIN_FRAMES)
        batch = np.zeros((len(chunk), feat, T), dtype=np.float32)      # zero frames past the end == the reference's own padding
        uf = np.zeros(len(chunk), dtype=np.int32)
        for r, i in enumerate(chunk):
            batch[r, :, :frames[i]] = mels[i].T
            uf[r] = max(frames[i], MIN_FRAMES)
        out = voc.generate(torch.as_tensor(batch), seed=seed, utterance_ids=[int(ids[i]) for i in chunk], kernel=kernel,
                           utt_frames=uf)
        wave = out['wave'].cpu().numpy()
        voc.check()
        for r, i in enumerate(chunk):
            waves[i] = wave[r, :(uf[r] - 1) * voc.hop].copy()
    return waves


def _rate_kw(mu_bias, n):
    """The keyword that carries the speaking-rate biases of n sentences to the Synthesizer: none when every bias is 0, so an
    unbiased call is exactly the call made without biases.  Refuses bad biases (ValueError) before anything runs."""
    from .tacotron.engine import mu_bias_array
    b = mu_bias_array(mu_bias, n)
    return {} if b is None else {'mu_bias': b}


def synthesize_batch(synth, wavernn_engine, texts, seed=0, utterance_offset=0, kernel='auto', max_rows=32, allow_pack=True,
                     mu_bias=None):
    """synth: tacotron.synthesizer.Synthesizer (loaded); wavernn_engine: engine.WaveRNNEngine; texts: pinyin strings.
    Returns (list of float64 waves, list of mels [T_b, 80]) for sentences utterance_offset ... of a larger set.
    mu_bias: speaking-rate bias, a scalar or one per text (Synthesizer.mels; positive speaks faster)."""
    mels, _ = synth.mels(texts, seed=seed, utterance_offset=utterance_offset, **_rate_kw(mu_bias, len(texts)))
    ids = [utterance_offset + b for b in range(len(mels))]
    return vocode_ragged(wavernn_engine, mels, ids, seed=seed, max_rows=max_rows, kernel=kernel, allow_pack=allow_pack), list(mels)


def synthesize_sharded(synth, wavernn_engine, texts, seed=0, group=None, kernel='auto', max_rows=32, mu_bias=None):
    """All ranks call this with the SAME `texts` (and `mu_bias`, a scalar or one speaking-rate bias per text); every rank
    returns all waves (input order) and all mels.
    One process per GPU (`torch.distributed`); the only collective is the final all-gather of the padded waves."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    mels, _ = synth.mels(texts, seed=seed, utterance_offset=0, **_rate_kw(mu_bias, len(texts)))   # replicated (module docstring)
    n = len(mels)
    frames = [int(m.shape[0]) for m in mels]
    mine = deal_round_robin(frames, world)[rank]
    local = vocode_ragged(wavernn_engine, [mels[i] for i in mine], mine, seed=seed, max_rows=max_rows, kernel=kernel)
    if world == 1:
        out = [None] * n
        for i, w in zip(mine, local):
            out[i] = w
        return out, list(mels)
    hop = wavernn_engine.hop
    lens = [(max(f, MIN_FRAMES) - 1) * hop for f in frames]
    per_rank = (n + world - 1) // world
    nccl = dist.get_backend(group) == 'nccl'
    dev = torch.device('cuda', torch.cuda.current_device()) if nccl else torch.device('cpu')
    buf = torch.zeros((per_rank, max(lens) if lens else 1), dtype=torch.float64, device=dev)
    for r, w in enumerate(local):
        buf[r, :len(w)] = torch.as_tensor(w, device=dev)
    parts = [torch.empty_like(buf) for _ in range(world)]
    dist.all_gather(parts, buf, group=group)
    shares = deal_round_robin(frames, world)
    out = [None] * n
    for r, share in enumerate(shares):
        host = parts[r].cpu().numpy()
        for k, i in enumerate(share):
            out[i] = host[k, :lens[i]].copy()
    return out, list(mels)


def _host(x):
    return x.cpu().numpy() if hasattr(x, 'cpu') else np.asarray(x)


def _session_rows(engine, max_rows, chunk_steps):
    """Checks a streaming service's rows and chunk against its vocoder engine; True: the sessions run on the tensor cores."""
    cap = int(getattr(engine, 'max_session_rows', 32))
    if not 1 <= int(max_rows) <= cap:
        raise ValueError(f'max_rows must be 1..{cap} (the most sessions one launch of this engine takes)')
    if int(chunk_steps) < 1:
        raise ValueError('chunk_steps must be >= 1')
    tc = int(max_rows) > 32                  # the push kernel runs at most 32 sessions per launch
    if tc and int(chunk_steps) % int(engine.hop):
        raise ValueError(f'above 32 rows the sessions run on the tensor cores: chunk_steps must be a multiple of hop ({engine.hop})')
    return tc


def _advance(engine, active, chunk_steps):
    """One launch over the (key, session) pairs `active` -> ([(key, wave piece, finished)], the pairs still active)."""
    pieces = engine.advance([s for _, s in active], chunk_steps)
    out, still = [], []
    for (key, s), (_labels, wave) in zip(active, pieces):
        finished = s.done
        out.append((key, _host(wave), finished))
        if finished:
            s.close()
        else:
            still.append((key, s))
    return out, still


class StreamingVocoder:
    """Continuous batching of vocoder sessions on one engine.  `submit` queues requests; every `step` admits queued requests
    first come first served into free rows (at most `max_rows` sessions per launch), advances every session by up to
    `chunk_steps` samples in one launch and returns [(key, wave piece float64 numpy, finished)].  A key's pieces concatenate to
    the wave vocode_ragged gives its mel with the same seed and id; mels shorter than MIN_FRAMES are zero-padded to it, as there.

    `max_rows` is the service's capacity, up to the engine's `max_session_rows`.  Up to 32 rows the sessions run on the push
    kernel; above 32 they run on the tensor cores (which then also serve the one-shot reference, `kernel='tc'`), and
    `chunk_steps` must be a multiple of the engine's hop."""

    def __init__(self, engine, seed=0, chunk_steps=2750, max_rows=32):
        self._tc = _session_rows(engine, max_rows, chunk_steps)
        self.engine, self.seed = engine, int(seed)
        self.chunk_steps, self.max_rows = int(chunk_steps), int(max_rows)
        self._queue = collections.deque()       # (key, mel [T, feat], utterance id)
        self._active = []                       # (key, session) in admission order

    def submit(self, key, mel, utterance_id):
        """Queues mel [T, feat] in [0, 1]; the sampling noise is keyed by (seed, utterance_id) like a one-shot run."""
        m = np.asarray(mel, dtype=np.float32)
        if m.ndim != 2:
            raise ValueError(f'mel must be [T, feat], got {m.shape}')
        self._queue.append((key, m, int(utterance_id)))

    @property
    def pending(self) -> int:
        return len(self._queue)

    @property
    def active(self) -> int:
        return len(self._active)

    def idle(self) -> bool:
        return not self._queue and not self._active

    def step(self):
        while self._queue and len(self._active) < self.max_rows:
            key, m, uid = self._queue.popleft()
            T = max(m.shape[0], MIN_FRAMES)
            padded = np.zeros((m.shape[1], T), dtype=np.float32)         # zero frames past the end, as vocode_ragged pads
            padded[:, :m.shape[0]] = m.T
            kw = {'kernel': 'tc'} if self._tc else {}
            self._active.append((key, self.engine.open_session(padded, seed=self.seed, utterance_id=uid, **kw)))
        if not self._active:
            return []
        out, self._active = _advance(self.engine, self._active, self.chunk_steps)
        check = getattr(self.engine, 'check', None)
        if check is not None:
            check()                              # a timed-out run raises here instead of handing out NaN audio
        return out


class StreamingSynthesizer:
    """Text in, audio pieces out: continuous batching of text requests through Tacotron and vocoder sessions on one GPU.
    `submit` queues a pinyin text; every `step`
      * admits queued texts first come, first served, up to min(free rows, `max_admit`), and gives them ONE Tacotron batch
        (encode, decode, postnet: `synth.decode_device`), one device-side stop-token cut (`target_lengths`) and one batched
        session open from the postnet output (`engine.open_sessions(layout='taco')`), so no mel goes through the host;
      * advances every active session by up to `chunk_steps` samples in one launch,
    and returns [(key, wave piece float64 numpy, finished)] in admission order, like StreamingVocoder.step.  A request's mel is
    `Synthesizer.mels` of its admission group with the same ids, and its pieces concatenate to the one-shot generate of that mel
    (zero-padded to 21 frames when shorter) with (seed, utterance_id) on the same kernel family.  A sentence whose stop token
    fires at its first step has an empty mel: it finishes at admission with an empty piece, after the pieces of the sessions.

    Everything runs on the current stream, in order: the Tacotron kernels never run beside the vocoder's persistent kernels,
    whose co-residency on the SMs they could break.  `max_rows` > 32 runs tensor-core sessions, and `chunk_steps` must then be
    a multiple of the engine's hop.

    `decode_steps` = k bounds the Tacotron work done before each vocoder run, whatever the sentence lengths (None: the whole
    decode at admission, as above).  Admitted texts get one encoder batch and one open of decoder sessions
    (`synth.open_decodes`); in-flight decodes plus active vocoder sessions stay within `max_rows`, and in-flight decodes within
    128.  Every step then advances all in-flight decodes by at most k steps in ONE launch, gives the decodes that finished one
    postnet, one stop-token cut (`synth.finish_decodes`) and one batched vocoder open, and runs the vocoder.  A request's first
    piece comes in the step its decode finishes.  Its frames are bit for bit those of the batch decoder (`taco_decoder_kernel`,
    which b200tts_taco_decode runs for B >= 2) on its admission's encoder output with its id, seed and bias, and its pieces
    concatenate to the one-shot generate of the resulting mel on the same kernel family.  A text admitted alone is therefore
    decoded on that kernel too, and its mel differs in bits from the default mode's, which decodes a batch of one on the
    single-sentence kernel."""

    def __init__(self, synth, engine, seed=0, chunk_steps=2750, max_rows=32, max_admit=None, decode_steps=None):
        self._tc = _session_rows(engine, max_rows, chunk_steps)
        if max_admit is not None and int(max_admit) < 1:
            raise ValueError('max_admit must be >= 1 (or None: as many as there are free rows)')
        self.synth, self.engine, self.seed = synth, engine, int(seed)
        self.chunk_steps, self.max_rows = int(chunk_steps), int(max_rows)
        self.max_admit = None if max_admit is None else int(max_admit)
        if decode_steps is not None and int(decode_steps) < 1:
            raise ValueError('decode_steps must be >= 1 (or None: the whole decode at admission)')
        self.decode_steps = None if decode_steps is None else int(decode_steps)
        self._decoding = []                     # (key, utterance id, decoder session) in admission order
        self._queue = collections.deque()       # (key, text, utterance id, speaking-rate bias)
        self._active = []                       # (key, session) in admission order
        self._mels = {}                         # key -> (postnet output of its batch, row, frames)
        self._gone = []                         # keys whose last piece the previous step returned

    def submit(self, key, text, utterance_id, mu_bias=0.0):
        """Queues a pinyin text; its prenet dropout and sampling noise are keyed by (seed, utterance_id).  A text the encoder
        would refuse, more than MAX_TOKENS symbols with its end mark, is refused here, and so is a speaking-rate bias `mu_bias`
        that is not a finite number in [-1, 1] (Synthesizer.mels; positive speaks faster)."""
        from .tacotron.engine import MAX_TOKENS, mu_bias_array
        n = len(self.synth.symbols.text_to_sequence(text))
        if n > MAX_TOKENS:
            raise ValueError(f'text of {n} symbols: the encoder takes at most {MAX_TOKENS}')
        if np.ndim(mu_bias) != 0:
            raise ValueError('mu_bias of one request must be a number')
        b = mu_bias_array(mu_bias, 1)
        self._queue.append((key, text, int(utterance_id), 0.0 if b is None else float(b[0])))

    @property
    def pending(self) -> int:
        return len(self._queue)

    @property
    def active(self) -> int:
        return len(self._active)

    @property
    def decoding(self) -> int:
        """Requests whose Tacotron decode is in flight (decode_steps mode)."""
        return len(self._decoding)

    def idle(self) -> bool:
        return not self._queue and not self._active and not self._decoding

    def mel(self, key):
        """The [T, 80] float32 mel in [0, 1] of an admitted request, until the step after the one that returned its last piece."""
        from .tacotron.synthesizer import unit_mel
        post, b, frames = self._mels[key]
        return unit_mel(_host(post[b, :frames]))

    def _admit(self):
        k = min(len(self._queue), self.max_rows - len(self._active))
        if self.max_admit is not None:
            k = min(k, self.max_admit)
        if k <= 0:
            return []
        batch = [self._queue.popleft() for _ in range(k)]
        keys = [b[0] for b in batch]
        ids = [b[2] for b in batch]
        post, lens = self.synth.decode_device([b[1] for b in batch], ids, seed=self.seed,
                                              **_rate_kw([b[3] for b in batch], k))      # per-row biases, one batch
        return self._open_vocoder(keys, ids, post, lens)

    def _open_vocoder(self, keys, ids, post, lens):
        """Vocoder sessions for the rows of a postnet output [n, T, 80] with device target lengths `lens`; returns the finished
        (key, empty piece, True) of the rows whose mel is empty."""
        frames = [int(f) for f in _host(lens)]
        if min(frames) < 0:
            raise RuntimeError('Tacotron decoder kernel gave up waiting for a peer thread block (nsteps < 0); results are invalid')
        k = len(keys)
        for b, key in enumerate(keys):
            self._mels[key] = (post, b, frames[b])
        rows = [b for b in range(k) if frames[b] > 0]
        if rows:
            mels = post if len(rows) == k else post[rows]
            sessions = self.engine.open_sessions(mels, [frames[b] for b in rows], seed=self.seed, utterance_ids=[ids[b] for b in rows],
                                                 kernel='tc' if self._tc else 'auto', layout='taco')
            self._active += [(keys[b], s) for b, s in zip(rows, sessions)]
        return [(keys[b], np.zeros(0, dtype=np.float64), True) for b in range(k) if frames[b] == 0]

    def _decode_slice(self):
        """decode_steps mode: admits queued texts into decoder sessions, advances every in-flight decode by at most
        decode_steps steps in one launch, and hands the decodes that finished to the vocoder."""
        from .tacotron.engine import MAX_DECODE_SESSIONS
        k = min(len(self._queue), self.max_rows - len(self._active) - len(self._decoding), MAX_DECODE_SESSIONS - len(self._decoding))
        if self.max_admit is not None:
            k = min(k, self.max_admit)
        if k > 0:
            batch = [self._queue.popleft() for _ in range(k)]
            ids = [b[2] for b in batch]
            biases = [b[3] for b in batch]
            sessions = self.synth.open_decodes([b[1] for b in batch], ids, seed=self.seed, mu_bias=biases if any(biases) else None)
            self._decoding += [(b[0], b[2], s) for b, s in zip(batch, sessions)]
        if not self._decoding:
            return []
        self.synth.engine.advance_decodes([s for _, _, s in self._decoding], self.decode_steps)
        done = [d for d in self._decoding if d[2].done]
        self._decoding = [d for d in self._decoding if not d[2].done]
        if not done:
            return []
        post, lens = self.synth.finish_decodes([s for _, _, s in done])
        empty = self._open_vocoder([d[0] for d in done], [d[1] for d in done], post, lens)
        for _, _, s in done:
            s.close()
        return empty

    def step(self):
        for key in self._gone:
            self._mels.pop(key, None)
        empty = self._admit() if self.decode_steps is None else self._decode_slice()
        out = []
        if self._active:
            out, self._active = _advance(self.engine, self._active, self.chunk_steps)
        out += empty
        self._gone = [key for key, _piece, finished in out if finished]
        check = getattr(self.engine, 'check', None)
        if out and check is not None:
            check()                              # a timed-out run raises here instead of handing out NaN audio
        return out


def synthesize_stream(synth, wavernn_engine, text, seed=0, utterance_id=0, chunk_steps=2750, mu_bias=0.0):
    """One sentence as a stream: yields its Tacotron mel [T, 80] first, then its wave pieces (float64 numpy) as the vocoder
    makes them.  The pieces concatenate to synthesize_batch's wave of the sentence with utterance_offset = utterance_id and
    the same speaking-rate bias `mu_bias`."""
    mels, _ = synth.mels([text], seed=seed, utterance_offset=utterance_id, **_rate_kw(mu_bias, 1))
    mel = mels[0]
    yield mel
    sv = StreamingVocoder(wavernn_engine, seed=seed, chunk_steps=chunk_steps, max_rows=1)
    sv.submit(0, mel, utterance_id)
    while True:
        for _key, piece, finished in sv.step():
            yield piece
            if finished:
                return
