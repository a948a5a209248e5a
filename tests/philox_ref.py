"""An independent numpy statement of the library's noise streams: Philox4x32-10 (Salmon, Moraes, Dror and Shaw, "Parallel
random numbers: as easy as 1, 2, 3", SC 2011) and the four ways the library turns its words into noise.

Every stream keys Philox with the 64-bit seed (key words seed & 0xFFFFFFFF, seed >> 32) and puts the 64-bit utterance id in
counter words 2 and 3.  Words 0 and 1 are:

    stream                    word 0   word 1                                     value of word x
    WaveRNN RAW Exp(1) noise  step     class // 4                                 u = ((x >> 9) + 0.5) / 2^23,  q = -log(u)
    WaveRNN MOL uniforms      step     j = 0, 1, 2 (words 0..10 used)             fma((x >> 8) / 2^24, 1 - 2e-5, 1e-5) in fp32
    Griffin-Lim phase         frame    0x80000000 | bin // 4                      (x >> 8) / 2^24
    Tacotron prenet keep flag step     0x40000000 | (layer * P // 4 + unit // 4)  x >> 31

and the value of class c, bin k or unit j is output word c % 4, k % 4 or j % 4 of its counter.  Products of two 32-bit
words fit in uint64, so the round function needs no wide multiply."""
import numpy as np

U32 = np.uint64(0xFFFFFFFF)
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = 0x9E3779B9, 0xBB67AE85            # Weyl increments of the key

RAW_TAG, MOL_TAG, GL_TAG, TACO_TAG = 0, 0, 0x80000000, 0x40000000


def key_of(seed):
    """A Python int seed (any sign) -> the two 32-bit key words, as the library's uint64 seed argument takes it."""
    s = int(seed) & 0xFFFFFFFFFFFFFFFF
    return s & 0xFFFFFFFF, s >> 32


def philox4x32_10(ctr, key):
    """ctr: [..., 4] integer array of 32-bit counter words; key: (k0, k1).  Returns the [..., 4] uint64 output words."""
    c = [np.asarray(ctr[..., i], dtype=np.uint64) & U32 for i in range(4)]
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = _M0 * c[0], _M1 * c[2]
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & U32, p1 >> np.uint64(32), p1 & U32
        c = [hi1 ^ c[1] ^ np.uint64(k0), lo1, hi0 ^ c[3] ^ np.uint64(k1), lo0]
        k0, k1 = (k0 + _W0) & 0xFFFFFFFF, (k1 + _W1) & 0xFFFFFFFF
    return np.stack(c, axis=-1)


def _counters(w0, w1, ids):
    """Broadcast word 0, word 1 and the uint64 ids into [..., 4] counters."""
    ids = np.asarray(ids, dtype=np.uint64)
    w0, w1, ids = np.broadcast_arrays(np.asarray(w0, dtype=np.uint64), np.asarray(w1, dtype=np.uint64), ids)
    return np.stack([w0, w1, ids & U32, ids >> np.uint64(32)], axis=-1)


def ids_of(utterance_offset, B):
    """Utterance ids utterance_offset + b, b < B, wrapping modulo 2^64 as the library's uint64 arithmetic does."""
    return np.array([(int(utterance_offset) + b) & 0xFFFFFFFFFFFFFFFF for b in range(B)], dtype=np.uint64)


def raw_words(seed, ids, step0, n_steps, n_classes):
    """The words behind the RAW noise: [n_steps, B, n_classes] uint64, word of class c at (step, utterance)."""
    s = np.arange(step0, step0 + n_steps, dtype=np.uint64)[:, None, None]
    c4 = np.arange(n_classes // 4, dtype=np.uint64)[None, None, :]
    w = philox4x32_10(_counters(s, RAW_TAG | c4, np.asarray(ids)[None, :, None]), key_of(seed))
    return w.reshape(n_steps, len(ids), n_classes)


def raw_uniform(x):
    """RAW word -> u in (0, 1), float64 (exact: 24 significant bits)."""
    return ((np.asarray(x) >> np.uint64(9)).astype(np.float64) + 0.5) / 2.0 ** 23


def raw_exponential(seed, ids, step0, n_steps, n_classes):
    """(u, q = -log u) of the RAW stream, both float64, [n_steps, B, n_classes]."""
    u = raw_uniform(raw_words(seed, ids, step0, n_steps, n_classes))
    return u, -np.log(u)


_MOL_A = np.float64(np.float32(1.0) - np.float32(2e-5))       # 1.0f - 2e-5f, an fp32 constant
_MOL_B = np.float64(np.float32(1e-5))


def mol_uniform(seed, ids, step0, n_steps):
    """The 11 uniforms per (step, utterance) of the MOL stream, [n_steps, B, 11] float32.  (x >> 8) / 2^24 has 24 significant
    bits and so has _MOL_A: their product is exact in float64 (48 bits), and adding _MOL_B (lowest bit 2^-40) stays within 53
    bits, so the float32 rounding of the float64 sum is the single rounding of the fused multiply-add."""
    s = np.arange(step0, step0 + n_steps, dtype=np.uint64)[:, None, None]
    j = np.arange(3, dtype=np.uint64)[None, None, :]
    w = philox4x32_10(_counters(s, MOL_TAG | j, np.asarray(ids)[None, :, None]), key_of(seed))
    w = w.reshape(n_steps, len(ids), 12)[..., :11]
    a = (w >> np.uint64(8)).astype(np.float64) / 2.0 ** 24
    return (a * _MOL_A + _MOL_B).astype(np.float32)


def gl_uniform(seed, ids, T, n_bins):
    """The Griffin-Lim phase uniforms, [B, T, n_bins] float32 (exact)."""
    t = np.arange(T, dtype=np.uint64)[None, :, None]
    k = np.arange(n_bins, dtype=np.uint64)[None, None, :]
    w = philox4x32_10(_counters(t, GL_TAG | (k >> np.uint64(2)), np.asarray(ids)[:, None, None]), key_of(seed))
    x = np.take_along_axis(w, np.broadcast_to(k & np.uint64(3), w.shape[:-1]).astype(np.int64)[..., None], axis=-1)[..., 0]
    return ((x >> np.uint64(8)).astype(np.float64) / 2.0 ** 24).astype(np.float32)


def taco_keep(seed, ids, steps, P):
    """Tacotron prenet keep flags, [B, steps, 2, P] uint8: layer L, unit j at decoder step s."""
    s = np.arange(steps, dtype=np.uint64)[None, :, None, None]
    L = np.arange(2, dtype=np.uint64)[None, None, :, None]
    j = np.arange(P, dtype=np.uint64)[None, None, None, :]
    w1 = TACO_TAG | (L * np.uint64(P // 4) + (j >> np.uint64(2)))
    w = philox4x32_10(_counters(s, w1, np.asarray(ids)[:, None, None, None]), key_of(seed))
    x = np.take_along_axis(w, np.broadcast_to(j & np.uint64(3), w.shape[:-1]).astype(np.int64)[..., None], axis=-1)[..., 0]
    return (x >> np.uint64(31)).astype(np.uint8)


def word1_range(stream, **domain):
    """[lo, hi] of counter word 1 a stream uses over its domain: RAW n_classes, GL n_bins, Tacotron P (prenet units)."""
    if stream == 'raw':
        return RAW_TAG, RAW_TAG + domain['n_classes'] // 4 - 1
    if stream == 'mol':
        return MOL_TAG, MOL_TAG + 2
    if stream == 'gl':
        return GL_TAG, GL_TAG | (domain['n_bins'] - 1) // 4
    if stream == 'taco':
        return TACO_TAG, TACO_TAG | (domain['P'] // 4 + (domain['P'] - 1) // 4)
    raise ValueError(stream)
