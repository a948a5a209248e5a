"""The noise streams without a device: tests/philox_ref.py against Random123's published Philox4x32-10 known answers and
against the library's own host path of philox4x32_10, the counter map that keeps the four streams apart, and the argument
refusals of the noise dumps."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

import philox_ref as pr

# Random123 1.09, kat_vectors: philox4x32 10 rounds (counter words, key words -> output words)
KAT = [
    ((0x00000000, 0x00000000, 0x00000000, 0x00000000), (0x00000000, 0x00000000),
     (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff, 0xffffffff, 0xffffffff, 0xffffffff), (0xffffffff, 0xffffffff),
     (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
]


@pytest.mark.parametrize('ctr,key,want', KAT)
def test_reference_philox_known_answers(ctr, key, want):
    got = pr.philox4x32_10(np.array([ctr], dtype=np.uint64), key)[0]
    assert [int(x) for x in got] == list(want)


def test_seed_splits_into_key_words():
    assert pr.key_of(0xA4093822299F31D0) == (0x299F31D0, 0xA4093822)
    assert pr.key_of(-1) == (0xFFFFFFFF, 0xFFFFFFFF)
    assert pr.key_of(2 ** 64) == (0, 0)
    assert [int(i) for i in pr.ids_of(2 ** 64 - 2, 3)] == [2 ** 64 - 2, 2 ** 64 - 1, 0]


_HOST_MAIN = r'''
#include <cstdio>
#include "common.cuh"
int main() {
  unsigned c0, c1, c2, c3, k0, k1;
  while (std::scanf("%x %x %x %x %x %x", &c0, &c1, &c2, &c3, &k0, &k1) == 6) {
    uint32_t c[4] = {c0, c1, c2, c3};
    b200tts::philox4x32_10(c, ((uint64_t)k1 << 32) | k0);
    std::printf("%08x %08x %08x %08x\n", c[0], c[1], c[2], c[3]);
  }
  return 0;
}
'''


def test_library_host_philox_matches_reference():
    """common.cuh's philox4x32_10 compiled for the host (its 64-bit-product branch) against the reference: the known answers
    and 2000 random counters and keys."""
    from tacotronv2_wavernn_chinese_b200 import build
    rs = np.random.RandomState(0)
    ctr = np.concatenate([np.array([k[0] for k in KAT], dtype=np.uint64),
                          rs.randint(0, 2 ** 32, size=(2000, 4), dtype=np.uint64)])
    key = np.concatenate([np.array([k[1] for k in KAT], dtype=np.uint64), rs.randint(0, 2 ** 32, size=(2000, 2), dtype=np.uint64)])
    with tempfile.TemporaryDirectory(prefix='philox_host_') as tmp:
        src, exe = os.path.join(tmp, 'host.cu'), os.path.join(tmp, 'host')
        with open(src, 'w') as f:
            f.write(_HOST_MAIN)
        subprocess.run([build._nvcc(), '-std=c++17', '-I', build.CSRC, '-o', exe, src], check=True, capture_output=True)
        lines = ''.join(' '.join(f'{int(v):08x}' for v in list(c) + list(k)) + '\n' for c, k in zip(ctr, key))
        out = subprocess.run([exe], input=lines, check=True, capture_output=True, text=True).stdout.split('\n')
    got = np.array([[int(w, 16) for w in ln.split()] for ln in out if ln], dtype=np.uint64)
    want = np.stack([pr.philox4x32_10(c[None], (int(k[0]), int(k[1])))[0] for c, k in zip(ctr, key)])
    assert got.shape == want.shape and np.array_equal(got, want)
    assert [tuple(int(x) for x in g) for g in got[:3]] == [k[2] for k in KAT]


def _ranges(bits_max=15, n_bins_max=1025, P_max=2 ** 31 - 4):
    """Counter word-1 range of each stream over the largest domain the library accepts: RAW models of up to 2^15 classes
    (b200tts_wavernn_create: bits <= 15), Griffin-Lim at n_fft = 2048 (1025 bins), any prenet width P that is a multiple of 4.
    Each range grows with its parameter, so its largest instance covers every smaller one."""
    return {'raw': pr.word1_range('raw', n_classes=2 ** bits_max), 'mol': pr.word1_range('mol'),
            'gl': pr.word1_range('gl', n_bins=n_bins_max), 'taco': pr.word1_range('taco', P=P_max)}


def test_stream_counters_are_disjoint():
    """No two streams that can share a (seed, utterance id) read the same counter: their word-1 ranges are pairwise disjoint.
    RAW and MOL overlap, and may: a WaveRNN model samples one way or the other, never both."""
    r = _ranges()
    for lo, hi in r.values():
        assert 0 <= lo <= hi < 2 ** 32
    assert r['raw'] == (0, 2 ** 13 - 1) and r['mol'] == (0, 2) and r['gl'] == (2 ** 31, 2 ** 31 + 256)
    assert r['taco'] == (2 ** 30, 2 ** 31 - 3)
    names = sorted(r)
    for i, a in enumerate(names):
        for b in names[i + 1:]:
            if {a, b} == {'raw', 'mol'}:
                continue
            (alo, ahi), (blo, bhi) = r[a], r[b]
            assert ahi < blo or bhi < alo, f'{a} {r[a]} and {b} {r[b]} share counters'


def test_taco_layers_and_units_have_their_own_words():
    """Within the Tacotron stream, each (layer, unit) of a step reads its own (word 1, output word) pair: the keep flags of
    one step are 2 P distinct Philox output words."""
    for P in (4, 8, 256, 1028):
        L, j = np.meshgrid(np.arange(2), np.arange(P), indexing='ij')
        slot = (pr.TACO_TAG | (L * (P // 4) + j // 4)) * 4 + j % 4
        assert np.unique(slot).size == 2 * P


def _lib():
    from tacotronv2_wavernn_chinese_b200 import build, _lib
    build.build_lib()
    return _lib.load()


def test_dump_refusals_before_any_cuda_call():
    """The noise dumps refuse what would run their counters out of range, before any CUDA call: a WaveRNN dump whose last step
    step0 + n_steps - 1 would pass 2^31 - 2 (the kernel computes step0 + s in int), and a keep-flag dump of a prenet width
    that is not a multiple of 4 (its layers would share counter words)."""
    lib = _lib()
    buf = (ctypes.c_float * 64)()
    big = 2 ** 31 - 1
    for step0, n in ((big - 1, 2), (big, 1), (1, big), (2 ** 30, 2 ** 30)):
        assert lib.b200tts_philox_exponential(0, 1, 0, 1, step0, n, 4, buf, None) == -1, (step0, n)
        assert lib.b200tts_philox_mol_uniform(0, 1, 0, 1, step0, n, buf, None) == -1, (step0, n)
    assert lib.b200tts_philox_exponential(0, 1, 0, 1, -1, 1, 4, buf, None) == -1
    assert lib.b200tts_philox_mol_uniform(0, 1, 0, 1, -1, 1, buf, None) == -1
    for P in (5, 6, 7, 258):
        assert lib.b200tts_taco_philox_masks(0, 1, 0, 1, 1, P, buf, None) == -1, P
