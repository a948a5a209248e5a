"""fold_with_overlap geometry without a device: b200tts_wavernn_fold_geometry is host arithmetic only, so it is checked here against
the oracle's fold_with_overlap (fatchord_version.py:293-340) over a dense sweep of utterance lengths, together with the rule
every fold-conditioning path on the GPU applies: fold u reads sample u * stride + t while that is before the end, zero after."""
import ctypes

import numpy as np

from oracle import wavernn_oracle as wo
from test_wavernn_fold_gpu import CKPT_CASES, FOLD_CASES, LINEAR_CASES, geometry, grid_kernel_for

HOP, EINVAL = 275, -1

# (target, overlap): the production defaults, both goldens' geometries, every geometry of the GPU sweep, and more small strides
SWEEP = sorted({(11000, 550), (2750, 550), (2700, 500), (2, 3), (100, 20), (275, 2), (548, 2), (1, 549)}
               | {(target, overlap) for _, target, overlap in FOLD_CASES})


def _lib():
    from tacotronv2_wavernn_chinese_b200 import _lib, build
    build.build_lib()
    return _lib.load()


def _geometry(lib, T, target, overlap, hop=HOP):
    nf, fl = ctypes.c_int(), ctypes.c_int()
    rc = lib.b200tts_wavernn_fold_geometry(T, hop, target, overlap, ctypes.byref(nf), ctypes.byref(fl))
    return rc, nf.value, fl.value


def test_fold_geometry_equals_the_oracle_fold():
    lib = _lib()
    checked = 0
    for target, overlap in SWEEP:
        stride = target + overlap
        # every length up to 300 frames; strides under 20 samples make thousands of folds, so those stop at 120 frames
        for T in range(1, 301 if stride >= 20 else 121):
            S = T * HOP
            rc, nf, L = _geometry(lib, T, target, overlap)
            if S <= overlap:
                assert rc == EINVAL, (T, target, overlap)
                continue
            assert rc == 0, (T, target, overlap, lib.b200tts_last_error())
            x = np.arange(1, S + 1, dtype=np.float64).reshape(1, S, 1)
            folded = wo.fold_with_overlap(x, target, overlap)
            assert folded.shape == (nf, L, 1), (T, target, overlap)
            assert (nf, L) == geometry(T, target, overlap)[:2]
            pos = np.arange(nf)[:, None] * stride + np.arange(L)[None, :]
            assert np.array_equal(folded[:, :, 0], np.where(pos < S, pos + 1, 0)), (T, target, overlap)
            checked += 1
    assert checked > 4000


def test_fold_geometry_refusals():
    lib = _lib()
    for T, target, overlap in [(21, 100, 1), (21, 100, 0), (21, 100, -3), (21, 0, 20), (21, -1, 20),
                               (2, 100, 550), (2, 100, 551), (1, 100, 10000),            # T * hop <= overlap
                               (21, 2 ** 31 - 1100, 550), (21, 2 ** 31 - 1, 2),           # L = target + 2 * overlap overflows an int
                               (2 ** 31 // HOP + 1, 11000, 550)]:                        # T * hop overflows an int
        rc, _, _ = _geometry(lib, T, target, overlap)
        assert rc == EINVAL, (T, target, overlap)
        assert lib.b200tts_last_error()
    assert _geometry(lib, 2, 100, 549)[:2] == (0, 1)                                     # S = overlap + 1: one fold
    assert _geometry(lib, 21, 2 ** 31 - 1 - 1100, 550) == (0, 1, 2 ** 31 - 1)            # the longest fold an int holds
    assert _geometry(lib, 21, 100, 20, hop=0)[0] == EINVAL
    import torch
    if not torch.cuda.is_available():
        assert lib.b200tts_device_count() <= 0          # the geometry above was computed without a device


def test_gpu_fold_table_covers_every_edge():
    """The teacher-forced table of test_wavernn_fold_gpu.py puts the fold count on every dispatch boundary and the last fold on
    every edge of fold_with_overlap's padding."""
    geoms = [geometry(*g) + g for g in FOLD_CASES]
    counts = {g[0] for g in geoms}
    assert {1, 2, 8, 9, 16, 17, 32, 33, 64, 65, 128, 129, 256, 257} <= counts           # push G = 8/16/32, wide grid W2/W4/W4x2
    assert max(counts) > 1024 and any(264 < n <= 528 for n in counts)                   # utterance kernel G = 8 and G = 4
    assert all(T >= 21 for T, _, _ in FOLD_CASES)
    rem = [(r, st) for _, _, st, r, _, _, _ in geoms]
    assert any(r == 0 for r, _ in rem) and any(r == 1 for r, _ in rem) and any(r == st - 1 for r, st in rem)
    assert any(n == 1 and L > T * HOP for n, L, _, _, T, _, _ in geoms)                 # one fold longer than the utterance
    assert any(o % 2 == 1 for _, _, o in FOLD_CASES) and any(o == 2 for _, _, o in FOLD_CASES)
    assert any(t < o for _, t, o in FOLD_CASES)
    assert any(st % HOP == 0 for _, _, st, _, _, _, _ in geoms)
    assert any(np.gcd(st, HOP) == 1 for _, _, st, _, _, _, _ in geoms)
    # two folds summed inside the 20-hop fade-out, and a wave that ends more than one fold before total_len
    assert any((T - 21) * HOP <= u * st < (T - 1) * HOP for n, _, st, _, T, _, _ in geoms for u in range(1, n))
    assert any((n - 1) * st >= (T - 1) * HOP for n, _, st, _, T, _, _ in geoms)
    assert {grid_kernel_for(n) for n in counts} == {'wavernn_push_kernel', 'wavernn_grid_kernel'}
    assert set(CKPT_CASES) <= set(FOLD_CASES) and set(LINEAR_CASES) <= set(FOLD_CASES)
