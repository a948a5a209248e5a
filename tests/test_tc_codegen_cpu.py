"""Code generation of the tensor-core WaveRNN step (csrc/wavernn_tc.cuh), checked on the CPU with nvcc.

The step's speed rests on its wgmma being asynchronous: a stage's MMAs run while the warpgroup waits for and issues the next
stage.  ptxas silently serializes every wgmma of the kernel (waits for each one to finish, notes C7510-C7519 under -v) when the
code between an MMA and its wait branches or runs short of registers.  No GPU test notices that; this one does.
"""
import os
import re
import subprocess

import pytest

from conftest import ROOT

KERNEL = '_ZN7b200tts17wavernn_tc_kernelENS_6TcArgsE'
CSRC = os.path.join(ROOT, 'tacotronv2_wavernn_chinese_b200', 'csrc')
# the 16 bytes left are outside every MMA chain: three words of warpgroup 2 (40 registers) in its per-block loop, one of the
# consumers in fc3's per-group loop
MAX_SPILL_BYTES = 16


@pytest.fixture(scope='module')
def compiled(tmp_path_factory):
    from tacotronv2_wavernn_chinese_b200 import build
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip('nvcc not found')
    d = tmp_path_factory.mktemp('tc_codegen')
    src = d / 'tc.cu'
    src.write_text('#include "wavernn_tc.cuh"\n')
    cubin = d / 'tc.cubin'
    res = subprocess.run([nvcc, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '--expt-relaxed-constexpr',
                          '-I', CSRC, '-cubin', '-Xptxas', '-v', '-o', str(cubin), str(src)], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    sass = subprocess.run([os.path.join(os.path.dirname(nvcc), 'cuobjdump'), '-sass', str(cubin)],
                          capture_output=True, text=True, check=True).stdout
    return res.stdout + res.stderr, sass


def test_no_wgmma_serialization_note(compiled):
    log, _ = compiled
    notes = [l for l in log.splitlines() if re.search(r'\(C751\d\)', l) and KERNEL in l]
    assert not notes, notes


def test_spills_bounded(compiled):
    log, _ = compiled
    m = re.search(r'Function properties for ' + KERNEL + r'\s*\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads', log)
    assert m, log
    assert int(m.group(1)) <= MAX_SPILL_BYTES and int(m.group(2)) <= MAX_SPILL_BYTES, m.group(0)


def test_wgmma_waits_only_at_chunk_ends(compiled):
    """Per stage 6 HGMMA; a full drain (DEPBAR gsb0 0x0) right after an HGMMA only ends a K = 128 chunk (every 4th stage),
    and the stages inside a chunk keep one group in flight (DEPBAR gsb0 0x1)."""
    _, sass = compiled
    body = sass.split('Function : ' + KERNEL, 1)[1].split('Function : ', 1)[0]
    ins = [m.group(1).strip() for m in re.finditer(r'/\*[0-9a-f]{4,}\*/\s+([^;]*);', body)]
    hgmma = [i for i, s in enumerate(ins) if s.startswith('HGMMA')]
    assert hgmma and len(hgmma) % 24 == 0, len(hgmma)
    drain_after = sum(1 for i in hgmma if i + 1 < len(ins) and re.match(r'WARPGROUP\.DEPBAR\.LE gsb0, 0x0$', ins[i + 1]))
    keep_one = sum(1 for s in ins if re.match(r'WARPGROUP\.DEPBAR\.LE gsb0, 0x1$', s))
    assert drain_after <= len(hgmma) // 24, (drain_after, len(hgmma))
    assert keep_one == len(hgmma) // 12, (keep_one, len(hgmma))
