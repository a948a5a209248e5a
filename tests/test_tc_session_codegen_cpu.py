"""Code generation of the tensor-core session kernel (wavernn_tc_session_kernel, csrc/wavernn_tc.cuh), checked on the CPU with
nvcc: its wgmma stay asynchronous like the one-shot kernel's (no C751x serialization note, the same waits), and the spills its
session rows add stay outside every GEMM, whose MMA chains hold the accumulators in registers."""
import os
import re
import subprocess

import pytest

from conftest import ROOT

KERNEL = '_ZN7b200tts25wavernn_tc_session_kernelENS_6TcArgsENS_8TcSessIOE'
CSRC = os.path.join(ROOT, 'tacotronv2_wavernn_chinese_b200', 'csrc')
# the session state loads and saves and the per-row frames of the conditioning warps (40 registers); none inside a GEMM
MAX_SPILL_BYTES = 256


@pytest.fixture(scope='module')
def compiled(tmp_path_factory):
    from tacotronv2_wavernn_chinese_b200 import build
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip('nvcc not found')
    d = tmp_path_factory.mktemp('tc_session_codegen')
    src = d / 'tc.cu'
    src.write_text('#include "wavernn_tc.cuh"\n')
    cubin = d / 'tc.cubin'
    res = subprocess.run([nvcc, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '--expt-relaxed-constexpr',
                          '-I', CSRC, '-cubin', '-Xptxas', '-v', '-o', str(cubin), str(src)], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    sass = subprocess.run([os.path.join(os.path.dirname(nvcc), 'cuobjdump'), '-sass', str(cubin)],
                          capture_output=True, text=True, check=True).stdout
    body = sass.split('Function : ' + KERNEL, 1)[1].split('Function : ', 1)[0]
    ins = [m.group(1).strip() for m in re.finditer(r'/\*[0-9a-f]{4,}\*/\s+([^;]*);', body)]
    return res.stdout + res.stderr, ins


def test_no_wgmma_serialization_note(compiled):
    log, _ = compiled
    assert KERNEL in log
    notes = [l for l in log.splitlines() if re.search(r'\(C751\d\)', l) and KERNEL in l]
    assert not notes, notes


def test_spills_bounded(compiled):
    log, _ = compiled
    m = re.search(r'Function properties for ' + KERNEL + r'\s*\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads', log)
    assert m, log
    assert int(m.group(1)) <= MAX_SPILL_BYTES and int(m.group(2)) <= MAX_SPILL_BYTES, m.group(0)


def test_wgmma_waits_only_at_chunk_ends(compiled):
    _, ins = compiled
    hgmma = [i for i, s in enumerate(ins) if s.startswith('HGMMA')]
    assert hgmma and len(hgmma) % 96 == 0, len(hgmma)
    drain_after = sum(1 for i in hgmma if i + 1 < len(ins) and re.match(r'WARPGROUP\.DEPBAR\.LE gsb0, 0x0$', ins[i + 1]))
    keep_one = sum(1 for s in ins if re.match(r'WARPGROUP\.DEPBAR\.LE gsb0, 0x1$', s))
    assert drain_after <= len(hgmma) // 24, (drain_after, len(hgmma))
    assert keep_one == len(hgmma) // 12, (keep_one, len(hgmma))


def test_no_local_memory_inside_a_gemm(compiled):
    """A GEMM is 16 stages x 6 HGMMA = 96 in a row; no spill load or store may sit between its first and its last."""
    _, ins = compiled
    hgmma = [i for i, s in enumerate(ins) if s.startswith('HGMMA')]
    spans = [(hgmma[j], hgmma[j + 95]) for j in range(0, len(hgmma), 96)]
    local = [i for i, s in enumerate(ins) if re.search(r'\b(STL|LDL)\b', s)]
    inside = [ins[i] for i in local if any(a <= i <= b for a, b in spans)]
    assert not inside, inside
