"""Builds csrc/libb200tts.so for sm_90a with nvcc (cross-compiles without a GPU).

    python -m tacotronv2_wavernn_chinese_b200.build [--force]

The library is built IN-TREE (git-ignored).
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, 'csrc')
LIB = os.path.join(CSRC, 'libb200tts.so')
# One translation unit per model stage, so that no stage's device code can change the code ptxas generates for another's.
SOURCES = ['api.cu', 'wavernn.cu', 'tacotron.cu', 'taco_session.cu', 'griffin_lim.cu', 'mel_analysis.cu', 'resample.cu']
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
              '-Xcompiler', '-fPIC', '--expt-relaxed-constexpr']


def _nvcc() -> str:
    for cand in (os.environ.get('NVCC'), shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
        if cand and os.path.isfile(cand):
            return cand
    raise RuntimeError('nvcc not found (set NVCC=/path/to/nvcc)')


def _stale() -> bool:
    if not os.path.isfile(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cu', '.cuh', '.h'))]
    deps.append(os.path.join(os.path.dirname(PKG), 'include', 'b200tts.h'))
    return any(os.path.getmtime(d) > t for d in deps if os.path.isfile(d))


def _run(cmd: list[str]) -> str:
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError('nvcc failed:\n' + ' '.join(cmd) + '\n' + res.stdout + res.stderr)
    return res.stderr


def build_lib(force: bool = False, verbose: bool = False) -> str:
    """Compiles the CUDA library if it is missing or older than its sources; returns its path.

    The translation units compile concurrently into objects in a temporary directory, then link into one shared library."""
    if not force and not _stale():
        return LIB
    nvcc = _nvcc()
    flags = NVCC_FLAGS + (['-Xptxas', '-v'] if verbose else [])
    with tempfile.TemporaryDirectory(prefix='b200tts_build_') as tmp:
        objs = [os.path.join(tmp, os.path.splitext(s)[0] + '.o') for s in SOURCES]
        cmds = [[nvcc] + flags + ['-c', '-o', o, os.path.join(CSRC, s)] for s, o in zip(SOURCES, objs)]
        with ThreadPoolExecutor(max_workers=len(cmds)) as pool:
            logs = list(pool.map(_run, cmds))
        logs.append(_run([nvcc, '-shared', '-gencode', 'arch=compute_90a,code=sm_90a', '-o', LIB + '.tmp'] + objs))
    if verbose:
        print(''.join(logs))
    os.replace(LIB + '.tmp', LIB)
    return LIB


if __name__ == '__main__':
    print(build_lib(force='--force' in sys.argv, verbose='-v' in sys.argv))
