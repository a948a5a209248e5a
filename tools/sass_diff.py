"""Compares the SASS of two builds of the library kernel by kernel.

    python tools/sass_diff.py OLD.so NEW.so

Runs `cuobjdump -sass` on each file and splits the listing at its `Function : <name>` lines.  The fatbin and ELF headers
between the functions (identifiers, source file names, architecture lines) are not compared, nor is the padding between
columns, so a change that only moves kernels between translation units passes.  Every instruction and its encoding is.
Prints the kernels present in one build only and the kernels whose instructions differ, and exits non-zero if there is
either.

ptxas does not always give taco_grid_kernel the same code: compiled several times at once on a loaded machine, some builds of
the same source come out with a different schedule (16 more SASS lines).  A difference in that kernel alone is worth one
rebuild on an idle machine before it is taken as a change.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys


def _cuobjdump() -> str:
    for cand in (os.environ.get('CUOBJDUMP'), shutil.which('cuobjdump'), '/usr/local/cuda/bin/cuobjdump'):
        if cand and os.path.isfile(cand):
            return cand
    raise RuntimeError('cuobjdump not found (set CUOBJDUMP=/path/to/cuobjdump)')


def kernels(path: str) -> dict[str, str]:
    """Function name -> its SASS lines, for every function of every cubin in `path`."""
    out = subprocess.run([_cuobjdump(), '-sass', path], capture_output=True, text=True, check=True).stdout
    funcs: dict[str, list[str]] = {}
    cur = None
    for line in out.splitlines():
        s = line.strip()
        if s.startswith('Function : '):
            cur = s[len('Function : '):]
            if cur in funcs:
                raise ValueError(f'{path}: {cur} is compiled into more than one translation unit')
            funcs[cur] = []
        elif cur is not None:
            if s.startswith(('Fatbin ', 'code for ', 'arch = ', 'code version = ', 'host = ', 'compile_size = ',
                             'identifier = ', 'ptxasOptions = ')) or s.startswith('.') or not s:
                if s.startswith(('Fatbin ', 'code for ')):
                    cur = None
                continue
            funcs[cur].append(' '.join(s.split()))     # column widths follow the longest line of the whole cubin
    return {k: '\n'.join(v) for k, v in funcs.items()}


def main(argv: list[str]) -> int:
    if len(argv) != 2:
        print(__doc__.strip(), file=sys.stderr)
        return 2
    a, b = (kernels(p) for p in argv)
    only_a, only_b = sorted(set(a) - set(b)), sorted(set(b) - set(a))
    common = sorted(set(a) & set(b))
    differ = [k for k in common if a[k] != b[k]]
    print(f'{len(a)} kernels in {argv[0]}, {len(b)} in {argv[1]}, {len(common)} in both')
    for k in only_a:
        print(f'  only in {argv[0]}: {k}')
    for k in only_b:
        print(f'  only in {argv[1]}: {k}')
    for k in differ:
        n = sum(1 for x, y in zip(a[k].splitlines(), b[k].splitlines()) if x != y)
        print(f'  SASS differs: {k} ({n} lines differ, {len(a[k].splitlines())} vs {len(b[k].splitlines())} lines)')
    same = len(common) - len(differ)
    print(f'{same} of {len(common)} common kernels have identical SASS')
    return 0 if not (only_a or only_b or differ) else 1


if __name__ == '__main__':
    sys.exit(main(sys.argv[1:]))
