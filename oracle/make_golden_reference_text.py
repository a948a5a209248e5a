"""Writes two small fixtures from the reference checkout, so that the tests comparing with it run without it:

  tests/golden/train_txt_token_cover.txt: pinyin column of a greedy cover of train.txt lines holding every token
  tests/golden/wavernn_hparams_reference.json: repr() of every value of the reference's wavernn_hparams.py

    python oracle/make_golden_reference_text.py /path/to/reference
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def tokens(line):
    return set(line.strip().split('|')[-1].strip().split(' '))


def main(ref):
    lines = open(os.path.join(ref, 'train.txt'), encoding='utf-8').read().splitlines()
    todo = set().union(*(tokens(l) for l in lines))
    cover = []
    while todo:
        best = max(lines, key=lambda l: len(tokens(l) & todo))
        cover.append(best)
        todo -= tokens(best)
    with open(os.path.join(GOLDEN, 'train_txt_token_cover.txt'), 'w', encoding='utf-8') as f:
        f.write('\n'.join(l.strip().split('|')[-1].strip() for l in cover) + '\n')
    ns = {}
    exec(open(os.path.join(ref, 'wavernn_hparams.py'), encoding='utf-8').read(), ns)
    vals = {k: repr(v) for k, v in ns.items() if not k.startswith('__')}
    with open(os.path.join(GOLDEN, 'wavernn_hparams_reference.json'), 'w', encoding='utf-8') as f:
        json.dump(vals, f, indent=1, sort_keys=True)
    print(len(cover), 'lines;', len(vals), 'hparams')


if __name__ == '__main__':
    if len(sys.argv) != 2:
        raise SystemExit(__doc__)
    main(sys.argv[1])
