"""The reference's OWN `ForwardLocationSensitiveAttention.__call__` with its speaking-rate branch switched on -- container-only
test tooling next to oracle/ref_harness_taco_attention.py, which runs the shipped file unmodified.

Both attention files of the reference ship the branch disabled (attention.py:163-165, forward_attention.py:163-165):

    if not self.is_training and False:
        delta_val = -0.04
        mu = tf.clip_by_value(mu + delta_val, 0.0, 1.0)

`ReferenceRateAttention(w, memory, file, mu_bias)` parses `file` (attention.py: no window; forward_attention.py: the window)
from the reference checkout and edits its syntax tree in memory: the test of that one `if` loses its `and False`, and the
constant -0.04 becomes mu_bias.  Nothing is written anywhere; every other statement runs as written.  The edited class is
executed in the namespace of ref_harness_taco_attention's import of forward_attention.py (the numpy stand-in for tensorflow
and the module-level helpers, which the two files share: checked below) and called on the attention object that harness
builds from the checkpoint weights.  Used by oracle/make_golden_taco_rate.py.
"""
from __future__ import annotations

import ast
import os

import numpy as np

import ref_harness_taco_attention as R

CLASS = 'ForwardLocationSensitiveAttention'


class _EnableRateBias(ast.NodeTransformer):
    """`if not self.is_training and False:` around `delta_val = -0.04` -> `if not self.is_training:`, delta_val = delta."""

    def __init__(self, delta):
        self.delta, self.edits = float(np.float32(delta)), 0

    def visit_If(self, node):
        self.generic_visit(node)
        assigns = [n for n in node.body if isinstance(n, ast.Assign) and any(getattr(t, 'id', None) == 'delta_val' for t in n.targets)]
        t = node.test
        if assigns and isinstance(t, ast.BoolOp) and isinstance(t.op, ast.And) and len(t.values) == 2 \
                and isinstance(t.values[1], ast.Constant) and t.values[1].value is False:
            assert ast.unparse(t.values[0]) == 'not self.is_training' and ast.unparse(assigns[0].value) == '-0.04'
            node.test = t.values[0]
            assigns[0].value = ast.copy_location(ast.Constant(self.delta), assigns[0].value)
            self.edits += 1
        return node


def _parse(file):
    path = os.path.join(R.REF_ROOT, 'tacotron/models', file)
    with open(path, encoding='utf-8') as f:
        return path, ast.parse(f.read(), path)


def edited_class(base_module, file, mu_bias):
    """The attention class of reference file `file` with the speaking-rate branch switched on at mu_bias (None: as shipped),
    defined in a copy of `base_module`'s namespace (ref_harness_taco_attention.import_reference: forward_attention.py on the
    numpy stand-in)."""
    path, tree = _parse(file)
    _, base = _parse('forward_attention.py')
    outside = lambda t: [ast.dump(n) for n in t.body if not (isinstance(n, ast.ClassDef) and n.name == CLASS)]
    assert outside(tree) == outside(base), f'{path}: module-level code differs from forward_attention.py'
    edit = _EnableRateBias(0.0 if mu_bias is None else mu_bias)
    cls = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == CLASS]
    assert len(cls) == 1
    cls = cls[0]
    if mu_bias is not None:
        cls = edit.visit(cls)
        assert edit.edits == 1, f'{path}: expected one disabled speaking-rate branch, found {edit.edits}'
    ns = dict(base_module.__dict__)
    exec(compile(ast.fix_missing_locations(ast.Module(body=[cls], type_ignores=[])), path, 'exec'), ns)
    return ns[CLASS]


class ReferenceRateAttention(R.ReferenceAttention):
    """R.ReferenceAttention for ONE sentence whose `__call__` is the edited class's (mu_bias None: the shipped file's): same
    6-tuple, same inputs."""

    def __init__(self, w, memory, file='forward_attention.py', mu_bias=0.0):
        super().__init__(w, memory)
        self.cls = edited_class(self.mod, file, mu_bias)
