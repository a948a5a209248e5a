import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a real H100 (run with -m gpu)')
    config.addinivalue_line('markers', 'reference: needs the reference checkout')


@pytest.fixture(scope='session', autouse=True)
def _bounded_blas_pool():
    """The oracles run thousands of tiny matvecs; more than 4 BLAS threads buys nothing (measured: 61 s with 4, 64 s with 8)
    and, on a busy or over-committed host, spinning worker threads can stretch the suite from one minute to tens of minutes."""
    try:
        from threadpoolctl import threadpool_limits
    except Exception:
        yield
        return
    with threadpool_limits(limits=min(4, os.cpu_count() or 1)):
        yield


GOLDEN = os.path.join(ROOT, 'tests', 'golden')
REF_CKPT_COPY = os.path.join(ROOT, 'oracle', '_ref', 'latest_weights.pyt')


def load_ckpt_state_dict():
    """The shipped checkpoint, from /root/reference (container) or the git-ignored travel copy oracle/_ref/."""
    import numpy as np
    import torch
    for p in ('/root/reference/logs_wavernn/checkpoints/latest_weights.pyt', REF_CKPT_COPY):
        if os.path.isfile(p):
            sd = torch.load(p, map_location='cpu', weights_only=False)
            return {k: v.numpy() for k, v in sd.items()}
    return None


@pytest.fixture(scope='session')
def ckpt_state_dict():
    sd = load_ckpt_state_dict()
    if sd is None:
        pytest.skip('shipped checkpoint not available (neither /root/reference nor oracle/_ref/)')
    return sd
