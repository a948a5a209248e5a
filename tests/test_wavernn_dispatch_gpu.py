"""Which step kernel a generate call runs, and how many kernels it launches, for every rule of the dispatch (csrc/wavernn.cu):
kernel=auto by row count, the explicit kernels, fold-with-overlap, packed rows, the debug buffers, the 256-row tensor-core slices
and the memory-budget cut.  A refused call launches nothing.  Synthetic weights, 21 frames, a few steps unless a wave is asked for.
The launch counts pin what each path launches (bench.py reports them as gpu_launches), so no change to the dispatch alters them
unnoticed."""
import os

import numpy as np
import pytest

from tacotronv2_wavernn_chinese_b200 import synth
from test_wavernn_gpu import engine_for, torch_cuda  # noqa: F401  (torch_cuda is a fixture)

pytestmark = pytest.mark.gpu

T, STEPS = 21, 8
UTT, GRID, PUSH, TC = 'wavernn_utt_kernel', 'wavernn_grid_kernel', 'wavernn_push_kernel', 'wavernn_tc_kernel'

_models = {}


def _engine(**dims):
    """Engine of synthetic weights with `dims` over the default hparams (hop_length follows the upsample factors)."""
    from tacotronv2_wavernn_chinese_b200.engine import WaveRNNEngine
    key = tuple(sorted(dims.items()))
    if key not in _models:
        d = dict(synth.DEFAULT_DIMS, **dims)
        d['hop_length'] = int(np.prod(d['upsample_factors']))
        _models[key] = WaveRNNEngine(synth.synth_state_dict(3, d), d)
    return _models[key]


def _packed(eng, kernel='auto'):
    from tacotronv2_wavernn_chinese_b200 import pipeline as pl
    frames = [21, 23, 22]
    return eng.generate(synth.synth_mels(4, len(frames), max(frames)), seed=1, kernel=kernel,
                        utt_frames=np.array(frames, np.int32), pack=pl.pack_schedule(frames, 2))


def _run(eng, rows, **kw):
    kw.setdefault('max_steps', STEPS)
    kw.setdefault('want_wave', False)
    return eng.generate(synth.synth_mels(rows, rows, T), seed=7, **kw)


def _budget(rows, **kw):
    """rows under a 100 MB conditioning budget: 1.85 MB per row -> ranges of 32 rows."""
    def call(eng):
        os.environ['B200TTS_MAX_COND_BYTES'] = '100e6'
        try:
            return _run(eng, rows, **kw)
        finally:
            del os.environ['B200TTS_MAX_COND_BYTES']
    return call


# (case, call, step kernel of the last launch, kernels launched)
CASES = [(f'auto {b}', (lambda b: lambda e: _run(e, b))(b), k, n) for b, k, n in [
    (1, PUSH, 4), (8, PUSH, 4), (9, PUSH, 4), (16, PUSH, 4), (17, PUSH, 4), (32, PUSH, 4), (33, GRID, 4), (64, GRID, 4),
    (65, GRID, 4), (128, GRID, 4), (129, TC, 3), (256, TC, 3),
    (300, GRID, 7)]] + [                                                        # one 256-row tensor-core slice, then a 44-row tail
    ('grid 20', lambda e: _run(e, 20, kernel='grid'), PUSH, 4),
    ('grid 200', lambda e: _run(e, 200, kernel='grid'), GRID, 4),
    ('utterance 3', lambda e: _run(e, 3, kernel='utterance'), UTT, 3),
    ('tc 1', lambda e: _run(e, 1, kernel='tc'), TC, 3),
    ('tc 40', lambda e: _run(e, 40, kernel='tc'), TC, 3),
    ('fold 10 folds', lambda e: _run(e, 1, fold=(550, 50), max_steps=0), PUSH, 4),
    ('fold 48 folds', lambda e: _run(e, 1, fold=(100, 20), max_steps=0), GRID, 4),
    ('fold utterance', lambda e: _run(e, 1, fold=(550, 50), max_steps=0, kernel='utterance'), UTT, 4),
    ('packed rows', _packed, PUSH, 5),
    ('300 rows with logits', lambda e: _run(e, 300, return_logits=True), GRID, 4),      # debug buffers: never sliced
    # 7 push launches, not one on the tensor cores: the budget cuts every path, although only the wide grid allocates the
    # sample-rate buffer it bounds
    ('200 rows under a budget', _budget(200), PUSH, 28),
    ('200 rows under a budget, full length with a wave', _budget(200, max_steps=0, want_wave=True), PUSH, 35),
]


@pytest.mark.parametrize('case,call,kernel,launches', CASES, ids=[c[0] for c in CASES])
def test_dispatch_table(torch_cuda, case, call, kernel, launches):
    eng, _ = engine_for('synth5')
    n = eng.launch_count
    call(eng)
    eng.check()
    assert (eng.last_kernel(), eng.launch_count - n) == (kernel, launches), case


def _refused(eng, call, text):
    from tacotronv2_wavernn_chinese_b200._lib import B200TTSError
    n = eng.launch_count
    with pytest.raises(B200TTSError) as e:
        call()
    assert e.value.code == -1 and text in str(e.value), str(e.value)          # -1 = B200TTS_EINVAL
    assert eng.launch_count == n, f'a refused call launched work: {e.value}'


def test_packed_rows_need_the_push_kernel(torch_cuda):
    eng, _ = engine_for('synth5')
    _refused(eng, lambda: _packed(eng, kernel='utterance'), 'packed generation needs the push kernel')


def test_model_without_the_grid_kernel(torch_cuda):
    """rnn_dims = fc_dims = 256: 1024 classes are not 8 per CTA of 64, so only the utterance kernel runs it."""
    eng = _engine(rnn_dims=256, fc_dims=256)
    n = eng.launch_count
    _run(eng, 3)
    assert (eng.last_kernel(), eng.launch_count - n) == (UTT, 3)
    _refused(eng, lambda: _run(eng, 3, kernel='grid'), 'kernel=grid was requested')


def test_fir_too_wide_for_the_tensor_core_kernel(torch_cuda):
    """Upsample factors (8, 15, 15): hop 1 800 x 5 taps = 9 000 FIR floats, more than the tensor-core kernel's 8 192-float slot
    but within what the push kernel's shared memory holds.  kernel=auto gives 129 rows to the wide grid; kernel=tc is refused
    before anything is launched."""
    eng = _engine(upsample_factors=(8, 15, 15))
    n = eng.launch_count
    _run(eng, 8)
    assert (eng.last_kernel(), eng.launch_count - n) == (PUSH, 4)
    n = eng.launch_count
    _run(eng, 129)
    assert (eng.last_kernel(), eng.launch_count - n) == (GRID, 4)
    _refused(eng, lambda: _run(eng, 129, kernel='tc'), 'kernel=tc needs')


@pytest.mark.parametrize('rows,kernel', [(8, PUSH), (64, GRID), (129, TC)])
def test_phase_cycles_belong_to_the_last_call(torch_cuda, rows, kernel):
    """debug_phase_cycles returns the counters of a profiled call, and refuses after a call that recorded none."""
    from tacotronv2_wavernn_chinese_b200._lib import B200TTSError
    eng, _ = engine_for('synth5')
    os.environ['B200TTS_GRID_PROF'] = '1'
    try:
        _run(eng, rows)
    finally:
        del os.environ['B200TTS_GRID_PROF']
    assert eng.last_kernel() == kernel
    pc = eng.debug_phase_cycles()
    assert np.isfinite(pc).all() and (pc >= 0).all() and pc.sum() > 0, pc
    _run(eng, rows)
    with pytest.raises(B200TTSError) as e:
        eng.debug_phase_cycles()
    assert 'no phase profile recorded' in str(e.value)
