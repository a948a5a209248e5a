"""Ad-hoc kernel timing on the GPU box (development aid; bench.py is the contract)."""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from tacotronv2_wavernn_chinese_b200 import synth
from tacotronv2_wavernn_chinese_b200.engine import WaveRNNEngine

kernels = sys.argv[1].split(',') if len(sys.argv) > 1 else ['utterance']
batches = [int(x) for x in sys.argv[2].split(',')] if len(sys.argv) > 2 else [1, 132, 256]
steps = int(sys.argv[3]) if len(sys.argv) > 3 else 2000
eng = WaveRNNEngine(synth.synth_state_dict(0), synth.DEFAULT_DIMS, device=0)
for k in kernels:
    for B in batches:
        mels = torch.as_tensor(synth.synth_mels(1, B, 80)).cuda()
        for it in range(2):
            eng.generate(mels, seed=1, kernel=k, max_steps=steps, want_wave=False)
            ms = eng.last_kernel_ms()
        if os.environ.get('B200TTS_GRID_PROF') and k == 'grid':
            pc = eng.debug_phase_cycles() / steps
            if B <= 32:                                      # push kernel: 11 slots of thread 0 (see PUSH_MARK)
                names = ['P01poll', 'P01gate', 'P2gemm', 'P2gate', 'hh1', 'P3gemm', 'P3gate+hh2', 'P4gemm', 'P4gate+cond', 'P5gemm', 'P5sample', '-']
                print('   cycles/step:', ' '.join(f'{n}={v:.0f}' for n, v in zip(names, pc.reshape(-1))), f' total {pc.sum():.0f}')
            else:
                print('   cycles/step per phase (compute, barrier):', ' | '.join(f'P{i}: {a:.0f},{b:.0f}' for i, (a, b) in enumerate(pc)), f' total {pc.sum():.0f}')
        if os.environ.get('B200TTS_GRID_PROF') and k == 'tc':
            # per job (mean over the CTAs of its role): exchange wait, GEMM, epilogue; summed over the groups of a step
            pc = (eng.debug_phase_cycles() / steps).reshape(4, 3)
            print('   cycles/step (wait, gemm, epilogue):', ' | '.join(f'{n}: {a:.0f},{b:.0f},{c:.0f}' for n, (a, b, c) in
                                                                zip(['GRU-2 x1', 'fc1', 'fc2', 'fc3'], pc)))
        print(f'kernel={k} B={B} steps={steps}: {ms:.1f} ms -> {ms*1e3/steps:.1f} us/step, {B*steps/ms*1e3/1e6:.3f} M samples/s', flush=True)
