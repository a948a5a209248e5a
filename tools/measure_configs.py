"""Measures the BASELINE.json configs that bench.py does not print (2, 4, 5) on one GPU and writes configs.json
(into the directory given as the first argument, default: the working directory).
Development / documentation aid; inputs: synthetic WaveRNN weights, the shipped Tacotron checkpoint (oracle/_ref travel copy)."""
import json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np, torch
from tacotronv2_wavernn_chinese_b200 import synth
from tacotronv2_wavernn_chinese_b200.engine import WaveRNNEngine

out = {}
voc = WaveRNNEngine(synth.synth_state_dict(0), synth.DEFAULT_DIMS, device=0)

def timed(fn, reps=2):
    best = None
    for _ in range(reps):
        torch.cuda.synchronize(); t0 = time.perf_counter(); r = fn(); torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        best = dt if best is None else min(best, dt)
    return best, r

# ---- config 2: one utterance, 5 s of audio ----
mel = synth.synth_mels(1235, 1, 402)
dt, r = timed(lambda: voc.generate(mel, seed=1))
n = r['wave'].shape[1]
dtf, rf = timed(lambda: voc.generate(mel, seed=1, fold=(11000, 550)))
out['config2'] = dict(frames=402, samples=n, audio_s=n / 22050, unbatched_s=dt, unbatched_khz=n / dt / 1e3, unbatched_rtf=dt / (n / 22050),
                      us_per_step=dt / (402 * 275) * 1e6, fold_s=dtf, fold_khz=n / dtf / 1e3, fold_rtf=dtf / (n / 22050),
                      n_folds=int(rf['labels'].shape[0]))
print('config2', out['config2'], flush=True)

# ---- config 4 / 5: Tacotron on real sentences ----
from taco_common import real_taco_weights, sentences
w = real_taco_weights()
if w is not None:
    from oracle import tacotron_oracle as to
    from tacotronv2_wavernn_chinese_b200.pipeline import synthesize_batch
    from tacotronv2_wavernn_chinese_b200.tacotron.engine import TacoDecoderEngine
    from tacotronv2_wavernn_chinese_b200.tacotron.synthesizer import Synthesizer
    from tacotronv2_wavernn_chinese_b200.tacotron.text import Symbols
    s = sentences()
    syn = Synthesizer(); syn.symbols = Symbols(s['symbols']); syn.engine = TacoDecoderEngine(w, device=0); syn.step = 206500
    txt = lambda k: syn.symbols.sequence_to_text(s['sentences'][k]['ids'][:-1])
    dt, (mels, info) = timed(lambda: syn.mels([txt('241')], seed=1238, max_iters=800))
    nst = int(info['decode']['nsteps'][0])
    t0 = time.perf_counter(); mem = to.encoder(w, s['sentences']['241']['ids']); d = to.decode(w, mem, seed=1238, max_iters=800); to.postnet(w, d['frames']); cpu = time.perf_counter() - t0
    out['config4'] = dict(tokens=51, decoder_steps=nst, gt_frames=s['sentences']['241']['frames'], gpu_s=dt, us_per_decoder_step=dt / nst * 1e6,
                          mel_frames_per_s=nst / dt, cpu_oracle_s=cpu, cpu_steps=int(d['n_steps']))
    print('config4', out['config4'], flush=True)
    for nb in (8, 64):
        texts = [txt(str(i)) for i in range(1, nb + 1)]
        dt, (waves, mm) = timed(lambda: synthesize_batch(syn, voc, texts, seed=7), reps=1 if nb == 64 else 2)
        dtt, _ = timed(lambda: syn.mels(texts, seed=7), reps=1)
        tot = sum(len(x) for x in waves)
        out[f'config5_b{nb}'] = dict(sentences=nb, total_samples=tot, audio_s=tot / 22050, pipeline_s=dt, tacotron_s=dtt, samples_per_s=tot / dt,
                                     rtf=dt / (tot / 22050), mel_frames=[int(x.shape[0]) for x in mm][:8])
        print(f'config5_b{nb}', out[f'config5_b{nb}'], flush=True)
out_dir = sys.argv[1] if len(sys.argv) > 1 else '.'
os.makedirs(out_dir, exist_ok=True)
json.dump(out, open(os.path.join(out_dir, 'configs.json'), 'w'), indent=1)
