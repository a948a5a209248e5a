"""H100-native (sm_90a) WaveRNN sample-generation loop and Tacotron-2 decoder step.

Drop-in for the hot paths of lturing/tacotronv2_wavernn_chinese behind that
project's own Python surface (`wavernn_gen.py --file`, `WaveRNN.generate`).
All compute goes through the C-ABI library `csrc/libb200tts.so`
(declared in include/b200tts.h); there is no CPU fallback.
"""
__version__ = "0.1.0"
