# Tacotron-2 hyper-parameters read by tacotron_synthesize.py -- TF-free stand-in for the reference's
# tacotron_hparams.py (which builds a tf.contrib.training.HParams).  Only the values the inference path consumes are kept,
# under the reference's names and with the reference's values (tacotron_hparams.py:66-237 there).
import ast


class HParams:
    """Attribute bag with `parse('a=1,b=True')` overrides, the subset of tf.contrib.training.HParams the CLI used."""

    def __init__(self, **kw):
        self.__dict__.update(kw)

    def values(self):
        return dict(self.__dict__)

    def parse(self, overrides):
        new = HParams(**self.__dict__)
        for item in filter(None, (s.strip() for s in overrides.split(','))):
            key, _, val = item.partition('=')
            if key not in new.__dict__:
                raise KeyError(f'unknown hparam {key!r}')
            try:
                new.__dict__[key] = ast.literal_eval(val)
            except (ValueError, SyntaxError):
                new.__dict__[key] = val
        return new


hparams = HParams(
    # audio / mel scaling
    num_mels=80, sample_rate=22050, hop_size=275, win_size=1100,
    max_abs_value=4.0, symmetric_mels=True, clip_outputs=True, lower_bound_decay=0.1,
    # Griffin-Lim mel inversion (tacotron/datasets/audio.py:122-137, :176-186 there; tacotron_synthesize.py --griffin_lim)
    n_fft=2048, fmin=95, fmax=7600, min_level_db=-100, ref_level_db=20, magnitude_power=2., power=1.5, griffin_lim_iters=60,
    preemphasize=True, preemphasis=0.97, signal_normalization=True, allow_clipping_in_normalization=True,
    # mel analysis of recorded audio (tacotron/datasets/preprocessor.py:52-121 there; tacotron_hparams.py:68-69, 90-93)
    rescale=True, rescaling_max=0.999,
    trim_silence=True, trim_fft_size=2048, trim_hop_size=512, trim_top_db=25,
    # model
    outputs_per_step=1, stop_at_any=True, batch_norm_position='after',
    embedding_dim=128,
    enc_conv_num_layers=3, enc_conv_kernel_size=(5,), enc_conv_channels=256, encoder_lstm_units=256,
    smoothing=False, attention_dim=128, attention_filters=32, attention_kernel=(31,),
    synthesis_constraint=False, synthesis_constraint_type='window', attention_win_size=2,
    prenet_layers=[256, 256], decoder_layers=2, decoder_lstm_units=256, max_iters=2000,
    postnet_num_layers=5, postnet_kernel_size=(5,), postnet_channels=256,
    predict_linear=False,
    tacotron_zoneout_rate=0.1, tacotron_dropout_rate=0.5,
    tacotron_synthesis_batch_size=1,
    tacotron_input='./train.txt',
)
