# Hyper-parameters consumed by wavernn_gen.py through `hp.configure(<this file>)`.
# Names and values are the contract of the reference's wavernn_hparams.py (same keys, same numbers),
# so a checkpoint trained there (logs_wavernn/checkpoints/latest_weights.pyt) loads unchanged.

# --- where things live -----------------------------------------------------------------------------
feature_path = './wavernn_training_data.txt'
voc_model_id = 'wavernn'          # checkpoint family under logs_wavernn/
ignore_tts = True

# --- signal processing shared by every model -------------------------------------------------------
sample_rate = 22050
n_fft = 2048
fft_bins = n_fft // 2 + 1
num_mels = 80
hop_length = 275                  # 12.5 ms
win_length = 1100                 # 50 ms
fmin = 95
min_level_db = -100
ref_level_db = 20
bits = 10                         # 2**bits softmax classes
mu_law = True                     # labels are mu-law companded
peak_norm = True

# --- vocoder architecture ---------------------------------------------------------------------------
voc_mode = 'RAW'                  # 'RAW' = softmax over 2**bits labels; 'MOL' = mixture of 10 logistics (no mu-law)
voc_upsample_factors = (5, 5, 11) # product must equal hop_length
voc_rnn_dims = 512
voc_fc_dims = 512
voc_compute_dims = 128
voc_res_out_dims = 128
voc_res_blocks = 10

# --- training knobs (kept for file compatibility; training is out of scope here) --------------------
voc_batch_size = 32
voc_lr = 1e-4
voc_checkpoint_every = 1000
voc_gen_at_checkpoint = 5
voc_total_steps = 500_000
voc_test_samples = 50
voc_pad = 2                       # conditioning network looks 2 frames beyond each side
voc_seq_len = hop_length * 5
voc_clip_grad_norm = 4

# --- generation --------------------------------------------------------------------------------------
voc_gen_batched = False
voc_target = 11_000
voc_overlap = 550
