"""Generates the fixtures of the host-side and training checks against the REFERENCE'S OWN CODE, executed under the
TensorFlow API stand-in of tf_shim.py, so that those checks run without the reference present:
    refshim_live.npz      a few decode steps of synthesize.py's loop + SSRN, the variable names the graph asked for
    refshim_host.npz      data_load.load_data("synthesize") ids and vocabulary, utils.guided_attention, the Noam
                          schedule, utils.spectrogram2wav / load_spectrograms on seeded inputs
    refshim_train.npz     the Text2Mel and SSRN training-graph losses on seeded batches
The inputs are the ones tests/test_reference_shim.py and tests/test_train.py regenerate from the same seeds.  Needs a
checkout of the reference at tf_shim.REFERENCE; run from the repo root:
    python tests/golden/make_golden_refchecks.py
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
import tf_shim                                                   # noqa: E402
from dc_tts_b200.hyperparams import Hyperparams as hp            # noqa: E402
from dc_tts_b200.params import init_params, synthetic_text       # noqa: E402
from oracle import ref_features as rf                            # noqa: E402
from oracle import ref_train as rtr                              # noqa: E402
from oracle import ref_vocoder as rv                             # noqa: E402

LR_STEPS = np.array([0, 1, 3999, 4000, 123456])
P = init_params(0, "perturbed")

# 1. a few decode steps of the loop and SSRN on their first 8 frames (test_reference_code_few_steps)
store = tf_shim.Store(P)
tf_shim.install(store)
L = synthetic_text(2, 40, seed=5)
r = tf_shim.synthesize(L, steps=3, with_ssrn=False)
_, z = tf_shim.run_ssrn(r["Y"][:, :8])
np.savez_compressed(os.path.join(HERE, "refshim_live.npz"), Y3=r["Y"][:, :3], p_hist=r["p_hist"], Y8=r["Y"][:, :8], Z8=z,
                    requested=np.array(sorted(store.requested)))

# 2. host-side pieces (test_text_adaptor / test_training_constants / test_vocoder_and_feature_composition)
tf_shim.install(tf_shim.Store({}))
import data_load as ref_dl                                       # noqa: E402
import hyperparams as ref_hp                                     # noqa: E402
import utils as ref_utils                                        # noqa: E402
ref_hp.Hyperparams.test_data = os.path.join(tf_shim.REFERENCE, "harvard_sentences.txt")
ids = ref_dl.load_data("synthesize")
char2idx, idx2char = ref_dl.load_vocab()
vocab = np.array([idx2char[i] for i in range(len(idx2char))])
assert all(char2idx[c] == i for i, c in enumerate(vocab))
ga = ref_utils.guided_attention()
lr = np.array([float(ref_utils.learning_rate_decay(hp.lr, gs)) for gs in LR_STEPS])
WAVS = {}
ref_utils.librosa = types.SimpleNamespace(
    stft=lambda y, n_fft=None, hop_length=None, win_length=None: rv.stft(np.asarray(y, np.float32), n_fft, hop_length, win_length),
    istft=lambda S, hop_length=None, win_length=None, window="hann": rv.istft(S, hop_length, win_length),
    effects=types.SimpleNamespace(trim=lambda y: (lambda se: (y[se[0]:se[1]], se))(rv.trim_indices(np.asarray(y)))),
    filters=types.SimpleNamespace(mel=lambda sr, n_fft, n_mels: rf.mel_basis(sr, n_fft, n_mels)),
    load=lambda fpath, sr=None: (WAVS[fpath], sr))
ref_hp.Hyperparams.n_iter = 3
rng = np.random.default_rng(0)
mag = rng.uniform(0.2, 0.8, (40, 1 + hp.n_fft // 2)).astype(np.float32)
wav = ref_utils.spectrogram2wav(mag)
t = np.arange(int(hp.sr * 0.8)) / hp.sr
y = (0.2 * np.sin(2 * np.pi * 300 * t) + 0.02 * rng.standard_normal(t.size)).astype(np.float32)
y[:2000] *= 1e-5
WAVS["LJ001-0001.wav"] = y
fname, mel, mg = ref_utils.load_spectrograms("LJ001-0001.wav")
assert fname == "LJ001-0001.wav"
ref_hp.Hyperparams.n_iter = hp.n_iter
np.savez_compressed(os.path.join(HERE, "refshim_host.npz"), ids=ids, vocab=vocab, guided_attention=ga, lr_steps=LR_STEPS,
                    lr=lr, wav=wav, mel=mel, mag=mg)

# 3. training-graph losses (test_oracle_losses / test_oracle_ssrn_losses)
tf_shim.install(tf_shim.Store(P))
L = synthetic_text(2, 50, seed=7)
mels = np.random.default_rng(3).uniform(0, 1, (2, hp.max_T, hp.n_mels)).astype(np.float32)
out = {}
for tag, seed, rate in (("drop", 11, hp.dropout_rate), ("nodrop", 0, 0.0)):
    ref_hp.Hyperparams.dropout_rate = rate
    ref, ncalls = tf_shim.run_train_graph(L, mels, lambda x, r_, i, s=seed: x * rtr.dropout_keep(x.shape, i, s, r_))
    ref_hp.Hyperparams.dropout_rate = hp.dropout_rate
    out["t2m_%s" % tag] = np.array([ref[k] for k in ("loss", "loss_mels", "loss_bd1", "loss_att")], np.float64)
    out["t2m_%s_ncalls" % tag] = np.array(ncalls)
smels = np.random.default_rng(3).uniform(0, 1, (2, 12, hp.n_mels)).astype(np.float32)
smags = np.random.default_rng(4).uniform(0, 1, (2, 48, 1 + hp.n_fft // 2)).astype(np.float32)
ref, ncalls = tf_shim.run_train_graph_ssrn(smels, smags, lambda x, r_, i: x * rtr.dropout_keep(x.shape, i, 9, r_))
out["ssrn"] = np.array([ref[k] for k in ("loss", "loss_mags", "loss_bd2")], np.float64)
out["ssrn_ncalls"] = np.array(ncalls)
np.savez_compressed(os.path.join(HERE, "refshim_train.npz"), **out)
print("reference-check fixtures written to %s" % HERE)
