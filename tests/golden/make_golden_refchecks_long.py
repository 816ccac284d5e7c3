"""Generates refshim_long_text.npz: the reference's OWN synthesis and training graphs (train.py Graph, executed under the
TensorFlow API stand-in of tf_shim.py) with the reference's Hyperparams.max_N raised to 300, as a user with longer texts
edits hyperparams.py:
    synth_*      one sess.run of Graph(mode="synthesize") on six utterances of 200..299 characters padded to 300, with
                 prev_max_attentions 0, 191, 192, 250, 297, 299 (the last two at the window's edge): Y, max_attentions,
                 the alignments under each window (align_win, keys p..p+2, zero rows past N) and the largest |alignment|
                 outside it (align_outside, exactly 0 in the reference)
    t2m_*        the losses of Graph(num=1, mode="train") at (B, N, T) = (2, 300, 53) and at a bucket with N_b = 250,
                 (3, 250, 149), with the shared dropout mask of oracle/ref_train.dropout_keep
The inputs are regenerated from the seeds below by tests/test_long_text_reference.py and tests/test_gpu_long_text.py.
Needs a checkout of the reference at tf_shim.REFERENCE; run from the repo root:
    python tests/golden/make_golden_refchecks_long.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
import tf_shim                                                   # noqa: E402
from dc_tts_b200.hyperparams import Hyperparams as hp            # noqa: E402
from dc_tts_b200.params import init_params, synthetic_bucket     # noqa: E402
from oracle import ref_train as rtr                              # noqa: E402

LONG_N = 300
SYNTH_PMA = (0, 191, 192, 250, 297, 299)
SYNTH_LENGTHS = (290, 260, 250, 299, 298, 200)
T2M_CASES = (("t2m_2x300x53", 2, 300, 53, 11), ("t2m_3x250x149", 3, 250, 149, 4))


def long_text(B, lengths, seed, N=LONG_N):
    """(B, N) ids: lengths[b] characters uniform in [2, 31], then E, then P padding."""
    rng = np.random.default_rng(seed)
    L = np.zeros((B, N), np.int32)
    for b, n in enumerate(lengths):
        L[b, :n] = rng.integers(2, 32, n)
        L[b, n] = 1
    return L


def synth_inputs():
    L = long_text(len(SYNTH_PMA), SYNTH_LENGTHS, seed=4)
    mels = np.random.default_rng(5).uniform(0, 1, (len(SYNTH_PMA), hp.max_T, hp.n_mels)).astype(np.float32)
    return L, mels, np.asarray(SYNTH_PMA, np.int32)


def window_summary(alignments, pma, win=3):
    """(B, win, T) alignments of keys p..p+win-1 (zero rows past N) and (B,) max |alignment| outside the window."""
    B, N, T = alignments.shape
    aw = np.zeros((B, win, T), np.float32)
    outside = np.zeros(B, np.float32)
    for b, p in enumerate(pma):
        hi = min(p + win, N)
        aw[b, :hi - p] = alignments[b, p:hi]
        rest = np.concatenate([alignments[b, :p], alignments[b, hi:]], 0)
        outside[b] = np.abs(rest).max() if rest.size else 0.0
    return aw, outside


def train_inputs(B, N, T, seed):
    return synthetic_bucket(B, N, T, seed=seed)


def dropout_hook(seed):
    return lambda x, r_, i: x * rtr.dropout_keep(x.shape, i, seed, r_)


if __name__ == "__main__":
    tf_shim.install(tf_shim.Store(init_params(0, "perturbed")))
    import hyperparams as ref_hp                                 # noqa: E402  (the reference's, on sys.path after install)
    old_ref, old = ref_hp.Hyperparams.max_N, hp.max_N
    ref_hp.Hyperparams.max_N = hp.max_N = LONG_N
    try:
        out = {}
        L, mels, pma = synth_inputs()
        o = tf_shim.run_graph(L, mels, pma)
        aw, outside = window_summary(np.asarray(o["alignments"], np.float32), pma)
        out.update(synth_Y=o["Y"].astype(np.float32), synth_max_attentions=o["max_attentions"], synth_align_win=aw,
                   synth_align_outside=outside)
        for tag, B, N, T, seed in T2M_CASES:
            Lb, mb = train_inputs(B, N, T, seed)
            ref, ncalls = tf_shim.run_train_graph(Lb, mb, dropout_hook(seed))
            out[tag] = np.array([ref[k] for k in ("loss", "loss_mels", "loss_bd1", "loss_att")], np.float64)
            out[tag + "_ncalls"] = np.array(ncalls)
    finally:
        ref_hp.Hyperparams.max_N, hp.max_N = old_ref, old
    np.savez_compressed(os.path.join(HERE, "refshim_long_text.npz"), **out)
    print("long-text fixture written to %s" % HERE)
