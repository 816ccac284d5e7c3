"""Generates refshim_train_overcap.npz: the losses of the reference's OWN training graphs (train.py Graph(num, mode="train"),
executed under the TensorFlow API stand-in of tf_shim.py) at the stock max_N = 180, max_T = 210 on batches LONGER than
that, which the reference trains as they come (data_load.py:122-129 caps nothing; train.py:91-95 pads the alignments with
-1 to (max_N, max_T) and crops them to it, so the guided-attention loss covers the table's corner only):
    t2m_2x187x53_drop / _nodrop     Text2Mel, N_b = 187 > max_N
    t2m_2x60x233_drop / _nodrop     Text2Mel, T_b = 233 > max_T
    t2m_3x200x240_drop / _nodrop    Text2Mel, both past the table
    ssrn_T233                       SSRN, mels (2, 233, n_mels), mags (2, 932, F)
"_drop" cases use the shared dropout mask of oracle/ref_train.dropout_keep (the case's seed), "_nodrop" dropout_rate 0.
The inputs are regenerated from the seeds below by tests/test_overcap_reference.py and tests/test_gpu_train_overcap.py.
Needs a checkout of the reference at tf_shim.REFERENCE; run from the repo root:
    python tests/golden/make_golden_refchecks_overcap.py
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

SHAPES = ((2, 187, 53, 11), (2, 60, 233, 5), (3, 200, 240, 4))
T2M_CASES = tuple(("t2m_%dx%dx%d_%s" % (B, N, T, tag), B, N, T, seed if rate else 0, rate)
                  for B, N, T, seed in SHAPES for tag, rate in (("drop", hp.dropout_rate), ("nodrop", 0.0)))
SSRN_T = 233


def train_inputs(B, N, T):
    return synthetic_bucket(B, N, T, seed=N + T)


def ssrn_batch(T):
    mels = np.random.default_rng(3).uniform(0, 1, (2, T, hp.n_mels)).astype(np.float32)
    mags = np.random.default_rng(4).uniform(0, 1, (2, 4 * T, 1 + hp.n_fft // 2)).astype(np.float32)
    return mels, mags


def dropout_hook(seed):
    return lambda x, r_, i: x * rtr.dropout_keep(x.shape, i, seed, r_)


if __name__ == "__main__":
    tf_shim.install(tf_shim.Store(init_params(0, "perturbed")))
    import hyperparams as ref_hp                                 # noqa: E402  (the reference's, on sys.path after install)
    assert (ref_hp.Hyperparams.max_N, ref_hp.Hyperparams.max_T) == (180, 210) == (hp.max_N, hp.max_T)
    out = {}
    for tag, B, N, T, seed, rate in T2M_CASES:
        L, mels = train_inputs(B, N, T)
        ref_hp.Hyperparams.dropout_rate = rate
        try:
            ref, ncalls = tf_shim.run_train_graph(L, mels, dropout_hook(seed))
        finally:
            ref_hp.Hyperparams.dropout_rate = hp.dropout_rate
        out[tag] = np.array([ref[k] for k in ("loss", "loss_mels", "loss_bd1", "loss_att")], np.float64)
        out[tag + "_ncalls"] = np.array(ncalls)
    mels, mags = ssrn_batch(SSRN_T)
    ref, ncalls = tf_shim.run_train_graph_ssrn(mels, mags, dropout_hook(9))
    out["ssrn_T%d" % SSRN_T] = np.array([ref[k] for k in ("loss", "loss_mags", "loss_bd2")], np.float64)
    out["ssrn_T%d_ncalls" % SSRN_T] = np.array(ncalls)
    np.savez_compressed(os.path.join(HERE, "refshim_train_overcap.npz"), **out)
    print("over-capacity training-graph fixture written to %s" % HERE)
