"""Generates refshim_train_bucket.npz: the losses of the reference's OWN training graphs (train.py Graph(num, mode="train"),
executed under the TensorFlow API stand-in of tf_shim.py) on length-bucketed batches at their own shapes, as the
reference's get_batch (data_load.py:122-129, dynamic_pad=True) feeds them:
    t2m_37x53_drop / _nodrop   Text2Mel, B = 2, N = 37, T = 53, with (seed 11) and without the shared dropout mask
    t2m_120x171_drop           Text2Mel, B = 2, N = 120, T = 171, dropout seed 5
    ssrn_T9 / ssrn_T53         SSRN, B = 2, mels (2, T, n_mels), mags (2, 4T, F), dropout seed 9
The inputs are the ones tests/test_train_bucketed.py regenerates from the same seeds (params.synthetic_bucket).  Needs a
checkout of the reference at tf_shim.REFERENCE; run from the repo root:
    python tests/golden/make_golden_refchecks_bucket.py
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

T2M_CASES = (("t2m_37x53_drop", 37, 53, 11, hp.dropout_rate), ("t2m_37x53_nodrop", 37, 53, 0, 0.0),
             ("t2m_120x171_drop", 120, 171, 5, hp.dropout_rate))
SSRN_CASES = (("ssrn_T9", 9), ("ssrn_T53", 53))


def ssrn_batch(T):
    mels = np.random.default_rng(3).uniform(0, 1, (2, T, hp.n_mels)).astype(np.float32)
    mags = np.random.default_rng(4).uniform(0, 1, (2, 4 * T, 1 + hp.n_fft // 2)).astype(np.float32)
    return mels, mags


if __name__ == "__main__":
    tf_shim.install(tf_shim.Store(init_params(0, "perturbed")))
    import hyperparams as ref_hp                                 # noqa: E402  (the reference's, on sys.path after install)
    out = {}
    for tag, N, T, seed, rate in T2M_CASES:
        L, mels = synthetic_bucket(2, N, T, seed=7)
        ref_hp.Hyperparams.dropout_rate = rate
        try:
            ref, ncalls = tf_shim.run_train_graph(L, mels, lambda x, r_, i, s=seed: x * rtr.dropout_keep(x.shape, i, s, r_))
        finally:
            ref_hp.Hyperparams.dropout_rate = hp.dropout_rate
        out[tag] = np.array([ref[k] for k in ("loss", "loss_mels", "loss_bd1", "loss_att")], np.float64)
        out[tag + "_ncalls"] = np.array(ncalls)
    for tag, T in SSRN_CASES:
        mels, mags = ssrn_batch(T)
        ref, ncalls = tf_shim.run_train_graph_ssrn(mels, mags, lambda x, r_, i: x * rtr.dropout_keep(x.shape, i, 9, r_))
        out[tag] = np.array([ref[k] for k in ("loss", "loss_mags", "loss_bd2")], np.float64)
        out[tag + "_ncalls"] = np.array(ncalls)
    np.savez_compressed(os.path.join(HERE, "refshim_train_bucket.npz"), **out)
    print("bucketed training-graph fixture written to %s" % HERE)
