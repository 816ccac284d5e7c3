"""Generates refshim_summaries.npz: the summaries the reference's OWN training graphs register (train.py Graph(num,
mode="train"), executed under the TensorFlow API stand-in of tf_shim.py with tf.summary.scalar / tf.summary.image replaced
by recorders), on fixed batches fed the way tf_shim.run_train_graph feeds them, with the hash dropout mask:
    t2m_*    Text2Mel, L / mels = params.synthetic_bucket(2, 37, 53, seed=7), dropout seed 11
    ssrn_*   SSRN, mels / mags = make_golden_refchecks_bucket.ssrn_batch(9), dropout seed 9
For each graph: `<g>_tags` (every registered tag, in registration order), `<g>_value_<i>` (the scalar or image tensor of
tag i) and the graph's alignments and Y (Text2Mel) or Z (SSRN).  This pins which tags exist and which tensor each one
shows.  Needs a checkout of the reference at tf_shim.REFERENCE; run from the repo root:
    python tests/golden/make_golden_refchecks_summaries.py
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
from make_golden_refchecks_bucket import ssrn_batch              # noqa: E402
from oracle import ref_train as rtr                              # noqa: E402

T2M_SHAPE, T2M_SEED = (2, 37, 53), 11
SSRN_T, SSRN_SEED = 9, 9


def t2m_batch():
    return synthetic_bucket(*T2M_SHAPE, seed=7)


def _graph(num, batch, seed, recorded):
    """train.Graph(num, mode="train") on `batch` (what get_batch returns), as tf_shim.run_train_graph builds it."""
    import train as ref_train
    tf_shim._State.scope = []
    tf_shim._State.layer_counts = {}
    tf_shim._State.dropout_hook = lambda x, r_, i: x * rtr.dropout_keep(x.shape, i, seed, r_)
    tf_shim._State.dropout_calls = 0
    del recorded[:]
    real = ref_train.get_batch
    ref_train.get_batch = lambda: batch
    try:
        return ref_train.Graph(num=num, mode="train")
    finally:
        ref_train.get_batch = real
        tf_shim._State.dropout_hook = None


if __name__ == "__main__":
    tf = tf_shim.install(tf_shim.Store(init_params(0, "perturbed")))
    recorded = []
    tf.summary.scalar = lambda name, tensor, **k: recorded.append((name, np.asarray(tensor, np.float64)))
    tf.summary.image = lambda name, tensor, **k: recorded.append((name, np.asarray(tensor, np.float32)))
    out = {}
    L, mels = t2m_batch()
    g = _graph(1, (tf_shim._t(L), tf_shim._t(mels), None, None, 1), T2M_SEED, recorded)
    out["t2m_alignments"], out["t2m_Y"] = np.asarray(g.alignments, np.float32), np.asarray(g.Y, np.float32)
    out["t2m_tags"] = np.array([t for t, _ in recorded])
    for i, (_, v) in enumerate(recorded):
        out["t2m_value_%d" % i] = v
    mels, mags = ssrn_batch(SSRN_T)
    g = _graph(2, (tf_shim._t(np.zeros((len(mels), 4), np.int32)), tf_shim._t(mels), tf_shim._t(mags), None, 1), SSRN_SEED, recorded)
    out["ssrn_Z"] = np.asarray(g.Z, np.float32)
    out["ssrn_tags"] = np.array([t for t, _ in recorded])
    for i, (_, v) in enumerate(recorded):
        out["ssrn_value_%d" % i] = v
    np.savez_compressed(os.path.join(HERE, "refshim_summaries.npz"), **out)
    print("summary fixture written to %s: %s" % (HERE, {k: v.shape for k, v in out.items()}))
