"""The oracles at max_N = 300 against the reference's own code at that max_N (refshim_long_text.npz, generator
tests/golden/make_golden_refchecks_long.py): the synthesis graph with windows below, at and past key 192 and at the
window's edge (oracle/ref_torch.py and oracle/ref_numpy.py), and the Text2Mel training losses on the (300, max_T)
guided-attention table at (2, 300, 53) and at a bucket with N_b = 250 (the bucket-shape oracle tests/ref_train_bucket.py).
Where a checkout of the reference is present the same checks also run against it live.  The GPU side
(tests/test_gpu_long_text.py) compares the kernels with the same fixture and these oracles."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, golden
from dc_tts_b200.hyperparams import Hyperparams as hp
from dc_tts_b200.params import init_params
from oracle import ref_numpy as rn
from oracle import ref_torch as rt
from oracle import ref_train as rtr

import ref_train_bucket as rtb

sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_golden_refchecks_long import LONG_N, T2M_CASES, dropout_hook, synth_inputs, train_inputs, window_summary  # noqa: E402

HAVE_REF = os.path.isfile("/root/reference/train.py")
LOSSES = ("loss", "loss_mels", "loss_bd1", "loss_att")


@pytest.fixture(scope="module")
def P():
    return init_params(0, "perturbed")


@pytest.fixture(autouse=True)
def max_n_300(monkeypatch):
    monkeypatch.setattr(hp, "max_N", LONG_N)


def _check_synth(Y, M, A, g, pma, rows=slice(None)):
    assert np.abs(np.asarray(Y) - g["synth_Y"][rows]).max() < 2e-5
    assert np.array_equal(np.asarray(M), g["synth_max_attentions"][rows])
    aw, outside = window_summary(np.asarray(A, np.float32), pma)
    assert np.abs(aw - g["synth_align_win"][rows]).max() < 1e-5
    assert (outside == 0).all() and (g["synth_align_outside"][rows] == 0).all()


def test_fixture_shapes():
    g = golden("refshim_long_text.npz")
    L, mels, pma = synth_inputs()
    assert L.shape == (6, LONG_N) and g["synth_Y"].shape == (6, hp.max_T, hp.n_mels)
    assert (L[:, 192:] != 0).any(axis=1).all()                    # every text runs past key 192


def test_torch_oracle_synthesis_graph_vs_reference_at_max_n_300(P):
    g = golden("refshim_long_text.npz")
    L, mels, pma = synth_inputs()
    o = rt.text2mel_forward(P, L, mels, pma)
    _check_synth(o["Y"].numpy(), o["max_attentions"].numpy(), o["alignments"].numpy(), g, pma)


def test_numpy_oracle_synthesis_graph_vs_reference_at_max_n_300(P):
    g = golden("refshim_long_text.npz")
    L, mels, pma = synth_inputs()
    o = rn.text2mel_forward(P, L, mels, pma)
    _check_synth(o["Y"], o["max_attentions"], o["alignments"], g, pma)


def _bucket_oracle(P, B, N, T, seed):
    L, mels = train_inputs(B, N, T, seed)
    W = {n: torch.tensor(np.asarray(P[n], np.float32)) for n in rtr.text2mel_names()}
    with torch.no_grad():
        return rtb.forward(W, L, mels, seed, hp.dropout_rate)


def test_bucket_oracle_losses_vs_reference_training_graph_at_max_n_300(P):
    g = golden("refshim_long_text.npz")
    for tag, B, N, T, seed in T2M_CASES:
        o = _bucket_oracle(P, B, N, T, seed)
        for i, k in enumerate(LOSSES):
            ref = g[tag][i]
            assert abs(float(o[k]) - ref) < 2e-6 * max(1.0, abs(ref)), (tag, k, float(o[k]), ref)


@pytest.fixture
def ref_at_300(P):
    import tf_shim
    tf_shim.install(tf_shim.Store(P))
    import hyperparams as ref_hp
    old = ref_hp.Hyperparams.max_N
    ref_hp.Hyperparams.max_N = LONG_N
    yield tf_shim
    ref_hp.Hyperparams.max_N = old


@pytest.mark.skipif(not HAVE_REF, reason="/root/reference is not present on this machine")
def test_reference_live_at_max_n_300(P, ref_at_300):
    """The reference's graphs re-run at max_N = 300: the two edge windows of the synthesis case and the (2, 300, 53)
    training losses, against the fixture and the oracles."""
    g = golden("refshim_long_text.npz")
    L, mels, pma = synth_inputs()
    rows = slice(4, 6)                                    # windows at 297 and 299
    r = ref_at_300.run_graph(L[rows], mels[rows], pma[rows])
    _check_synth(r["Y"], r["max_attentions"], r["alignments"], g, pma[rows], rows)
    tag, B, N, T, seed = T2M_CASES[0]
    Lb, mb = train_inputs(B, N, T, seed)
    ref, _ = ref_at_300.run_train_graph(Lb, mb, dropout_hook(seed))
    o = _bucket_oracle(P, B, N, T, seed)
    for i, k in enumerate(LOSSES):
        assert abs(ref[k] - g[tag][i]) < 1e-12 * max(1.0, abs(ref[k])), k
        assert abs(float(o[k]) - ref[k]) < 2e-6 * max(1.0, abs(ref[k])), k
