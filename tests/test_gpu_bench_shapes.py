"""GPU parity at the shapes the benchmark runs (BASELINE configs 2, 3, 4): SSRN B=32 T=210, TextEnc B=32,
the 210-frame autoregressive loop at B=32 and B=1 -- the kernel configurations that produce the headline
numbers (conv_ln_tc_kernel<32> on launches wider than the device, the persistent cluster decode) against the
oracle.  Reference: networks.py:214-292, synthesize.py:45-57, hyperparams.py:39-47 (B=32)."""
import numpy as np
import pytest
import torch

from dc_tts_b200.hyperparams import Hyperparams as hp
from dc_tts_b200.params import synthetic_text
from oracle import ref_torch as rt

pytestmark = pytest.mark.gpu
TOL = 1e-3
B = 32


@pytest.fixture()
def default_engine(engine):
    engine.set_tensor_path(1)
    engine.set_option("decode_mode", 1)
    yield engine


def test_ssrn_config3_b32_t210(default_engine, params):
    """BASELINE config 3: every wide SSRN block runs conv_ln_tc_kernel<32> on more CTAs than the device has SMs."""
    Y = np.random.default_rng(0).uniform(0, 1, (B, hp.max_T, hp.n_mels)).astype(np.float32)
    _, Z = default_engine.ssrn(Y, want_logits=False)
    Z = Z.cpu().numpy()
    worst = 0.0
    with torch.no_grad():
        for b0 in range(0, B, 8):                                   # oracle in slabs (memory), all 32 utterances
            _, Zr = rt.SSRN(params, torch.from_numpy(Y[b0:b0 + 8]))
            worst = max(worst, float(np.abs(Z[b0:b0 + 8] - Zr.numpy()).max()))
    assert worst < TOL, worst


def test_textenc_config4_b32(default_engine, params):
    L = synthetic_text(B, 100, seed=0)
    K, V = default_engine.textenc(L)
    with torch.no_grad():
        Kr, Vr = rt.TextEnc(params, L)
    assert np.abs(K.cpu().numpy() - Kr.numpy()).max() < TOL
    assert np.abs(V.cpu().numpy() - Vr.numpy()).max() < TOL


def _oracle_rows(params, L, rows, steps):
    r = rt.synthesize(params, L[rows], steps=steps, literal=False, record=True)
    return r["Y"].numpy(), r["p_hist"].numpy(), r["margin_hist"].numpy()


def _compare_prefix(Y, P, Yo, Po, margin, steps):
    """Free-running comparison up to the first frame whose argmax feedback is a near-tie (margin < 1e-4 in
    probability): past it two correct float32 implementations may legitimately follow different windows."""
    checked = 0
    for i in range(Yo.shape[0]):
        bad = np.nonzero(margin[i] < 1e-4)[0]
        n = int(bad[0]) + 1 if bad.size else steps
        assert np.array_equal(P[i, :n], Po[i, :n]), (i, n)
        assert np.abs(Y[i, :n] - Yo[i, :n]).max() < TOL, (i, n)
        checked += n
    return checked


@pytest.mark.parametrize("decode_mode", [1, 0], ids=["cluster", "graph"])
def test_generate_config4_b32_210_frames(default_engine, params, decode_mode):
    """The benchmark's own workload (32 synthetic 100-character utterances, 210 frames, free running): four
    utterances spread over different clusters are checked against the oracle's schedule (synthesize.py:45-57)."""
    e = default_engine
    e.set_option("decode_mode", decode_mode)
    try:
        L = synthetic_text(B, 100, seed=0)
        rows = [0, 9, 18, 31]
        Y, P, _, _ = e.text2mel_generate(L)
        Yo, Po, margin = _oracle_rows(params, L, rows, hp.max_T)
        checked = _compare_prefix(Y.cpu().numpy()[rows], P.cpu().numpy()[rows], Yo, Po, margin, hp.max_T)
        assert checked >= 2 * hp.max_T                              # not everything may hide behind a tie
        if decode_mode == 1:
            frames, utt, clusters = e.decode_stats()
            # every cluster co-resident: 32 utterances go 5 per cluster when 7 clusters of 16 CTAs fit the device
            assert clusters <= e.get_option("decode_max_clusters") and 0 < utt <= B * hp.max_T and frames <= clusters * hp.max_T
            # the recompute count must equal the number of window moves of the whole batch
            Pn = P.cpu().numpy()
            assert utt == int((np.diff(Pn, axis=1) != 0).sum())
    finally:
        e.set_option("decode_mode", 1)


def test_generate_config2_b1_210_frames(default_engine, params):
    """BASELINE config 2: one utterance, all 210 frames, persistent decode (one cluster, G = 1)."""
    L = synthetic_text(1, 100, seed=0)
    Y, P, _, _ = default_engine.text2mel_generate(L)
    Yo, Po, margin = _oracle_rows(params, L, [0], hp.max_T)
    assert _compare_prefix(Y.cpu().numpy(), P.cpu().numpy(), Yo, Po, margin, hp.max_T) >= 100


@pytest.mark.parametrize("Bn", [2, 3, 5, 8, 13, 17, 23])
def test_cluster_decode_equals_graph_decode(default_engine, Bn):
    """Ragged group sizes (last cluster partly filled, 1 to 4 utterances per cluster): the persistent kernel and the
    graph-per-frame loop follow the same windows and agree to float32 re-association noise."""
    e = default_engine
    L = np.concatenate([synthetic_text(1, 30 + (11 * i) % 140, seed=100 + i) for i in range(Bn)])
    steps = 70
    Y1, P1, _, _ = e.text2mel_generate(L, steps=steps)
    e.set_option("decode_mode", 0)
    try:
        Y0, P0, _, _ = e.text2mel_generate(L, steps=steps)
    finally:
        e.set_option("decode_mode", 1)
    same = (P0 == P1).all(dim=1)                                    # a near-tie may split a trajectory; most must agree
    assert int(same.sum()) >= Bn - 1
    assert (Y0[same] - Y1[same]).abs().max().item() < 1e-4
    assert (Y1[:, steps:] == 0).all()
