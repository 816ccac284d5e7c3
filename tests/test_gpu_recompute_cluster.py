"""The receptive-field recompute of the persistent decode with 2 to 5 utterances per cluster.  Every A slab of the
recompute is fetched once per cluster and multicast to its 16 CTAs, and a stage is refilled only when all 16 have
multiplied it, so the slab sequence must stay in step across the CTAs however many utterances of a cluster move in a
frame.  Forced (every utterance at every frame) and natural (moved and unmoved utterances interleaved in a cluster)."""
import numpy as np
import pytest

from dc_tts_b200.hyperparams import Hyperparams as hp
from dc_tts_b200.params import synthetic_text
from oracle import ref_torch as rt
from test_gpu_bench_shapes import _compare_prefix  # the near-tie rule of the benchmark-shape tests

pytestmark = pytest.mark.gpu


@pytest.fixture
def cluster_engine(engine):
    engine.set_tensor_path(1)
    engine.set_option("decode_mode", 1)
    yield engine
    engine.set_option("decode_force_prepass", 0)
    engine.set_option("decode_mode", 1)


def _graph_decode(e, L, steps):
    e.set_option("decode_mode", 0)
    try:
        return e.text2mel_generate(L, steps=steps)
    finally:
        e.set_option("decode_mode", 1)


def _per_cluster(B, clusters):
    G = -(-B // clusters)
    return G, [list(range(c * G, min(B, (c + 1) * G))) for c in range(clusters)]


@pytest.mark.parametrize("B", [14, 21, 28, 32])
def test_forced_recompute_utterances_per_cluster(cluster_engine, params, B):
    """On a device with seven 16-CTA clusters (H100 SXM) these batches run 2, 3, 4 and 5 utterances per cluster, all
    recomputing at every frame: cluster 0 against the oracle, the whole batch against the graph-per-frame decode."""
    e = cluster_engine
    steps = 120                                                     # past j = 96: recomputes before and after t = 0 leaves the window
    L = synthetic_text(B, 100, seed=0)
    e.set_option("decode_force_prepass", 1)
    try:
        Y, P, _, _ = e.text2mel_generate(L, steps=steps)
        frames, utt, clusters = e.decode_stats()
    finally:
        e.set_option("decode_force_prepass", 0)
    assert utt == B * (steps - 1) and frames == clusters * (steps - 1), (frames, utt, clusters)
    _, groups = _per_cluster(B, clusters)
    rows = groups[0]
    r = rt.synthesize(params, L[rows], steps=steps, literal=False, record=True)
    checked = _compare_prefix(Y.cpu().numpy()[rows], P.cpu().numpy()[rows, :steps], r["Y"].numpy(), r["p_hist"].numpy(),
                              r["margin_hist"].numpy(), steps)
    assert checked >= min(len(rows), 2) * 60                        # not everything may hide behind a tie
    Y0, P0, _, _ = _graph_decode(e, L, steps)
    same = (P0 == P).all(dim=1)
    assert int(same.sum()) >= B - 1
    assert (Y0[same] - Y[same]).abs().max().item() < 1e-4


@pytest.mark.parametrize("B", [21, 32])
def test_natural_moves_interleaved(cluster_engine, B):
    """Texts of mixed lengths: in most frames with a move only some utterances of a cluster move.  The recompute counts
    must equal the window moves (per utterance, and per cluster-frame with any move), and the output must match the
    graph-per-frame decode."""
    e = cluster_engine
    L = np.concatenate([synthetic_text(1, 30 + (11 * i) % 140, seed=100 + i) for i in range(B)])
    Y, P, _, _ = e.text2mel_generate(L)
    frames, utt, clusters = e.decode_stats()
    moved = np.diff(P.cpu().numpy()[:, :hp.max_T], axis=1) != 0     # (B, T - 1): frame j >= 1 moved its window
    _, groups = _per_cluster(B, clusters)
    assert utt == int(moved.sum())
    assert frames == sum(int(moved[g].any(axis=0).sum()) for g in groups)
    mixed = sum(int((moved[g].any(axis=0) & ~moved[g].all(axis=0)).sum()) for g in groups if len(g) > 1)
    assert mixed > 0                                                # frames in which moved and unmoved utterances share a cluster
    Y0, P0, _, _ = _graph_decode(e, L, hp.max_T)
    same = (P0 == P).all(dim=1)
    assert int(same.sum()) >= B - 1
    assert (Y0[same] - Y[same]).abs().max().item() < 1e-4
