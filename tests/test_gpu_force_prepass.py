"""The receptive-field recompute of the persistent decode in its worst case: option decode_force_prepass makes every
utterance take it at every frame j >= 1, as if its attention window had moved.  The reference recomputes the whole
receptive field every frame (quirk Q1, synthesize.py:45-54), so the output must not change.  This covers what the
natural window moves reach only by chance: recomputes at j < 96 (source rows before the utterance start, TF's causal
zero padding) and five utterances of one cluster recomputing in the same frame."""
import numpy as np
import pytest

from dc_tts_b200.hyperparams import Hyperparams as hp
from dc_tts_b200.params import synthetic_text
from oracle import ref_torch as rt
from test_gpu_bench_shapes import _compare_prefix  # the near-tie rule of the benchmark-shape tests

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B,rows", [(32, [0, 1, 2, 3, 4]), (1, [0])], ids=["b32_full_cluster", "b1"])
def test_forced_recompute_every_frame(engine, params, B, rows):
    """B = 1 runs one utterance in one cluster.  The host gives each cluster the fewest utterances that keep every cluster
    co-resident, so five utterances share a cluster only when the batch needs it: B = 32 on a device with seven 16-CTA
    clusters (H100 SXM) runs five per cluster, and rows 0..4 are cluster 0, all recomputing together.  (B = 5 would run
    one utterance per cluster.)"""
    e = engine
    e.set_tensor_path(1)
    e.set_option("decode_mode", 1)
    e.set_option("decode_force_prepass", 1)
    try:
        L = synthetic_text(B, 100, seed=0)
        Y, P, _, _ = e.text2mel_generate(L)
        frames, utt, clusters = e.decode_stats()
    finally:
        e.set_option("decode_force_prepass", 0)
    steps = hp.max_T
    assert utt == B * (steps - 1), (utt, B)
    assert frames == clusters * (steps - 1), (frames, clusters)
    if B == 32 and clusters == 7:
        assert -(-B // clusters) == len(rows)                     # rows 0..4 fill cluster 0
    r = rt.synthesize(params, L[rows], steps=steps, literal=False, record=True)
    Yo, Po, margin = r["Y"].numpy(), r["p_hist"].numpy(), r["margin_hist"].numpy()
    checked = _compare_prefix(Y.cpu().numpy()[rows], P.cpu().numpy()[rows], Yo, Po, margin, steps)
    assert checked >= min(len(rows), 2) * 100                      # not everything may hide behind a tie
