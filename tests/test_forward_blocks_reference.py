"""CPU pins of tests/ref_forward_blocks.py, the float64 block references of the full-sequence block tests
(tests/test_gpu_forward_blocks.py): every block kind, both paddings and the transposed conv against oracle/ref_numpy.py in
float64; the ragged mode against the oracle run on each utterance alone; the dense attention against the oracle; and the
error scales S against a float32 restatement (well inside tau S: S is neither vacuous nor too tight)."""
import numpy as np
import pytest

import ref_decode_blocks as rb
import ref_forward_blocks as rf
from dc_tts_b200.arch import NETWORKS
from dc_tts_b200.hyperparams import Hyperparams as hp
from oracle import ref_numpy as rn
from dc_tts_b200.params import init_params


@pytest.fixture(scope="module")
def P():
    return init_params(0, "perturbed")


def _input(cin, B, L, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((B, L, cin))
    return np.abs(x) if cin == hp.n_mels else x


def _oracle_block(P, net, l, x):
    s = "%s/%s" % (net, l.scope)
    x = np.asarray(x, np.float64)
    if l.kind == "HC":
        return rn.hc(P, x, s, l.rate, l.pad)
    if l.kind == "D":
        return rn.conv1d_transpose(P, x, s)
    return rn.conv1d(P, x, s, l.rate, l.pad, l.act)


def _close(got, want, what):
    assert np.abs(got - want).max() <= 1e-12 * max(1.0, np.abs(want).max()), what


@pytest.mark.parametrize("net", list(NETWORKS))
def test_blocks_match_the_oracle(P, net):
    """Every block of every network (SAME and causal convs at dilations 1-27, highway blocks, the transposed convs) on all
    rows of two utterances, and on a subset of rows, at 1e-12; S bounds |out| (the error scale carries the value's size)."""
    layers = NETWORKS[net]()
    for i, l in enumerate(layers):
        x = _input(l.cin, 2, 23, i)
        want = _oracle_block(P, net, l, x)
        p = rf.block_params(P, net, l)
        Lout = want.shape[1]
        for b in range(2):
            got, S = rf.block_rows(p, l, x[b], np.arange(Lout))
            _close(got, want[b], l.scope)
            assert (S > 0).all() and (S >= np.abs(got) - 1e-12).all(), l.scope
        rows = np.array([0, 1, Lout // 2, Lout - 2, Lout - 1])
        got, _ = rf.block_rows(p, l, x[1], rows)
        _close(got, want[1][rows], l.scope + " (row subset)")


def test_extra_shift_is_the_shifted_feed(P):
    """AudioEnc's first block with extra_shift = -1 on mels is the block on the mels read one frame back (train.py:51)."""
    from dc_tts_b200.arch import audioenc_layers
    l = audioenc_layers()[0]
    p = rf.block_params(P, "Text2Mel/AudioEnc", l)
    x = _input(l.cin, 1, 30, 5)[0]
    got, _ = rf.block_rows(p, l, x, np.arange(30), extra_shift=-1)
    want = _oracle_block(P, "Text2Mel/AudioEnc", l, rb.shifted_feed(x)[None])[0]
    _close(got, want, "extra_shift")
    assert rf.tap_shifts(l, -1) == [-1]


def test_tap_shifts():
    """The shifts api_synth.cu computes: SAME centres the taps (left = (k - 1) rate / 2), causal ends them at the row."""
    from collections import namedtuple
    Lay = namedtuple("Lay", "size rate pad")
    assert rf.tap_shifts(Lay(3, 9, "SAME")) == [-9, 0, 9]
    assert rf.tap_shifts(Lay(3, 27, "CAUSAL")) == [-54, -27, 0]
    assert rf.tap_shifts(Lay(1, 1, "SAME")) == [0]
    assert rf.tap_shifts(Lay(3, 3, "CAUSAL"), -1) == [-7, -4, -1]


@pytest.mark.parametrize("net", ["SSRN", "Text2Mel/AudioDec"])
def test_ragged_mode_is_each_utterance_alone(P, net):
    """Utterance b's chain on its live rows (n_b 2^(transposed convs before the block)) is the oracle's chain on that
    utterance alone, x[b, :n_b]; the rows past them are what the kernels store as zeros."""
    layers = NETWORKS[net]()
    L, n = 12, [1, 5, 12]
    x = _input(layers[0].cin, len(n), L, 3)
    for b, nb in enumerate(n):
        want = rn.run_chain(P, x[b:b + 1, :nb].astype(np.float64), net, layers)[0]
        ins, outs = rf.live_rows(layers, nb)
        cur = np.zeros((L, layers[0].cin))
        cur[:nb] = x[b, :nb]
        for i, l in enumerate(layers):
            got, _ = rf.block_rows(rf.block_params(P, net, l), l, cur[:ins[i]], np.arange(outs[i]))
            cur = np.zeros((outs[i] * L // nb, l.cout))
            cur[:outs[i]] = got
        _close(cur[:outs[-1]], want, "%s utterance %d" % (net, b))
    assert rf.live_rows(NETWORKS["SSRN"](), 3) == ([3] * 4 + [6] * 3 + [12] * 9, [3] * 3 + [6] * 3 + [12] * 10)


def test_dense_attention_matches_the_oracle():
    rng = np.random.default_rng(4)
    T, d, N = 21, hp.d, 37
    Q = rng.standard_normal((1, T, d))
    K, V = rng.standard_normal((1, N, d)), rng.standard_normal((1, N, d))
    R, A, M = rn.Attention(Q, K, V)
    r = rf.dense_attention(Q[0], np.concatenate([K[0], V[0]], 1))
    assert np.abs(r["R"] - R[0]).max() < 1e-12
    assert np.abs(r["A"] - A[0].T).max() < 1e-12
    assert np.array_equal(r["argmax"], M[0])
    assert (r["SA"] >= r["A"]).all()


def test_split_planes():
    x = np.array([1.0, 1 / 3, 1e-3, 3e-6, -7.25e3, 0.0], np.float32)
    hi, lo = rf.split_f16(x)
    assert np.array_equal(hi, x.astype(np.float16))
    j = hi.astype(np.float32) + lo.astype(np.float32)
    assert (np.abs(j - x) <= np.maximum(np.abs(x) * 2.0 ** -22, 2.0 ** -25)).all()


@pytest.mark.parametrize("net", list(NETWORKS))
def test_error_scale_bounds_a_float32_restatement(P, net):
    """The float32 restatement of every conv / highway block of the network lands below tau_fp32 / 4 of S, so S is a valid
    bound for float32 arithmetic with room for the kernels' summation orders; and above tau_fp32 / 1000 somewhere, so S is
    not vacuous."""
    layers = [l for l in NETWORKS[net]() if l.kind != "D"]
    worst = 0.0
    for i, l in enumerate(layers):
        x = _input(l.cin, 1, 50, 200 + i)[0].astype(np.float32)
        p = rf.block_params(P, net, l)
        ref, S = rf.block_rows(p, l, x, np.arange(50))
        got = rb.float32_block(p, l, x, np.arange(50), rf.tap_shifts(l))
        worst = max(worst, float((np.abs(got - ref) / S).max()))
    assert rf.TAU_FP32 / 1000 < worst < rf.TAU_FP32 / 4, worst


def test_deconv_scale_bounds_a_float32_restatement(P):
    from dc_tts_b200.arch import ssrn_layers
    l = [l for l in ssrn_layers() if l.kind == "D"][0]
    p = rf.block_params(P, "SSRN", l)
    x = _input(l.cin, 1, 40, 9)[0].astype(np.float32)
    ref, S = rf.block_rows(p, l, x, np.arange(80))
    got = rn.conv1d_transpose(P, x[None], "SSRN/" + l.scope)[0]       # the oracle in float32
    r = float((np.abs(got - ref) / S).max())
    assert rf.TAU_FP32 / 1000 < r < rf.TAU_FP32 / 4, r


def test_attention_scale_bounds_a_float32_restatement():
    rng = np.random.default_rng(11)
    T, d, N = 40, hp.d, hp.max_N
    Q = rng.standard_normal((T, d)).astype(np.float32)
    KV = (3 * rng.standard_normal((N, 2 * d))).astype(np.float32)
    r = rf.dense_attention(Q, KV)
    f = np.float32
    s = (Q @ KV[:, :d].T) * f(1 / np.sqrt(d))
    e = np.exp(s - s.max(1, keepdims=True))
    A = e / e.sum(1, keepdims=True)
    got = A @ KV[:, d:]
    assert (np.abs(got - r["R"][:, :d]) / r["S"][:, :d]).max() < rf.TAU_ATTN_FP32 / 4
    # the probabilities carry the 256-term score sums' rounding at full gain: half of tau, not a quarter
    assert (np.abs(A - r["A"]) / r["SA"]).max() < rf.TAU_ATTN_FP32 / 2
