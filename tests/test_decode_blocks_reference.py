"""CPU pins of tests/ref_decode_blocks.py, the float64 block references of the decode's block tests
(tests/test_gpu_decode_blocks.py): each block against oracle/ref_numpy.py run in float64, the blocks chained frame by frame
along a window path against tests/ref_window_path.forced_path, and the error scales S against a float32 restatement."""
import numpy as np
import pytest

import ref_decode_blocks as rb
from dc_tts_b200.arch import audiodec_layers, audioenc_layers
from dc_tts_b200.hyperparams import Hyperparams as hp
from dc_tts_b200.params import init_params, synthetic_text
from oracle import ref_numpy as rn

ENC, DEC = "Text2Mel/AudioEnc", "Text2Mel/AudioDec"


@pytest.fixture(scope="module")
def P():
    return init_params(0, "perturbed")


def _input(layer, T, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((T, layer.cin))
    return np.abs(x) if layer.cin == hp.n_mels else x           # mel inputs are in [0, 1]-like ranges; any sign elsewhere


def _oracle_block(P, net, layer, x):
    s = "%s/%s" % (net, layer.scope)
    x = x[None].astype(np.float64)
    if layer.kind == "HC":
        return rn.hc(P, x, s, layer.rate, "CAUSAL")[0]
    return rn.conv1d(P, x, s, layer.rate, "CAUSAL", layer.act)[0]


@pytest.mark.parametrize("net", [ENC, DEC])
def test_blocks_match_the_oracle(P, net):
    """Every AudioEnc and AudioDec block on all rows of a 40-row input, and on a trailing window of rows, at 1e-12."""
    layers = audioenc_layers() if net == ENC else audiodec_layers()
    for i, l in enumerate(layers):
        x = _input(l, 40, i)
        want = _oracle_block(P, net, l, x)
        got, S = rb.block(rb.block_params(P, net, l), l, x, np.arange(40))
        assert np.abs(got - want).max() <= 1e-12 * max(1.0, np.abs(want).max()), l.scope
        assert (S > 0).all() and (S >= np.abs(got) - 1e-12).all(), l.scope
        tail, _ = rb.block(rb.block_params(P, net, l), l, x, np.arange(25, 40))
        assert np.abs(tail - want[25:]).max() <= 1e-12 * max(1.0, np.abs(want).max()), l.scope


@pytest.mark.parametrize("p", [0, 7, hp.max_N - 3, hp.max_N - 2, hp.max_N - 1])
def test_attention_rows_match_the_oracle(P, p):
    """Monotonic attention under one window for every row, the windows at the end of the text with fewer live keys
    included: R, the argmax and the top-2 margin at 1e-12."""
    rng = np.random.default_rng(p)
    T, d, N = 12, hp.d, hp.max_N
    Q, K, V = rng.standard_normal((1, T, d)), rng.standard_normal((1, N, d)), rng.standard_normal((1, N, d))
    R, A, M = rn.Attention(Q, K, V, True, [p])
    r = rb.attention_rows(Q[0], np.concatenate([K[0], V[0]], 1), np.full(T, p), hp.attention_win_size)
    assert np.abs(r["R"] - R[0]).max() < 1e-12
    assert np.array_equal(r["argmax"], M[0])
    a = np.sort(A[0].T, axis=1)
    live = min(N, p + hp.attention_win_size) - p
    if live > 1:
        assert np.abs(r["margin"] - (a[:, -1] - a[:, -2])).max() < 1e-12
    else:
        assert np.isinf(r["margin"]).all()


def test_sigmoid_and_shifted_feed():
    x = np.linspace(-30, 30, 601)[:, None]
    y, S = rb.mel_sigmoid(x)
    assert np.abs(y - 1 / (1 + np.exp(-x))).max() < 1e-15 and (S >= y).all()
    Y = np.arange(12.0).reshape(4, 3)
    f = rb.shifted_feed(Y)
    assert not f[0].any() and np.array_equal(f[1:], Y[:-1])
    mels = Y[None]
    assert np.array_equal(f, np.concatenate((np.zeros_like(mels[:, :1]), mels[:, :-1]), 1)[0])   # rn.text2mel_forward's S


def _decode_along(P, L, path, steps):
    """The references chained frame by frame along `path` for one utterance, the AudioDec receptive field recomputed under
    each frame's window (the reference's full recompute restricted to the rows that reach Y[j])."""
    K, V = rn.TextEnc(P, L[None], np.float64)
    KV = np.concatenate([K[0], V[0]], 1)
    enc, dec = audioenc_layers(), audiodec_layers()
    pe = [rb.block_params(P, ENC, l) for l in enc]
    pd = [rb.block_params(P, DEC, l) for l in dec]
    rows = rb.audiodec_rows(dec, hp.max_T)
    T = hp.max_T
    Y = np.zeros((T, hp.n_mels))
    ae = [np.zeros((T, l.cout)) for l in enc]
    amax, margin = [], []
    for j in range(steps):
        x = rb.shifted_feed(Y)
        for i, l in enumerate(enc):
            ae[i][j] = rb.block(pe[i], l, x, [j])[0][0]
            x = ae[i]
        lo = max(0, j - rows[0] + 1)
        win = np.full(j + 1 - lo, path[j])
        a = rb.attention_rows(ae[-1][lo:j + 1], KV, win, hp.attention_win_size)
        amax.append(a["argmax"][-1])
        margin.append(a["margin"][-1])
        x = np.zeros((T, 2 * hp.d))
        x[lo:j + 1] = a["R"]
        for i, l in enumerate(dec):
            out = np.zeros((T, l.cout))
            r = np.arange(max(0, j - rows[i] + 1), j + 1)
            out[r] = rb.block(pd[i], l, x, r)[0]
            x = out
        Y[j] = rb.mel_sigmoid(x[j])[0]
    return Y, np.array(amax), np.array(margin)


def test_chained_references_follow_the_forced_path(P):
    """Frame by frame along a path with moves, a jump and a window at the end of the text: Y, the argmax and the margin of
    the float32 oracle's full recompute per frame (ref_window_path.forced_path), within float32 rounding."""
    import ref_window_path as rw
    L = synthetic_text(1, 60, seed=3)
    N, W = hp.max_N, hp.attention_win_size
    path = np.array([[0, 0, 1, 1, 9, 9, 2, N - W, N - 1, 4]])
    steps = path.shape[1]
    r = rw.forced_path(P, L, path)
    Y, amax, margin = _decode_along(P, L[0], path[0], steps)
    assert np.abs(Y[:steps] - r["Y"][0, :steps]).max() < 2e-5
    assert not r["Y"][0, steps:].any()
    sure = r["margin"][0] > 1e-4
    assert sure.sum() >= steps - 2 and np.array_equal(amax[sure], r["argmax"][0][sure])
    assert np.abs(margin - r["margin"][0])[np.isfinite(margin)].max() < 1e-5


@pytest.mark.parametrize("net", [ENC, DEC])
def test_error_scale_bounds_a_float32_restatement(P, net):
    """The float32 restatement of every block stays below TAU_FP32 / 4 of S on the test inputs, so S is a valid bound
    for float32 arithmetic with room for the kernels' other summation orders."""
    layers = audioenc_layers() if net == ENC else audiodec_layers()
    worst = 0.0
    for i, l in enumerate(layers):
        x = _input(l, 60, 100 + i).astype(np.float32)
        p = rb.block_params(P, net, l)
        ref, S = rb.block(p, l, x, np.arange(60))
        got = rb.float32_block(p, l, x, np.arange(60))
        worst = max(worst, float((np.abs(got - ref) / S).max()))
    assert worst < rb.TAU_FP32 / 4, worst


def test_attention_scale_bounds_a_float32_restatement():
    rng = np.random.default_rng(9)
    T, d, N = 40, hp.d, hp.max_N
    Q = rng.standard_normal((T, d)).astype(np.float32)
    KV = (3 * rng.standard_normal((N, 2 * d))).astype(np.float32)
    win = rng.integers(0, N, T)
    r = rb.attention_rows(Q, KV, win, hp.attention_win_size)
    f = np.float32
    got = np.zeros((T, d), f)
    for i in range(T):
        lo, hi = rb.window_keys(win[i], N, hp.attention_win_size)
        s = (KV[lo:hi, :d] @ Q[i]) * f(1 / np.sqrt(d))
        e = np.exp(s - s.max())
        got[i] = (e / e.sum()) @ KV[lo:hi, d:]
    assert (np.abs(got - r["R"][:, :d]) / r["S"][:, :d]).max() < rb.TAU_FP32 / 4
