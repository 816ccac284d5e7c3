"""MCD-DTW on the GPU (Engine.mcd_dtw, include/dctts.h: dctts_mcd_dtw) against the float64 restatement tests/ref_mcd.py
on the host copies of the same inputs: values within 1e-9 relative, paths and pair counts identical where the reference
reports no near-tie, the tie order on repeated frames, both the shared-memory and the global-memory route, ragged
batches bit for bit against each pair alone, the refusals, and no side effects on synthesis."""
import ctypes as C

import numpy as np
import pytest
import torch

import ref_mcd
from dc_tts_b200.engine import DcttsError

pytestmark = pytest.mark.gpu

RTOL = 1e-9
NEAR_TIE = 1e-9


def _run(e, X, nx, Y, ny, K=24):
    mcd, pairs, path = e.mcd_dtw(torch.from_numpy(X).cuda(), nx, torch.from_numpy(Y).cuda(), ny, K=K, want_path=True)
    return mcd.cpu().numpy(), pairs.cpu().numpy(), path.cpu().numpy()


def _check(e, X, nx, Y, ny, K=24, paths=True):
    mcd, pairs, path = _run(e, X, nx, Y, ny, K)
    ref = ref_mcd.mcd_batch(X, nx, Y, ny, K)
    np.testing.assert_allclose(mcd, ref["mcd"], rtol=RTOL, atol=1e-12)
    if paths:
        for b in range(len(nx)):
            if ref["margin"][b] > NEAR_TIE * max(1.0, ref["mcd"][b] * ref["pairs"][b]):
                assert pairs[b] == ref["pairs"][b], b
                np.testing.assert_array_equal(path[b], ref["path"][b])
    return mcd, pairs, path, ref


def _mels(rng, *shape):
    return rng.uniform(0, 1, shape).astype(np.float32)


@pytest.mark.parametrize("K", [24, 1, 79, 13])
def test_random_pairs_against_reference(engine, K):
    rng = np.random.default_rng(K)
    B, Tx, Ty = 6, 57, 43
    X, Y = _mels(rng, B, Tx, 80), _mels(rng, B, Ty, 80)
    nx = rng.integers(1, Tx + 1, B); nx[0] = Tx
    ny = rng.integers(1, Ty + 1, B); ny[1] = Ty
    _, pairs, path, ref = _check(e=engine, X=X, nx=nx, Y=Y, ny=ny, K=K)
    assert (ref["margin"] > 1e-6).sum() >= B - 1         # the inputs are (nearly all) tie-free, so the paths were compared
    for b in range(B):
        assert (path[b, pairs[b]:] == -1).all()


def test_tie_order_on_repeated_frames(engine):
    rng = np.random.default_rng(5)
    a, b, c = _mels(rng, 3, 80)
    seqs = [([a, a, a, b], [a, b, b]), ([a, b, b, c], [a, a, b, c, c]), ([a, a], [a, a, a]), ([b, a, a, b], [b, a, b]),
            ([a, a, a], [a]), ([c, c, b, b, a], [c, b, a, a])]
    Tx, Ty = max(len(s) for s, _ in seqs), max(len(s) for _, s in seqs)
    X, Y = np.zeros((len(seqs), Tx, 80), np.float32), np.zeros((len(seqs), Ty, 80), np.float32)
    nx, ny = [], []
    for k, (s, t) in enumerate(seqs):
        X[k, :len(s)], Y[k, :len(t)] = s, t
        nx.append(len(s)); ny.append(len(t))
    mcd, pairs, path = _run(engine, X, nx, Y, ny)
    ref = ref_mcd.mcd_batch(X, nx, Y, ny)
    np.testing.assert_array_equal(pairs, ref["pairs"])
    np.testing.assert_array_equal(path, ref["path"])
    np.testing.assert_allclose(mcd, ref["mcd"], rtol=RTOL, atol=1e-12)
    # (a a a b) against (a b b): the zero-cost cells (0..2, 0) first, then (3, 1), (3, 2)
    np.testing.assert_array_equal(path[0, :pairs[0]], [[0, 0], [1, 0], [2, 0], [3, 1], [3, 2]])


def test_identical_sequences(engine):
    rng = np.random.default_rng(6)
    X = _mels(rng, 3, 90, 80)
    n = np.array([90, 37, 1])
    mcd, pairs, path = _run(engine, X, n, X.copy(), n)
    assert (mcd == 0).all()
    np.testing.assert_array_equal(pairs, n)
    for b in range(3):
        np.testing.assert_array_equal(path[b, :n[b]], np.stack([np.arange(n[b])] * 2, 1))
        assert (path[b, n[b]:] == -1).all()


def test_known_time_warp(engine):
    rng = np.random.default_rng(7)
    x = _mels(rng, 40, 80)
    reps = rng.integers(1, 5, 40)
    y = np.repeat(x, reps, axis=0)
    for X, Y, swap in ((x, y, False), (y, x, True)):
        mcd, pairs, path = _run(engine, X[None], [len(X)], Y[None], [len(Y)])
        assert mcd[0] == 0 and pairs[0] == len(y)
        want = np.stack([np.repeat(np.arange(40), reps), np.arange(len(y))], 1)
        np.testing.assert_array_equal(path[0, :pairs[0]], want[:, ::-1] if swap else want)


def test_length_one_and_unequal_sizes(engine):
    rng = np.random.default_rng(8)
    X, Y = _mels(rng, 4, 30, 80), _mels(rng, 4, 70, 80)
    _, pairs, path, _ = _check(engine, X, [1, 30, 1, 17], Y, [70, 1, 1, 70])
    assert pairs.tolist() == [70, 30, 1, 70]
    np.testing.assert_array_equal(path[0, :70], np.stack([np.zeros(70, int), np.arange(70)], 1))
    np.testing.assert_array_equal(path[1, :30], np.stack([np.arange(30), np.zeros(30, int)], 1))


def test_global_memory_route(engine):
    """1500 x 1200 frames: the cepstra (2700 rows of 25 doubles) do not fit in shared memory."""
    rng = np.random.default_rng(9)
    X, Y = _mels(rng, 2, 1500, 80), _mels(rng, 2, 1200, 80)
    X[1, :400] = np.repeat(Y[1, :200], 2, axis=0)                       # a known stretch at the start of pair 1
    mcd, pairs, path, ref = _check(engine, X, [1500, 1500], Y, [1200, 1200])
    alone = _run(engine, X[1:], [1500], Y[1:], [1200])
    assert alone[0][0] == mcd[1] and alone[1][0] == pairs[1]
    np.testing.assert_array_equal(alone[2][0], path[1])


def test_ragged_batch_bit_for_bit(engine):
    """Each pair of a ragged batch, some in shared memory and one through global memory, gives what it gives alone."""
    rng = np.random.default_rng(10)
    Tx, Ty = 700, 650
    X, Y = _mels(rng, 5, Tx, 80), _mels(rng, 5, Ty, 80)
    X[:, 300:] = np.nan                                                  # never read past the lengths
    Y[:, 600:] = np.nan
    nx, ny = [210, 1, 300, 55, 300], [180, 9, 600, 55, 5]
    Xc = np.where(np.isnan(X), 0, X)
    Yc = np.where(np.isnan(Y), 0, Y)
    mcd, pairs, path, _ = _check(engine, Xc, nx, Yc, ny, paths=False)
    mcd2, pairs2, path2 = _run(engine, X, nx, Y, ny)
    assert np.array_equal(mcd, mcd2) and np.array_equal(pairs, pairs2) and np.array_equal(path, path2)
    for b in range(5):
        m1, p1, q1 = _run(engine, X[b:b + 1, :nx[b]].copy(), [nx[b]], Y[b:b + 1, :ny[b]].copy(), [ny[b]])
        assert m1[0] == mcd[b] and p1[0] == pairs[b]
        np.testing.assert_array_equal(q1[0, :p1[0]], path[b, :pairs[b]])


def test_refusals_before_launch(engine):
    X = torch.rand(2, 10, 80, device="cuda")
    Y = torch.rand(2, 12, 80, device="cuda")
    with pytest.raises(DcttsError, match="utterance 1 has X length 11"):
        engine.mcd_dtw(X, [10, 11], Y, [12, 12])
    with pytest.raises(DcttsError, match="utterance 0 has Y length 0"):
        engine.mcd_dtw(X, [10, 10], Y, [0, 12])
    with pytest.raises(DcttsError, match="K must be"):
        engine.mcd_dtw(X, [10, 10], Y, [12, 12], K=80)
    with pytest.raises(DcttsError, match="Y must be"):
        engine.mcd_dtw(X, [10, 10], Y[:1], [12])
    # the C entry point itself, past the Python checks
    lib, h = engine._lib, engine._h
    mcd = torch.full((2,), -7.0, dtype=torch.float64, device="cuda")
    pairs = torch.full((2,), -7, dtype=torch.int32, device="cuda")

    def call(nx, ny, K=24):
        nxh, nyh = np.array(nx, np.int32), np.array(ny, np.int32)
        return lib.dctts_mcd_dtw(h, C.c_void_p(X.data_ptr()), 10, C.c_void_p(nxh.ctypes.data), C.c_void_p(Y.data_ptr()), 12,
                                 C.c_void_p(nyh.ctypes.data), 2, K, C.c_void_p(mcd.data_ptr()), C.c_void_p(pairs.data_ptr()),
                                 None, None)
    for args, msg in ((([10, 0], [12, 12]), "utterance 1 has X length 0"), (([10, 10], [13, 12]), "utterance 0 has Y length 13"),
                      (([10, 10], [12, 12], 0), "K must be"), (([10, 10], [12, 12], 80), "K must be")):
        assert call(*args) != 0
        assert msg in lib.dctts_last_error(h).decode()
    torch.cuda.synchronize()
    assert (mcd == -7).all() and (pairs == -7).all()                   # nothing was launched
    big = torch.zeros(1, 10000, 80, device="cuda")
    with pytest.raises(DcttsError, match="utterance 0: three diagonals"):
        engine.mcd_dtw(big, [10000], big[:, :5], [5])


def test_no_side_effects_on_synthesis(engine):
    from dc_tts_b200.params import synthetic_text
    L = np.concatenate([synthetic_text(1, 40 + 7 * b, seed=b) for b in range(3)])
    Y1, P1, n1 = engine.text2mel_generate_until(L)
    Y1, P1, n1 = Y1.clone(), P1.clone(), n1.clone()
    rng = np.random.default_rng(11)
    _run(engine, _mels(rng, 4, 300, 80), [300, 2, 100, 7], _mels(rng, 4, 1400, 80), [1400, 3, 50, 1000])
    Y2, P2, n2 = engine.text2mel_generate_until(L)
    assert torch.equal(Y1, Y2) and torch.equal(P1, P2) and torch.equal(n1, n2)
