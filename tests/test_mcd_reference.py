"""The float64 MCD-DTW reference (tests/ref_mcd.py) pinned on the CPU: its cepstrum against scipy's orthonormal DCT, and
its DTW -- cost, path and tie rule -- against brute-force enumeration of every monotone path on small grids."""
import itertools

import numpy as np
import pytest
import scipy.fft

import ref_mcd


def _paths(nx, ny):
    """Every monotone path from (0, 0) to (nx - 1, ny - 1) with steps (1, 1), (1, 0), (0, 1), as lists of cells."""
    out = []

    def walk(i, j, acc):
        if (i, j) == (nx - 1, ny - 1):
            out.append(acc)
            return
        for di, dj in ((1, 1), (1, 0), (0, 1)):
            if i + di < nx and j + dj < ny:
                walk(i + di, j + dj, acc + [(i + di, j + dj)])
    walk(0, 0, [(0, 0)])
    return out


def _codes_back(path):
    """The steps of a path from its end, coded as the DTW's back-pointers: 0 diagonal, 1 advance X, 2 advance Y."""
    codes = []
    for (i0, j0), (i1, j1) in zip(path[-2::-1], path[::-1]):
        codes.append({(1, 1): 0, (1, 0): 1, (0, 1): 2}[(i1 - i0, j1 - j0)])
    return codes


def _brute(d):
    """(min cost, the minimum-cost path the tie rule picks): among the cheapest paths, the one whose steps, read from
    the end, prefer the diagonal, then advancing X, then advancing Y -- exact with integer costs."""
    best, chosen = None, None
    for p in _paths(*d.shape):
        c = sum(d[i, j] for i, j in p)
        key = (c, _codes_back(p))
        if best is None or key < best:
            best, chosen = key, p
    return best[0], np.array(chosen)


def test_dct_matrix_is_scipy_orthonormal_dct():
    rng = np.random.default_rng(0)
    for M in (5, 80):
        D = ref_mcd.dct_matrix(M)
        np.testing.assert_allclose(D @ D.T, np.eye(M), atol=1e-13)
        a = rng.standard_normal((7, M))
        np.testing.assert_allclose(a @ D.T, scipy.fft.dct(a, type=2, norm="ortho", axis=-1), atol=1e-12)


def test_cepstrum_is_dct_of_log_amplitude():
    rng = np.random.default_rng(1)
    mels = rng.uniform(0, 1, (9, 80)).astype(np.float32)
    a = (np.log(10.0) / 20.0) * (100.0 * mels.astype(np.float64) - 100.0 + 20.0)
    want = scipy.fft.dct(a, type=2, norm="ortho", axis=-1)[:, 1:25]
    np.testing.assert_allclose(ref_mcd.cepstrum(mels, 24), want, rtol=1e-12, atol=1e-12)
    # the log amplitude is the normalised dB undone: 20 log10(amplitude) = 100 x - 100 + 20
    np.testing.assert_allclose(20.0 * a / np.log(10.0), 100.0 * mels.astype(np.float64) - 80.0, atol=1e-12)


def test_local_cost():
    cx, cy = np.array([[0.0, 3.0]]), np.array([[4.0, 0.0], [0.0, 3.0]])
    d = ref_mcd.local_cost(cx, cy)
    np.testing.assert_allclose(d, [[10.0 / np.log(10.0) * np.sqrt(2.0 * 25.0), 0.0]])


@pytest.mark.parametrize("nx,ny", [(1, 1), (1, 4), (4, 1), (2, 3), (3, 3), (4, 3), (3, 5)])
def test_dtw_against_enumeration_random(nx, ny):
    rng = np.random.default_rng(nx * 10 + ny)
    for _ in range(5):
        d = rng.uniform(0, 1, (nx, ny))
        r = ref_mcd.dtw(d)
        cost, path = _brute(d)
        assert r["total"] == pytest.approx(cost, rel=1e-12)
        np.testing.assert_array_equal(r["path"], path)
        assert r["pairs"] == len(path) and r["mcd"] == pytest.approx(cost / len(path), rel=1e-12)


@pytest.mark.parametrize("nx,ny", [(2, 2), (2, 4), (3, 3), (4, 3), (4, 4)])
def test_dtw_tie_rule_against_enumeration(nx, ny):
    """Small integer costs: many cheapest paths, so the tie rule decides; sums of integers are exact."""
    rng = np.random.default_rng(100 + nx * 10 + ny)
    for _ in range(40):
        d = rng.integers(0, 3, (nx, ny)).astype(np.float64)
        r = ref_mcd.dtw(d)
        cost, path = _brute(d)
        assert r["total"] == cost
        np.testing.assert_array_equal(r["path"], path)


def test_dtw_all_equal_frames_path():
    """Every cost 0: the walk back takes the diagonal while it can, then advances the longer side only."""
    for nx, ny in ((5, 3), (3, 5), (4, 4), (1, 3)):
        r = ref_mcd.dtw(np.zeros((nx, ny)))
        k = min(nx, ny) - 1
        head = [(i, 0) for i in range(nx - k)] if nx >= ny else [(0, j) for j in range(ny - k)]
        i0, j0 = head[-1]
        want = head + [(i0 + s, j0 + s) for s in range(1, k + 1)]
        np.testing.assert_array_equal(r["path"], want)
        assert r["mcd"] == 0.0 and r["pairs"] == max(nx, ny)


def test_dtw_recovers_repeated_frames():
    rng = np.random.default_rng(3)
    x = rng.uniform(0, 1, (6, 80)).astype(np.float32)
    reps = np.array([1, 3, 2, 1, 4, 2])
    y = np.repeat(x, reps, axis=0)
    r = ref_mcd.mcd_dtw(x, y)
    np.testing.assert_array_equal(r["path"][:, 0], np.repeat(np.arange(6), reps))
    np.testing.assert_array_equal(r["path"][:, 1], np.arange(len(y)))
    assert r["mcd"] == 0.0 and r["pairs"] == len(y)


def test_mcd_batch_pads():
    rng = np.random.default_rng(4)
    X, Y = rng.uniform(0, 1, (2, 5, 80)), rng.uniform(0, 1, (2, 4, 80))
    out = ref_mcd.mcd_batch(X, [5, 2], Y, [4, 1])
    assert out["path"].shape == (2, 8, 2)
    assert (out["path"][1, out["pairs"][1]:] == -1).all()
    one = ref_mcd.mcd_dtw(X[1, :2], Y[1, :1])
    assert out["mcd"][1] == one["mcd"] and list(itertools.chain(*one["path"])) == list(out["path"][1, :2].ravel())
