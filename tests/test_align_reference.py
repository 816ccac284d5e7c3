"""The aligner's CPU reference (tests/ref_align.py) against brute-force enumeration of every admissible path."""
import numpy as np
import pytest

from ref_align import admissible, band, path_score, search


def _all_paths(T_b, e, w):
    """Every admissible path: 0 <= n_0 <= w - 1, steps in [0, w - 1], ending at e."""
    paths = [[n] for n in range(w)]
    for _ in range(T_b - 1):
        paths = [p + [p[-1] + s] for p in paths for s in range(w) if p[-1] + s <= e]
    return [p for p in paths if p[-1] == e]


def _brute(A, T_b, e, w):
    """The best score over every admissible path, and the path the tie rule picks among those that reach it: comparing
    from the last frame backward, the larger predecessor (the smaller step) first."""
    paths = _all_paths(T_b, e, w)
    scores = np.array([path_score(A, p) for p in paths])
    best = scores.max()
    top = [p for p, s in zip(paths, scores) if s == best]
    return best, max(top, key=lambda p: p[::-1][1:])


def _check(A, T_b, e, w):
    r = search(A, T_b, e, w)
    best, chars = _brute(A, T_b, e, w)
    assert r["score"] == best
    assert list(r["chars"]) == chars
    assert admissible(r["chars"], e, w)
    assert r["path"][0] == 0 and (r["path"][1:] == r["chars"][:-1]).all()
    assert r["durations"].sum() == T_b and r["durations"].shape == (A.shape[0],)
    assert (r["durations"] == np.bincount(r["chars"], minlength=A.shape[0])).all()
    return r


def _cases(seed, count):
    rng = np.random.default_rng(seed)
    for _ in range(count):
        w = int(rng.integers(1, 5))
        N = int(rng.integers(1, 9))
        T_b = int(rng.integers(1, 9))
        top = min(N - 1, (w - 1) * T_b)
        e = int(rng.integers(0, top + 1))
        yield w, N, T_b, e, rng


def test_random_cases():
    for w, N, T_b, e, rng in _cases(0, 300):
        A = rng.random((N, T_b)).astype(np.float32)
        A /= A.sum(0, keepdims=True)
        _check(A, T_b, e, w)


def test_exact_ties_follow_the_tie_rule():
    """Uniform A: every admissible path has the same score, bit for bit; the smaller step wins at every frame."""
    seen = 0
    for w, N, T_b, e, _ in _cases(1, 200):
        A = np.full((N, T_b), np.float32(1.0 / N))
        r = _check(A, T_b, e, w)
        if T_b > 1 and w > 1 and e > 0:
            seen += 1
            # walking back from e, each step is the smallest the band allows: stay as long as the start is reachable
            n = e
            for t in range(T_b - 1, 0, -1):
                plo, phi = band(t - 1, T_b, e, w)
                n = n - max(0, n - phi)
                assert r["chars"][t - 1] == n
    assert seen > 50


def test_floored_zeros():
    """Zeros and values below 1e-30 all cost log(1e-30f): ties among floored cells follow the same rule."""
    for w, N, T_b, e, rng in _cases(2, 200):
        A = rng.random((N, T_b)).astype(np.float32)
        A[rng.random((N, T_b)) < 0.6] = 0
        A[rng.random((N, T_b)) < 0.1] = np.float32(1e-35)
        _check(A, T_b, e, w)
    _check(np.zeros((5, 4), np.float32), 4, 3, 2)


@pytest.mark.parametrize("w", [1, 2, 3, 4])
def test_reachability_limit_and_one_frame(w):
    rng = np.random.default_rng(w)
    for T_b in range(1, 8):
        e = (w - 1) * T_b
        if e >= 9:
            continue
        A = rng.random((e + 1, T_b)).astype(np.float32)
        r = _check(A, T_b, e, w)
        if w > 1:          # at the limit the only path takes the largest step at every frame
            assert list(r["chars"]) == [(w - 1) * (t + 1) for t in range(T_b)]
    for N in range(1, 6):
        for e in range(min(N, w)):
            _check(rng.random((N, 1)).astype(np.float32), 1, e, w)
    with pytest.raises(ValueError):
        search(np.ones((9, 2), np.float32), 2, (w - 1) * 2 + 1, w)


def test_planted_diagonal_is_recovered():
    """A noisy alignment with a monotonic diagonal planted in it: the path follows it within one character."""
    rng = np.random.default_rng(7)
    for w, N, T in ((3, 60, 200), (2, 40, 120), (4, 150, 210)):
        true = np.minimum(N - 1, np.floor(np.arange(T) * (N - 1) / (T - 1) + 1e-9)).astype(np.int64)
        A = rng.random((N, T)).astype(np.float32) * 0.05
        A[true, np.arange(T)] += 1.0
        A /= A.sum(0, keepdims=True)
        r = search(A, T, N - 1, w)
        assert np.abs(r["chars"] - true).max() <= 1, (w, N, T)
        assert r["durations"].sum() == T
