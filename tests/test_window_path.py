"""utils.stretch_path, the speaking-rate rule of synthesize(duration_scale=...), on hand-built paths (no GPU)."""
import numpy as np
import pytest

from dc_tts_b200.utils import stretch_path


def _rule(p, n, factor):
    m = max(1, round(factor * n))
    return [p[min(n - 1, int(np.floor(j / factor)))] for j in range(m)]


def test_identity_and_padding():
    P = np.array([[0, 0, 1, 2, 2, 3], [0, 1, 1, -1, -1, -1]])
    out, n = stretch_path(P, [6, 3], 1.0)
    assert n.tolist() == [6, 3] and out.dtype == np.int32
    assert out[0].tolist() == [0, 0, 1, 2, 2, 3]
    assert out[1].tolist() == [0, 1, 1, 1, 1, 1]          # padded with the row's last window


@pytest.mark.parametrize("factor", [0.5, 0.7, 0.8, 1.25, 1.5, 2.0, 3.0])
def test_matches_the_rule(factor):
    rng = np.random.default_rng(int(factor * 100))
    P = np.cumsum(rng.integers(0, 2, size=(5, 60)), axis=1)
    lens = np.array([1, 2, 17, 40, 60])
    out, n = stretch_path(P, lens, factor)
    for b in range(5):
        want = _rule(P[b], int(lens[b]), factor)
        assert n[b] == len(want)
        assert out[b, :n[b]].tolist() == want
        assert (out[b, n[b]:] == want[-1]).all()


def test_lengths_round_half_to_even_and_never_below_one():
    P = np.zeros((3, 10), np.int64)
    _, n = stretch_path(P, [10, 2, 1], 1.25)               # 12.5 -> 12, 2.5 -> 2, 1.25 -> 1
    assert n.tolist() == [12, 2, 1]
    _, n = stretch_path(P, [1, 1, 3], 0.1)
    assert n.tolist() == [1, 1, 1]


def test_refusals():
    P = np.zeros((2, 200), np.int64)
    with pytest.raises(ValueError, match="utterance 1 stretched from 200 to 300"):
        stretch_path(P, [100, 200], 1.5, steps=210)
    with pytest.raises(ValueError, match="utterance 0 has length 0"):
        stretch_path(P, [0, 5], 1.5)
    with pytest.raises(ValueError, match="factor"):
        stretch_path(P, [5, 5], 0.0)
    with pytest.raises(ValueError, match="path must be"):
        stretch_path(P, [5, 5, 5], 1.0)
