"""CPU checks of the synthesis stream's grid and halos (tests/ref_synth_stream.py) on the float64 SSRN oracle.

  * The halos from the layer table are those of a perturbation: changing the mel row `left` frames before a committed
    run, or `right` frames after it, moves a committed magnitude row; a row one frame farther moves none.
  * Windowed float64 SSRN on the grid tiles the whole-sequence float64 SSRN at chunk 1, 7, 16 and 64, ragged lengths.
  * The grid covers every frame once, in order, with the last chunk final, and the pushes carry r rows per frame."""
import numpy as np
import pytest

import ref_synth_stream as rs
from dc_tts_b200.hyperparams import Hyperparams as hp


@pytest.fixture(scope="module")
def P():
    from dc_tts_b200.params import init_params
    return init_params(0, "perturbed")


def _Y(T, seed):
    return np.random.default_rng(seed).uniform(0.0, 0.99, (T, hp.n_mels))


def test_halo_from_the_layer_table():
    assert rs.halo() == (9, 8)


def test_halo_by_perturbation(P):
    left, right = rs.halo()
    T, a, e = 40, 18, 22                               # committed mel rows [a, e), well inside the sequence
    Y = _Y(T, 1)
    base = rs.ssrn64(P, Y[None])[0][4 * a:4 * e]

    def moved(row):
        Yp = Y.copy()
        Yp[row] += 0.25
        return np.abs(rs.ssrn64(P, Yp[None])[0][4 * a:4 * e] - base).max()
    assert moved(a - left) > 1e-9 and moved(e - 1 + right) > 1e-9
    assert moved(a - left - 1) == 0.0 and moved(e + right) == 0.0


@pytest.mark.parametrize("chunk", [1, 7, 16, 64])
def test_windows_tile_the_whole_sequence(P, chunk):
    left, right = rs.halo()
    for length, seed in ((37, 2), (9, 3)):
        Y = _Y(length, seed)
        whole = rs.ssrn64(P, Y[None])[0]
        tiled = rs.windowed_ssrn64(P, Y, length, chunk, left, right)
        assert tiled.shape == whole.shape
        assert np.abs(tiled - whole).max() <= 1e-12, (chunk, length)


@pytest.mark.parametrize("length", [1, 2, 15, 16, 17, 210])
@pytest.mark.parametrize("chunk", [1, 7, 16, 64, 210])
def test_grid(length, chunk):
    left, right = rs.halo()
    g = rs.chunks(length, chunk, left, right)
    assert [c[0] for c in g] == list(range(0, length, chunk))
    assert all(e == min(length, a + chunk) for a, e, *_ in g)
    assert [c[4] for c in g] == [False] * (len(g) - 1) + [True]
    assert all(0 <= s <= a and e <= t <= length and a - s <= left and t - e <= right for a, e, s, t, _ in g)
    assert sum(n for n, _ in rs.pushes(length, chunk)) == 4 * length
    assert all(rs.ready_frames(length, chunk, right, k) <= length for k in range(len(g)))
