"""The float64 streaming vocoder (tests/ref_stream_vocoder.py) against the whole-signal references, on the CPU.

  * One final push is fast Griffin-Lim on the whole spectrogram (tests/ref_fast_griffin_lim.py), plain and with momentum.
  * Pushed in pieces, the committed ranges tile [0, hop (T - 1)) once each, a committed sample never changes afterwards,
    and the de-emphasised pieces concatenate to scipy.signal.lfilter of the whole streamed waveform.
  * The frames below the first active one do not reach the committed samples, and the commit stops short of every
    frame that reads the reflected tail.
"""
import numpy as np
import pytest
import scipy.signal

from dc_tts_b200.hyperparams import Hyperparams
import ref_fast_griffin_lim as fg
import ref_stream_vocoder as sv
import ref_vocoder_stages as rs
from sample_rates import at_rate

SR = {1024: 16000, 2048: 22050, 4096: 44100}


def _amplitude(n, T, seed):
    mag = rs.make_mag(np.random.default_rng(seed), 1, T, n)[0]
    return rs.ref_prepare(mag, Hyperparams.power)          # (T, F) float64


@pytest.mark.parametrize("n", sorted(SR))
@pytest.mark.parametrize("momentum", [0.0, 0.99])
def test_one_final_push_is_fast_griffin_lim(n, momentum):
    with at_rate(SR[n], n) as H:
        S = _amplitude(n, 23, n)
        v = sv.StreamVocoder(n, H.hop_length, H.win_length, 4, momentum)
        out = v.push(S, final=True)
        ref = fg.fast_griffin_lim(S.T.copy(), 4, momentum)
        Ly = H.hop_length * (S.shape[0] - 1)
        assert v.spans == [(0, Ly)]
        np.testing.assert_allclose(v.y[:Ly], ref, rtol=0, atol=1e-12 * np.abs(ref).max())
        np.testing.assert_allclose(out, scipy.signal.lfilter([1], [1, -H.preemphasis], ref), rtol=0,
                                   atol=1e-11 * np.abs(out).max())


@pytest.mark.parametrize("n", sorted(SR))
@pytest.mark.parametrize("chunk,momentum", [(1, 0.0), (5, 0.99), (16, 0.0)])
def test_pieces_tile_the_waveform_and_deemphasise_as_one(n, chunk, momentum):
    with at_rate(SR[n], n) as H:
        T = 40
        S = _amplitude(n, T, chunk + n)
        v = sv.StreamVocoder(n, H.hop_length, H.win_length, 3, momentum)
        outs, held = [], []
        for a in range(0, T, chunk):
            outs.append(v.push(S[a:a + chunk], final=a + chunk >= T))
            held.append(v.y[:v.c].copy())
        Ly = H.hop_length * (T - 1)
        ends = [e for _, e in v.spans]
        assert [s for s, _ in v.spans] == [0] + ends[:-1] and ends[-1] == Ly
        assert sum(o.size for o in outs) == Ly
        for h in held:                                       # committed samples stay as they were committed
            assert np.array_equal(v.y[:h.size], h)
        whole = np.concatenate(outs)
        ref = scipy.signal.lfilter([1], [1, -H.preemphasis], v.y[:Ly])
        np.testing.assert_allclose(whole, ref, rtol=0, atol=1e-12 * np.abs(ref).max())
        assert len([o for o in outs if o.size]) > 1          # it streamed


@pytest.mark.parametrize("n", sorted(SR))
def test_active_frames_and_commit_bounds(n):
    with at_rate(SR[n], n) as H:
        hop, win = H.hop_length, H.win_length
        a0, a1 = sv.window_bounds(n, win)
        for c in (0, 1, a1 - 1, a1, a1 + 1, 5 * hop + 3, 40 * hop):
            lo = sv.first_active_frame(c, n, hop, win)
            assert hop * lo + a1 > c                         # frame lo reaches past c
            assert lo == 0 or hop * (lo - 1) + a1 <= c       # frame lo - 1 does not
        for A in (2, 3, 9, 64):
            Ly = hop * (A - 1)
            c = sv.commit_end(0, A, False, n, hop, win)
            assert 0 <= c <= Ly
            for t in range(A):                               # a frame whose window reads past Ly starts at or after c
                if hop * t + a1 > Ly:
                    assert c <= max(0, hop * t + a0), (A, t, c)
            assert sv.commit_end(0, A, True, n, hop, win) == Ly
