"""Fast Griffin-Lim in the oracle (tests/ref_fast_griffin_lim.py): momentum 0 is the reference's Griffin-Lim bit
for bit, and on the magnitudes of real-looking signals momentum 0.99 converges further in 50 iterations than plain
Griffin-Lim does, measured by the spectral convergence ||S - |STFT(x)||| / ||S||.  The GPU half is
test_gpu_vocoder_momentum.py; both take their signals from tests/ref_vocoder_stages.py."""
import numpy as np
import pytest

from dc_tts_b200.hyperparams import Hyperparams as hp
from oracle import ref_vocoder as rv

import ref_fast_griffin_lim as fg
from ref_vocoder_stages import POWERS, SIGNALS, amplitude, magnitude


def test_momentum_zero_is_griffin_lim_bit_for_bit():
    S = amplitude(magnitude("vibrato")[:20], hp.power)
    for dtype in (np.float32, np.float64):
        Sd = S.astype(dtype)
        assert np.array_equal(fg.fast_griffin_lim(Sd, 4, momentum=0.0), rv.griffin_lim(Sd, 4)), dtype
        y, hist = fg.fast_griffin_lim(Sd, 4, momentum=0.0, convergence=True)
        assert np.array_equal(y, rv.griffin_lim(Sd, 4)) and hist.shape == (5,)


def test_momentum_changes_the_update_and_keeps_float32():
    S = amplitude(magnitude("chirp")[:20], hp.power)
    y0 = fg.fast_griffin_lim(S, 3, momentum=0.0)
    y1 = fg.fast_griffin_lim(S, 3, momentum=0.99)
    assert y1.dtype == np.float32 and not np.array_equal(y0, y1)
    # one iteration: est_{-1} = 0, so the first update is the plain one whatever the momentum
    assert np.array_equal(fg.fast_griffin_lim(S, 1, momentum=0.99), rv.griffin_lim(S, 1))


def test_convergence_history_matches_its_definition():
    S = amplitude(magnitude("bursts")[:30], hp.power, np.float64)
    y, hist = fg.fast_griffin_lim(S, 3, momentum=0.5, convergence=True)
    assert hist[-1] == fg.spectral_convergence(S, rv.stft(y))
    y0, hist0 = fg.fast_griffin_lim(S, 0, momentum=0.5, convergence=True)
    assert hist0.shape == (1,) and hist0[0] == hist[0]


@pytest.mark.parametrize("power", POWERS)
@pytest.mark.parametrize("kind", SIGNALS)
def test_momentum_converges_further_in_50_iterations(kind, power):
    """Plain Griffin-Lim's history falls (within float32 noise) and momentum 0.99 ends 50 iterations lower."""
    S = amplitude(magnitude(kind), power)
    _, plain = fg.fast_griffin_lim(S, 50, momentum=0.0, convergence=True)
    _, fast = fg.fast_griffin_lim(S, 50, momentum=0.99, convergence=True)
    assert np.all(np.diff(plain) <= 1e-4 * plain[:-1]), plain
    assert plain[-1] < 0.8 * plain[0], (plain[0], plain[-1])
    assert fast[-1] < plain[-1], (kind, power, fast[-1], plain[-1])
