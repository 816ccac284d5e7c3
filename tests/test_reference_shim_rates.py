"""The reference's own utils.spectrogram2wav / get_spectrograms / load_spectrograms at 16, 44.1 and 48 kHz (n_fft 1024,
4096, 4096), with the restated librosa primitives standing in for librosa, against the oracle's composition (1e-6, as
test_reference_shim.py holds it at 22.05 kHz): from the committed fixture, and live wherever the reference exists."""
import os
import sys

import numpy as np
import pytest

from conftest import ROOT, golden
from dc_tts_b200.hyperparams import Hyperparams as hp
from sample_rates import at_rate

sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_golden_refshim_rates import RATES, rate_inputs, reference_outputs      # noqa: E402

HAVE_REF = os.path.isfile("/root/reference/utils.py")


def _check(ref, monkeypatch):
    from oracle import ref_features as rf
    from oracle import ref_vocoder as rv
    monkeypatch.setattr(hp, "n_iter", 3)
    for sr, n_fft in RATES:
        with at_rate(sr, n_fft) as H:
            mag, y = rate_inputs(sr, n_fft)
            mine, _, _ = rv.spectrogram2wav(mag, n_iter=3)
            w = ref["wav_%d" % sr]
            assert w.shape == mine.shape and np.abs(w - mine).max() <= 1e-6 * max(1.0, np.abs(mine).max()), sr
            mel, mg = rf.get_spectrograms(y)
            assert mg.shape[1] == 1 + n_fft // 2 and mel.shape[1] == H.n_mels
            assert int(ref["get_frames_%d" % sr]) == len(mg) and ref["get_mel_%d" % sr].shape == mel.shape, sr
            assert np.abs(ref["get_mel_%d" % sr] - mel).max() < 1e-6, sr
            assert np.abs(ref["load_mag_%d" % sr][:len(mg)] - mg).max() < 1e-6, sr
            mel, mg = rf.load_spectrograms(y)
            assert ref["load_mel_%d" % sr].shape == mel.shape and ref["load_mag_%d" % sr].shape == mg.shape, sr
            assert np.abs(ref["load_mel_%d" % sr] - mel).max() < 1e-6 and np.abs(ref["load_mag_%d" % sr] - mg).max() < 1e-6, sr


def test_sample_rates_vs_reference_output(monkeypatch):
    _check(golden("refshim_sample_rates.npz"), monkeypatch)


@pytest.mark.skipif(not HAVE_REF, reason="the reference is not present on this machine")
def test_sample_rates_vs_reference_code(monkeypatch):
    _check(reference_outputs(), monkeypatch)
