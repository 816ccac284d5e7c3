"""The float64 feature references of tests/ref_feature_stages.py, pinned on the CPU at every corpus rate: equal to the
oracle's get_spectrograms / load_spectrograms run in float64, the float32 oracle and a float32 restatement inside
tau * S, and each deliberately wrong variant outside it."""
import numpy as np
import pytest

from oracle import ref_features as rf
from oracle import ref_vocoder as rv

import ref_feature_stages as fs
from sample_rates import RATES, at_rate

# the wrong variants that the tolerances of tests/test_gpu_wav_features.py let through
OLD_BAR_MISSES = {"fp16_weights"}


def _clip(sr, seed=0):
    rng = np.random.default_rng(seed)
    return fs.clip(rng, 3 * sr, sr, lead=3000, tail=2000, tone=True, hush=True).astype(np.float32)


@pytest.mark.parametrize("sr", list(RATES))
def test_reference_equals_the_oracle_in_float64(sr):
    with at_rate(sr) as H:
        y = _clip(sr)
        s, e = rv.trim_indices(y)
        ref = fs.ref_features(y[s:e], sr, H.n_fft, H.hop_length, H.win_length)
        mel64, mag64 = rf.get_spectrograms(y, np.float64)
        assert mag64.dtype == np.float64 and mag64.shape == ref["a"].shape
        assert np.abs(mag64 - fs.normalise(ref["a"])).max() <= 1e-12
        assert np.abs(mel64 - fs.normalise(ref["mel"])).max() <= 1e-12
        mel_r, mag_r = rf.load_spectrograms(y, np.float64)
        T = ref["a"].shape[0]
        assert mel_r.shape[0] == -(-T // H.r) and np.array_equal(mag_r[:T], mag64) and not mag_r[T:].any()
        assert np.abs(mel_r[:-(-T // H.r)] - fs.normalise(ref["mel"][::H.r])).max() <= 1e-12
        # the float32 oracle is the same computation: unchanged by the dtype argument
        mel32, mag32 = rf.get_spectrograms(y)
        assert mel32.dtype == np.float32 and np.abs(mel32 - mel64).max() < 1e-5


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("sr", list(RATES))
def test_float32_chains_land_inside_the_bounds(sr, seed):
    with at_rate(sr) as H:
        tau = fs.TAU[H.n_fft]
        y = _clip(sr, seed)
        s, e = rv.trim_indices(y)
        ref = fs.ref_features(y[s:e], sr, H.n_fft, H.hop_length, H.win_length)
        mel_o, mag_o = rf.get_spectrograms(y)
        mag32, mel32 = fs.features32(y[s:e], H.n_fft, H.hop_length, H.win_length, ref["W"].astype(np.float32))
        for name, mag, mel in (("oracle", mag_o, mel_o), ("float32", mag32, mel32)):
            rm, _ = fs.check_mag(mag, ref, tau["mag"])
            rl, _ = fs.check_mel(mel, ref, tau["mel"])
            assert rm <= 1 and rl <= 1, (name, rm, rl)
        # the clip at 1, the 1e-5 floor and the 1e-8 clip are all reached
        n = fs.normalise(ref["a"])
        assert (n == 1).any() and (n == 1e-8).any() and (ref["a"] < 1e-5).any()


def _variants(y, s, e, H):
    """name -> (mag, mel, reference) of each wrong float32 chain."""
    n_fft, hop, win = H.n_fft, H.hop_length, H.win_length
    ref = fs.ref_features(y[s:e], H.sr, n_fft, hop, win)
    W = ref["W"]
    short = W.copy()
    for m in range(W.shape[0]):
        short[m, np.flatnonzero(W[m])[-1]] = 0.0                   # each filter's range one bin short at its end
    lpad = (n_fft - win) // 2
    sym = np.zeros(n_fft)
    sym[lpad:lpad + win] = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(win) / (win - 1))   # symmetric Hann
    shifted = np.zeros(n_fft)
    shifted[lpad + 1:lpad + 1 + win] = rv.hann_padded(n_fft, win, np.float64)[lpad:lpad + win]   # lpad one sample off
    out = {}
    W32 = W.astype(np.float32)
    out["fp16_weights"] = fs.features32(y[s:e], n_fft, hop, win, W.astype(np.float16)) + (ref,)
    out["range_short"] = fs.features32(y[s:e], n_fft, hop, win, short) + (ref,)
    out["symmetric_hann"] = fs.features32(y[s:e], n_fft, hop, win, W32, window=sym) + (ref,)
    out["lpad_off_by_one"] = fs.features32(y[s:e], n_fft, hop, win, W32, window=shifted) + (ref,)
    s1 = s + 4001                                                   # a trim start inside the sound
    out["preemph_reads_before_start"] = fs.features32(y[s1:e], n_fft, hop, win, W32, prev=y[s1 - 1]) + \
        (fs.ref_features(y[s1:e], H.sr, n_fft, hop, win),)
    return out


@pytest.mark.parametrize("sr", list(RATES))
def test_wrong_variants_exceed_their_bounds(sr):
    with at_rate(sr) as H:
        tau = fs.TAU[H.n_fft]
        y = _clip(sr)
        s, e = rv.trim_indices(y)
        misses = set()
        for name, (mag, mel, ref) in _variants(y, s, e, H).items():
            worst = max(fs.check_mag(mag, ref, tau["mag"])[0], fs.check_mel(mel, ref, tau["mel"])[0])
            assert worst > 3, (name, worst)
            if fs.old_tolerance_passes(mel, mag, fs.normalise(ref["mel"]), fs.normalise(ref["a"])):
                misses.add(name)
        assert misses == OLD_BAR_MISSES, misses


def test_off_by_one_lpad_is_at_the_odd_pad_of_44k():
    """n_fft 4096, win 2205: lpad = 945 is odd, where a (n_fft - win + 1) / 2 rounding would move the window."""
    with at_rate(44100) as H:
        assert (H.n_fft, H.win_length) == (4096, 2205) and (H.n_fft - H.win_length) // 2 == 945


def test_trim_margin_and_decision():
    """The float64 trim decision on a clip whose frames are far from -60 dB, and the margin it skips."""
    y = _clip(22050)
    mse = fs.ref_energies(y[None])[0]
    assert fs.trims_agree(rv.trim_indices(y.astype(np.float64)), y, 5e-7)
    assert abs(fs.trim_margin_db(1e-6) - 8.686e-6) < 1e-8
    with pytest.raises(AssertionError):
        s, e = rv.trim_indices(y.astype(np.float64))
        fs.trims_agree((s + 512, e), y, 5e-7)
    assert mse.max() > 0
