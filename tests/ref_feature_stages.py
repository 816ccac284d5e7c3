"""ORACLE (test infrastructure) -- float64 references and per-element bounds for the feature extraction
(`dctts_load_spectrograms_batch`, `dctts_get_spectrograms`, `dctts_feature_stage`): the trim energies, |X| and the mel
filterbank on the normalised dB scale, at any n_fft and rate.

The reference's input is the trimmed waveform pre-emphasised in float32 (a float32 product, then a float32 difference,
as numpy and the kernel form it).  Everything after it is float64: reflect padding, the periodic Hann window centred at
lpad = (n_fft - win) // 2, rfft, |X|, the float64 `oracle.ref_features.mel_basis`, 20 log10(max(1e-5, .)), the
normalisation and the clip to [1e-8, 1].  With A_t = sum_n |w_n y_pad[n]| of frame t (ref_vocoder_stages.ref_stft):

  |X_k|       linear bound  b = tau * A_t                       (the FFT is the vocoder's fft_half)
  mel_m       linear bound  b = sum_k w_mk (tau A_t + 2^-24 a_k len_m) + 2^-24 mel_m
              (len_m: the filter's non-zero bins; the last term rounds the weights to float32)
  normalised  any value in [f(max(0, a - b)) - Q, f(a + b) + Q],  f(a) = clip((20 log10 max(1e-5, a) - ref_db + max_db)
              / max_db, 1e-8, 1) and Q = 4 * 2^-24 (1 + |dB| / max_db) for log10f and the normalisation.  f is monotone,
              so away from the edges this is b * 20 / (ln 10 max_db a) + Q to first order; where a +- b crosses the 1e-5
              floor or a clip edge the bin is ill-conditioned and the interval says so for that bin alone.
  energies    |got - ref| <= tau * ref per frame (ref_vocoder_stages.check_energies)
  trims       equal to the float64 trim decision, unless a frame lies within 8.7 tau_energies dB of -60 dB

The measured "err / S" of an output is the smallest tau that passes its well-conditioned elements:
max (|got - ref| - Q - g 2^-24-terms) / (g * S), with g = 20 / (ln 10 max_db a) and S = A_t (|X|) or sum_k w_mk A_t (mel).
"""
import numpy as np
import scipy.fft

from dc_tts_b200.hyperparams import Hyperparams as hp
from oracle import ref_features as rf
from oracle import ref_vocoder as rv

import ref_vocoder_stages as rs
from ref_vocoder_stages import GUARD, LEVELS, guarded, intact, ref_energies  # noqa: F401  (re-exported for the test files)

EPS = 2.0 ** -24
# tau per n_fft for |X| and mel (the STFT's error model tau * A_t) and for the trim energies: about 3.5x the worst err / S
# measured on an H100 80GB HBM3 at 700 W over all rates of the size (DESIGN.md section 8d): mag 4.9e-8, 7.8e-8, 1.05e-7;
# mel 9.7e-9, 4.5e-9, 2.3e-9; energies 2.7e-7, 1.9e-7, 2.0e-7 at n_fft 1024, 2048, 4096.
TAU = {1024: dict(mag=1.7e-7, mel=3.4e-8, energies=9.3e-7),
       2048: dict(mag=2.7e-7, mel=1.6e-8, energies=6.7e-7),
       4096: dict(mag=3.7e-7, mel=8.2e-9, energies=6.8e-7)}


# ------------------------------------------------------------------------------------------------ float64 references
def as_float(wav):
    """int16 PCM as value / 32768 (exact), float32 as is -> float32."""
    return wav.astype(np.float32) / np.float32(32768.0) if wav.dtype == np.int16 else np.asarray(wav, np.float32)


def preemphasis32(y, prev=None):
    """utils.py:39 in float32: y[0], then y[u] - c * y[u - 1] (product and difference each rounded to float32).
    `prev` (a deliberately wrong variant): the first sample is y[0] - c * prev instead."""
    y = np.asarray(y, np.float32)
    c = np.float32(hp.preemphasis)
    first = y[:1] if prev is None else y[:1] - c * np.float32(prev)
    return np.concatenate([first, y[1:] - c * y[:-1]]).astype(np.float32)


def frames_of(length, hop):
    return 1 + length // hop


def ref_features(y, sr, n_fft, hop, win, n_mels=None):
    """Float64 features of the trimmed float32 waveform y -> dict(a (T, F) |X|, A (T,) sum |w y_pad|, mel (T, n_mels),
    W (n_mels, F) the float64 mel basis)."""
    n_mels = n_mels or hp.n_mels
    p = preemphasis32(y).astype(np.float64)
    T = frames_of(len(p), hop)
    yp = np.pad(p, n_fft // 2, mode="reflect")
    idx = np.arange(n_fft)[None, :] + hop * np.arange(T)[:, None]
    fr = yp[idx] * rv.hann_padded(n_fft, win, np.float64)
    a = np.abs(np.fft.rfft(fr, axis=-1))
    W = rf.mel_basis(sr, n_fft, n_mels)
    return dict(a=a, A=np.abs(fr).sum(-1), mel=a @ W.T, W=W)


def normalise(x):
    """utils.py:55-60 in float64: clip((20 log10 max(1e-5, x) - ref_db + max_db) / max_db, 1e-8, 1)."""
    db = 20.0 * np.log10(np.maximum(1e-5, x))
    return np.clip((db - hp.ref_db + hp.max_db) / hp.max_db, 1e-8, 1.0)


def features32(y, n_fft, hop, win, W, window=None, prev=None):
    """A float32 restatement: float32 window and frames, scipy's complex64 rfft, float32 |X|, float32 weights and
    accumulation, the dB step in float32 -> (mag (T, F), mel (T, n_mels)) normalised."""
    p = preemphasis32(y, prev)
    T = frames_of(len(p), hop)
    yp = np.pad(p, n_fft // 2, mode="reflect")
    idx = np.arange(n_fft)[None, :] + hop * np.arange(T)[:, None]
    w = rv.hann_padded(n_fft, win, np.float32) if window is None else np.asarray(window, np.float32)
    X = scipy.fft.rfft(yp[idx] * w, axis=-1)
    assert X.dtype == np.complex64
    a = np.abs(X)
    mel = a @ np.asarray(W, np.float32).T

    def norm32(x):
        db = np.float32(20.0) * np.log10(np.maximum(np.float32(1e-5), x))
        return np.clip((db - np.float32(hp.ref_db) + np.float32(hp.max_db)) / np.float32(hp.max_db), np.float32(1e-8),
                       np.float32(1.0))
    return norm32(a), norm32(mel)


def filter_lengths(W):
    return (W > 0).sum(-1)


# ------------------------------------------------------------------------------------------------ the bounds
def _unclipped(x):
    return (20.0 * np.log10(np.maximum(1e-5, x)) - hp.ref_db + hp.max_db) / hp.max_db


def check_normalised(got, a, S, Qlin, tau):
    """got (normalised, float32) against the float64 linear value a with linear bound tau * S + Qlin ->
    (worst ratio to the allowed interval, measured err / S over the well-conditioned elements)."""
    got = np.asarray(got, np.float64)
    b = tau * S + Qlin
    ref = normalise(a)
    lo, hi = normalise(np.maximum(a - b, 0.0)), normalise(a + b)
    db = 20.0 * np.log10(np.maximum(1e-5, a))
    Q = 4 * EPS * (1.0 + np.abs(db) / hp.max_db)
    d = got - ref
    ratio = np.where(d >= 0, d / (hi + Q - ref), -d / (ref - lo + Q))
    g = 20.0 / (np.log(10.0) * hp.max_db * np.maximum(a, 1e-5))
    ok = (a - b > 1e-5) & (_unclipped(a - b) > 1e-8) & (_unclipped(a + b) < 1.0) & (S > 0)
    meas = float(((np.abs(d) - Q - g * Qlin)[ok] / (g * S)[ok]).max()) if ok.any() else 0.0
    return float(ratio.max()), max(meas, 0.0)


def check_mag(got, ref, tau):
    """got (T, F) normalised magnitudes against ref_features' output."""
    return check_normalised(got, ref["a"], np.broadcast_to(ref["A"][:, None], ref["a"].shape), 0.0, tau)


def check_mel(got, ref, tau, rows=None):
    """got (n, n_mels) normalised mel rows of the frames `rows` (default all) against ref_features' output."""
    rows = np.arange(ref["a"].shape[0]) if rows is None else np.asarray(rows)
    W, mel, A = ref["W"], ref["mel"][rows], ref["A"][rows]
    S = A[:, None] * W.sum(-1)[None, :]
    Qlin = EPS * (filter_lengths(W)[None, :] + 1.0) * mel
    return check_normalised(got, mel, S, Qlin, tau)


def check_energies(got, y, tau):
    """Per-frame energies of one utterance y (float32) -> (ratio, err / ref)."""
    return rs.check_energies(np.asarray(got)[None], np.asarray(y, np.float32)[None], tau)


def trim_margin_db(tau):
    return 2 * 10.0 / np.log(10.0) * tau          # 8.7 tau dB: each of a frame's and the loudest frame's energy off by tau


def trims_agree(trim, y, tau):
    """The product's (start, end) of y equals the float64 trim decision -> True; False (not checked) when a frame's level
    lies within trim_margin_db(tau) of the -60 dB threshold."""
    mse = ref_energies(np.asarray(y, np.float32)[None])[0]
    db = 10 * np.log10(np.maximum(1e-10, mse)) - 10 * np.log10(np.maximum(1e-10, mse.max()))
    if np.abs(db + 60).min() < trim_margin_db(tau):
        return False
    want = rv.trim_indices(np.asarray(y, np.float32).astype(np.float64))
    assert tuple(int(v) for v in trim) == want, (tuple(trim), want)
    return True


# ------------------------------------------------------------------------------------------------ today's tolerances
def old_tolerance_passes(mel, mag, mel_ref, mag_ref):
    """The bar of tests/test_gpu_wav_features.py (1e-4 above 0.35 on the normalised scale, else rtol 2e-3 in amplitude
    plus 2e-6 of the peak) -> True when (mel, mag) pass it."""
    lin = lambda z: 10.0 ** ((np.asarray(z, np.float64) * hp.max_db - hp.max_db + hp.ref_db) / 20.0)
    for got, ref in ((mag, mag_ref), (mel, mel_ref)):
        g, r = lin(got), lin(ref)
        if not np.all(np.abs(g - r) <= 2e-6 * r.max() + 2e-3 * np.abs(r)):
            return False
        loud = np.asarray(ref) > 0.35
        if loud.any() and np.abs(np.asarray(got, np.float64) - ref)[loud].max() >= 1e-4:
            return False
    return True


# ------------------------------------------------------------------------------------------------ inputs
def clip(rng, n, sr, level=1.0, lead=0, tail=0, quiet=1e-5, tone=False, hush=False):
    """A speech-like float64 waveform of n samples at sr: a harmonic voice with vibrato and an envelope plus noise, scaled
    to `level`; `lead` / `tail` samples at `quiet` of it (trimmed away); `tone`: a loud 400 Hz full-scale stretch (the
    clip at 1); `hush`: a stretch at 1e-9 of the level inside (the 1e-5 floor and the 1e-8 clip)."""
    t = np.arange(n) / sr
    f0 = 110 + 120 * rng.random() + 6 * np.sin(2 * np.pi * 5 * t)
    ph = 2 * np.pi * np.cumsum(f0) / sr
    y = sum(0.25 / h * np.sin(h * ph + rng.random()) for h in range(1, 12))
    y = y * (0.55 + 0.45 * np.sin(2 * np.pi * 2.5 * t + rng.random())) + 0.03 * rng.standard_normal(n)
    y = 0.8 * y / max(1e-12, np.abs(y).max())
    if tone and n > 8:
        i, m = n // 3, max(2, n // 6)
        y[i:i + m] = 0.999 * np.sin(2 * np.pi * 400 * np.arange(m) / sr)
    if hush and n > 8:
        y[2 * n // 3:2 * n // 3 + max(2, n // 8)] *= 1e-9
    y *= level
    y[:lead] *= quiet
    if tail:
        y[n - tail:] *= quiet
    return y


def as_dtype(y, kind):
    """float64 -> int16 PCM (rounded, saturated) or float32."""
    if kind == "int16":
        return np.clip(np.round(y * 32767), -32768, 32767).astype(np.int16)
    return y.astype(np.float32)
