"""Resampling as librosa.load(fpath, sr=hp.sr) does it (librosa 0.6 / resampy 0.2 'kaiser_best'), on the CPU: the time
register of the device kernel (dctts_resample_time_register, no GPU) against the sequential float64 sum, the oracle
(oracle/ref_resample.py) as a resampler, the readers' native rates, the five-field transcript of the reference's other
corpora, and the mixed-rate wav route of the trainer with the oracle standing in for the device call."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

from dc_tts_b200 import _lib, trainer, utils
from dc_tts_b200.hyperparams import Hyperparams as hp
from oracle import ref_features as rf
from oracle import ref_resample as rr

REF = "/root/reference"
HAVE_REF = os.path.isdir(REF)
RATES = [8000, 11025, 16000, 24000, 32000, 44100, 48000, 96000]


def _segments(n_out, sr_in, sr_out):
    lib = _lib.load()
    cap = 4096
    t0, v0, st = np.zeros(cap, np.int64), np.zeros(cap), np.zeros(cap)
    n = lib.dctts_resample_time_register(n_out, sr_in, sr_out, t0.ctypes.data_as(C.POINTER(C.c_int64)),
                                         v0.ctypes.data_as(C.POINTER(C.c_double)), st.ctypes.data_as(C.POINTER(C.c_double)), cap)
    assert n >= 0
    return t0[:n], v0[:n], st[:n]


def _expand(n_out, t0, v0, st):
    """register(t) = v0 + (t - t0) step over each segment, in float64 (exact: see TimeSeg)."""
    reg = np.empty(n_out)
    ends = list(t0[1:]) + [n_out]
    for a, e, v, s in zip(t0, ends, v0, st):
        reg[a:e] = v + np.arange(e - a, dtype=np.float64) * s
    return reg


def _tie_binade(inc):
    """The binade [2^k, 2^(k+1)) whose grid g = 2^(k-52) has inc / g exactly halfway between integers, as k."""
    m, e = math.frexp(inc)
    mant = int(m * 2 ** 53)
    low = (mant & -mant).bit_length() - 1                       # lowest set bit of the 53-bit mantissa
    return (e - 53 + low) + 53                                  # g / 2 = 2^(e - 53 + low)


@pytest.mark.parametrize("sr_in", RATES)
def test_time_register_segments_equal_the_sequential_sum(sr_in):
    n_out = 1 << 24
    t0, v0, st = _segments(n_out, sr_in, 22050)
    assert t0[0] == 0 and np.all(np.diff(t0) > 0) and len(t0) < 200
    ref = rr.time_register(n_out, 22050.0 / sr_in)
    assert np.array_equal(_expand(n_out, t0, v0, st), ref)


def test_time_register_random_rate_pairs():
    rng = np.random.default_rng(0)
    ties = 0
    for _ in range(300):
        sr_in, sr_out = (int(v) for v in rng.integers(4000, 192001, 2))
        if sr_in == sr_out:
            continue
        n_out = int(rng.integers(1, 300000))
        t0, v0, st = _segments(n_out, sr_in, sr_out)
        ref = rr.time_register(n_out, float(sr_out) / sr_in)
        assert np.array_equal(_expand(n_out, t0, v0, st), ref), (sr_in, sr_out, n_out)
        ties += 2.0 ** _tie_binade(1. / (float(sr_out) / sr_in)) < ref[-1]
    assert ties > 20                                             # the round-half-to-even branch was exercised


def _i0_series(x):
    s, term, k = 0.0, 1.0, 0
    q = (x / 2.0) ** 2
    while term > 1e-300 and (k < 5 or term > s * 1e-18):
        s += term
        k += 1
        term *= q / (k * k)
    return s


def test_kaiser_window_and_table():
    M, beta = 2 * 64 * 512 + 1, rr.BETA
    w = rr.kaiser(M, beta)
    idx = np.r_[0:M:997, M // 2, M - 1]
    alpha = (M - 1) / 2.0
    ref = np.array([_i0_series(beta * math.sqrt(1 - ((n - alpha) / alpha) ** 2)) / _i0_series(beta) for n in idx])
    assert np.abs(w[idx] - ref).max() < 1e-15
    win, num_table, rolloff = rr.sinc_window()
    assert win.shape == (64 * 512 + 1,) and num_table == 512 and win[0] == rolloff == rr.ROLLOFF


def _tone(sr, f, seconds, amp=0.5, phase=0.3):
    t = np.arange(int(sr * seconds)) / sr
    return (amp * np.sin(2 * np.pi * f * t + phase)).astype(np.float32)


# Bounds are about twice the maxima measured on this oracle (DESIGN.md 8d).  Rates whose ratio times 512 is not an
# integer (48, 32, 24, 96 kHz) sample the filter with resampy's truncated index_step, which moves the cutoff: larger
# passband errors near it and less stopband attenuation than the exact ratios 1/2 (44.1 kHz) or above 1.
@pytest.mark.parametrize("sr_in,f,bound", [(44100, 3000.0, 1e-6), (16000, 5000.0, 3e-6), (8000, 3000.0, 3e-6),
                                           (11025, 4000.0, 1e-6), (48000, 9000.0, 1e-3), (24000, 9000.0, 1.5e-3),
                                           (32000, 9000.0, 3.5e-3), (96000, 8000.0, 5e-3)])
def test_oracle_passes_tones_below_the_rolloff(sr_in, f, bound):
    """A 0.5-amplitude tone below rolloff * min(sr_in, 22050) / 2 comes out as the analytic tone at 22050 Hz."""
    y = rr.librosa_resample(_tone(sr_in, f, 0.5), sr_in, 22050)
    n = int(0.5 * sr_in * (22050.0 / sr_in))
    ref = _tone(22050, f, n / 22050 + 1.0)[:y.size].astype(np.float64)
    err = np.abs(y[200:n - 200] - ref[200:n - 200]).max()
    assert err < bound, err


@pytest.mark.parametrize("sr_in,f,db", [(44100, 12500.0, -130), (44100, 15000.0, -130), (48000, 13000.0, -70),
                                        (96000, 20000.0, -70), (32000, 12000.0, -55)])
def test_oracle_attenuates_tones_above_the_new_nyquist(sr_in, f, db):
    y = rr.librosa_resample(_tone(sr_in, f, 0.5), sr_in, 22050)
    rms = np.sqrt(np.mean(y[300:-300].astype(np.float64) ** 2))
    assert 20 * np.log10(rms / (0.5 / np.sqrt(2))) < db, rms


@pytest.mark.parametrize("sr_in,bound", [(44100, 5e-5), (16000, 5e-5), (48000, 1.2e-3)])
def test_oracle_agrees_with_resample_poly_on_band_limited_noise(sr_in, bound):
    """White noise low-passed to 0.6 of the lower Nyquist frequency, against scipy's polyphase resampler."""
    import scipy.signal as ss
    from fractions import Fraction
    rng = np.random.default_rng(1)
    x = rng.standard_normal(int(sr_in * 0.6))
    sos = ss.butter(16, 0.6 * min(sr_in, 22050) / 2, fs=sr_in, output="sos")
    x = (0.2 * ss.sosfiltfilt(sos, x)).astype(np.float32)
    y = rr.librosa_resample(x, sr_in, 22050)
    fr = Fraction(22050, sr_in)
    z = ss.resample_poly(x.astype(np.float64), fr.numerator, fr.denominator, window=("kaiser", 14.0))
    m = min(y.size, z.size)
    err = np.abs(y[500:m - 500] - z[500:m - 500]).max() / np.abs(z).max()
    assert err < bound, err


def test_output_length_identity_and_too_short():
    for n, sr_in in [(1000, 44100), (999, 44100), (1001, 16000), (123457, 48000), (7, 8000)]:
        y = rr.librosa_resample(np.ones(n, np.float32), sr_in, 22050)
        ratio = 22050.0 / sr_in
        assert y.size == int(np.ceil(n * ratio))
        assert (y.size > int(n * ratio)) == (y[-1] == 0) or int(n * ratio) == y.size
        assert not y[int(n * ratio):].any()
    x = np.random.default_rng(0).standard_normal(500).astype(np.float32)
    assert rr.librosa_resample(x, 22050, 22050) is not None and np.array_equal(rr.librosa_resample(x, 22050, 22050), x)
    with pytest.raises(ValueError, match="too small"):
        rr.librosa_resample(np.ones(1, np.float32), 44100, 22050)


def test_read_pcm_returns_the_native_rate_and_stereo_is_scaled_then_averaged(tmp_path):
    from scipy.io import wavfile
    rng = np.random.default_rng(2)
    a = rng.integers(-20000, 20000, 3000).astype(np.int16)
    b = rng.integers(-20000, 20000, 3000).astype(np.int16)
    wavfile.write(str(tmp_path / "m.wav"), 44100, a)
    wavfile.write(str(tmp_path / "s.wav"), 16000, np.stack([a, b], 1))
    y, sr = utils._read_pcm(str(tmp_path / "m.wav"))
    assert sr == 44100 and y.dtype == np.int16 and np.array_equal(y, a)
    y, sr = utils._read_pcm(str(tmp_path / "s.wav"))
    want = ((a.astype(np.float32) / 32768.0 + b.astype(np.float32) / 32768.0) / 2).astype(np.float32)
    assert sr == 16000 and y.dtype == np.float32 and np.array_equal(y, want) and np.abs(y).max() < 1
    wavfile.write(str(tmp_path / "s22.wav"), hp.sr, np.stack([a, b], 1))
    assert np.array_equal(utils._load_wav(str(tmp_path / "s22.wav")), want)
    with pytest.raises(ValueError, match="sample rate"):
        utils._load_pcm(str(tmp_path / "m.wav"))


# ------------------------------------------------------------------------------------------- the other transcript format
def _five_field(root, lines):
    d = root / "kate"
    d.mkdir()
    (d / "transcript.csv").write_text("\n".join(lines) + "\n", encoding="utf-8")
    return str(d)


def test_five_field_transcript(tmp_path):
    """data_load.py:59-77: clips over 10 s skipped, the path joined as written, no normalisation (hp.vocab only)."""
    d = _five_field(tmp_path, ["a/one.wav|x|hello  there.|0|3.5", "a/two.wav|x|too long|0|10.5",
                               "b/three.wav|x|keep it?|1|10.0"])
    fpaths, lens, texts = trainer.load_train_data(d)
    assert fpaths == [os.path.join(d, "a/one.wav"), os.path.join(d, "b/three.wav")]
    idx = {c: i for i, c in enumerate(hp.vocab)}
    assert [t.tolist() for t in texts] == [[idx[c] for c in "hello  there.E"], [idx[c] for c in "keep it?E"]]
    assert lens == [len(t) for t in texts] and all(t.dtype == np.int32 for t in texts)


def test_five_field_transcript_names_the_line_of_a_character_outside_the_vocabulary(tmp_path):
    d = _five_field(tmp_path, ["a.wav|x|fine|0|1.0", "b.wav|x|Not fine|0|1.0"])
    with pytest.raises(ValueError, match=r"transcript.csv:2: character 'N' is not in hp.vocab"):
        trainer.load_train_data(d)


# ------------------------------------------------------------------------------------------- mixed-rate wav route
def _clip(rng, sr, seconds):
    n = int(sr * seconds)
    t = np.arange(n) / sr
    y = 0.3 * np.sin(2 * np.pi * rng.uniform(120, 300) * t) * (0.5 + 0.5 * np.sin(2 * np.pi * 3 * t)) + 0.03 * rng.standard_normal(n)
    lead, tail = int(rng.integers(800, 3000)) * sr // hp.sr, int(rng.integers(800, 3000)) * sr // hp.sr
    y[:lead] *= 1e-4
    y[n - tail:] *= 1e-4
    return np.round(np.clip(y, -1, 1) * 32767).astype(np.int16)


def oracle_features(pcms, rates=None):
    """What the batched device call returns, from the oracle: resample, then each utterance's load_spectrograms, padded."""
    rates = rates or [hp.sr] * len(pcms)
    out = [rf.load_spectrograms(rr.load(p, r, hp.sr)) for p, r in zip(pcms, rates)]
    T_b = max(m.shape[0] for m, _ in out)
    mels = np.zeros((len(out), T_b, hp.n_mels), np.float32)
    mags = np.zeros((len(out), hp.r * T_b, 1 + hp.n_fft // 2), np.float32)
    for b, (m, g) in enumerate(out):
        mels[b, :m.shape[0]] = m; mags[b, :g.shape[0]] = g
    return mels, mags


def test_mixed_rate_wav_route_yields_the_npy_routes_batches(tmp_path):
    from scipy.io import wavfile
    rng = np.random.default_rng(4)
    d = tmp_path / "LJSpeech-1.0"
    (d / "wavs").mkdir(parents=True)
    (tmp_path / "mels").mkdir(); (tmp_path / "mags").mkdir()
    lines = []
    for i in range(10):
        name, sr = "LJ%03d" % i, [hp.sr, 16000, 44100, 48000][i % 4]
        lines.append("%s|raw|%s" % (name, "".join(rng.choice(list("abcdefghij '"), int(rng.integers(10, 60))))))
        pcm = _clip(rng, sr, float(rng.uniform(0.25, 0.6)))
        wavfile.write(str(d / "wavs" / (name + ".wav")), sr, pcm)
        mel, mag = rf.load_spectrograms(rr.load(pcm, sr, hp.sr))
        np.save(tmp_path / "mels" / (name + ".npy"), mel); np.save(tmp_path / "mags" / (name + ".npy"), mag)
    (d / "transcript.csv").write_text("\n".join(lines) + "\n", encoding="utf-8")
    fpaths, lens, texts = trainer.load_train_data(str(d))
    loader = lambda p: trainer._load_spectrograms_npy(p, str(tmp_path / "mels"), str(tmp_path / "mags"))
    calls = []

    def features(pcms, rates=None):
        calls.append(rates)
        return oracle_features(pcms, rates)
    kw = dict(B=2, seed=5, epochs=2)
    npy = list(trainer.bucketed_batches(fpaths, lens, texts, loader=loader, prepro=True, **kw))
    with pytest.raises(ValueError, match="resample=True"):    # other rates are refused unless asked for
        list(trainer.bucketed_batches(fpaths, lens, texts, loader=None, prepro=False, features=features, **kw))
    calls.clear()
    wav = list(trainer.bucketed_batches(fpaths, lens, texts, loader=None, prepro=False, features=features, resample=True, **kw))
    assert len(npy) == len(wav) > 2 and any(r is not None for r in calls)
    for (L0, m0, g0, n0, k0), (L1, m1, g1, n1, k1) in zip(npy, wav):
        assert n0 == n1 and k0 == k1 and np.array_equal(L0, L1)
        assert np.array_equal(m0, m1) and np.array_equal(g0, g1)


# ------------------------------------------------------------------------------------------- the reference's own code
@pytest.fixture
def isolated_modules():
    """The reference's modules (and the stand-ins for TensorFlow and librosa they import) leave with the test."""
    before, path = set(sys.modules), list(sys.path)
    yield
    for m in set(sys.modules) - before:
        del sys.modules[m]
    sys.path[:] = path


def _ref_import(name):
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    import tf_shim
    tf_shim.install(tf_shim.Store({}))
    sys.path.insert(0, REF)
    return __import__(name)


@pytest.mark.skipif(not HAVE_REF, reason="the reference checkout is not present")
def test_reference_get_spectrograms_with_the_oracle_resampler(monkeypatch, tmp_path, isolated_modules):
    import types
    from oracle import ref_vocoder as rv
    from scipy.io import wavfile
    ref_utils = _ref_import("utils")
    rng = np.random.default_rng(6)
    pcm = _clip(rng, 44100, 0.5)
    path = str(tmp_path / "k.wav")
    wavfile.write(path, 44100, pcm)

    def load(fpath, sr=None):
        y, native = utils._read_pcm(fpath)
        return rr.load(y, native, sr), sr
    lib = types.SimpleNamespace(
        stft=lambda y, n_fft=None, hop_length=None, win_length=None: rv.stft(np.asarray(y, np.float32), n_fft, hop_length, win_length),
        effects=types.SimpleNamespace(trim=lambda y: (lambda se: (y[se[0]:se[1]], se))(rv.trim_indices(np.asarray(y)))),
        filters=types.SimpleNamespace(mel=lambda sr, n_fft, n_mels: rf.mel_basis(sr, n_fft, n_mels)),
        load=load)
    monkeypatch.setattr(ref_utils, "librosa", lib)
    mel, mag = ref_utils.get_spectrograms(path)
    mel2, mag2 = rf.get_spectrograms(rr.load(pcm, 44100, hp.sr))
    assert mel.shape == mel2.shape and np.abs(mel - mel2).max() < 1e-6 and np.abs(mag - mag2).max() < 1e-6


@pytest.mark.skipif(not HAVE_REF, reason="the reference checkout is not present")
def test_reference_load_data_on_a_five_field_transcript(monkeypatch, tmp_path, isolated_modules):
    import types
    ref_dl = _ref_import("data_load")
    import hyperparams as ref_hp

    class _Arr(np.ndarray):
        def tostring(self):                                     # numpy 1.x, which the reference was written for
            return self.tobytes()
    monkeypatch.setattr(ref_dl, "np", types.SimpleNamespace(array=lambda a, dt: np.array(a, dt).view(_Arr), int32=np.int32))
    d = _five_field(tmp_path, ["x/a.wav|r|abc def.|0|2.0", "x/b.wav|r|gone|0|12.0", "y/c.wav|r|why? ok|1|9.99"])
    monkeypatch.setattr(ref_hp.Hyperparams, "data", d)
    monkeypatch.setattr(ref_dl.hp, "data", d)
    fpaths, lens, texts = ref_dl.load_data()
    mine = trainer.load_train_data(d)
    assert fpaths == mine[0] and lens == mine[1]
    assert [np.frombuffer(t, np.int32).tolist() for t in texts] == [t.tolist() for t in mine[2]]
