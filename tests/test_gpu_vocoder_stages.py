"""The Griffin-Lim vocoder one stage at a time (dctts_vocoder_stage) against float64, and the feature extraction, at
n_fft 1024 (16 kHz), 2048 (22.05 kHz) and 4096 (44.1 kHz): the STFT kernels' three instantiations.

`tests/test_vocoder.py` compares whole waveforms with the float32 oracle to 2e-3 of the peak, about 1000x what a float32
implementation of the chain gets wrong; this file holds each stage of `dctts_spectrogram2wav` to its own float64 reference
and bound (tests/ref_vocoder_stages.py, whose float32 and degraded chains tests/test_vocoder_sizes.py checks on the CPU).
Every input and output lies inside a larger allocation with NaN guards on both sides; the guards and the outputs are
checked afterwards.  At 1024 and 4096 the stages run at the rate's (hop, win) plus win = n_fft and n_fft - 1; features are
held to the oracle composition with the tolerances of test_gpu_wav_features.py.  Engines are built and run inside
`at_rate` (Hyperparams at that corpus rate), because an engine reads hop and win from Hyperparams at call time.
Case ids name n_fft where it is not the hyperparameters' default 2048.
"""
import numpy as np
import pytest
import torch

from dc_tts_b200.engine import DcttsError
from dc_tts_b200.hyperparams import Hyperparams as hp
from oracle import ref_features as rf
from oracle import ref_vocoder as rv

import ref_vocoder_stages as rs
from ref_vocoder_stages import HOP_WIN, TAU
from sample_rates import at_rate

pytestmark = pytest.mark.gpu
SR = {1024: 16000, 2048: 22050, 4096: 44100}
LENGTHS = {2048: (2, 3, 4, 5, 8, 60, 513, 840), 1024: (2, 3, 5, 60, 840), 4096: (2, 3, 5, 60, 840)}
# the rate's own (hop, win) and the (T, B) of the de-emphasis and energy cases at 1024 and 4096
RATE_HOP_WIN = {1024: (200, 800), 4096: (551, 2205)}
RATE_T_B = ((3, 3), (840, 3), (60, 32))
_WORST = {}


def _record(n, stage, raw):
    _WORST[(n, stage)] = max(_WORST.get((n, stage), 0.0), float(raw))


def _pre(n):
    return "" if n == 2048 else "n%d-" % n


def _matrix():
    """(n_fft, hop, win, T, B, istft seed, stft_phase seed) for every (hop, win) and T of the size."""
    cases = []
    for n, hws in HOP_WIN.items():
        for i, ((hop, win), T) in enumerate((hw, T) for hw in hws for T in LENGTHS[n]):
            B = rs.case_batch(i)
            if T * hop > 120000 and B == 32:
                B = 3
            seeds = (T + hop, T * hop + 1) if n == 2048 else (T + hop + win, T * hop + win)
            cases.append((n, hop, win, T, B) + seeds)
    return cases


CASES = _matrix()
IDS = [_pre(c[0]) + "hop%d-win%d-T%d-B%d" % c[1:5] for c in CASES]
# de-emphasis and energies: the whole matrix at 2048 (with a quiet lead and tail for trimming to work on), the rate's
# (hop, win) at the other sizes
TAIL_CASES = [(n, hop, win, T, B, True) for n, hop, win, T, B, _, _ in CASES if n == 2048] + \
             [(n,) + RATE_HOP_WIN[n] + tb + (False,) for n in (1024, 4096) for tb in RATE_T_B]
TAIL_IDS = [_pre(c[0]) + "hop%d-win%d-T%d-B%d" % c[1:5] for c in TAIL_CASES]


@pytest.fixture(scope="module")
def engines():
    from dc_tts_b200.engine import Engine
    out = {}
    for n in SR:
        with at_rate(SR[n], n) as H:
            out[n] = Engine(0, hparams=H)
    yield out
    print("\nvocoder stages, worst err / bound scale: " +
          ", ".join("n_fft %d %s %.3g" % (k + (v,)) for k, v in sorted(_WORST.items())))
    for e in out.values():
        e.close()


@pytest.fixture
def eng(engines):
    """The default 2048-point engine at the default rate."""
    return engines[2048]


PREPARE = [(2048, T, B, p) for T, B in [(2, 1), (3, 3), (60, 32), (513, 3), (840, 32)] for p in (1.5, 1.0)] + \
          [(n, T, B, 1.5) for T, B in [(2, 1), (5, 3), (60, 32), (840, 3)] for n in (1024, 4096)]


@pytest.mark.parametrize("n,T,B,power", PREPARE, ids=[("%d-%d-%s" % (T, B, p)) if n == 2048 else "n%d-T%d-B%d" % (n, T, B)
                                                      for n, T, B, p in PREPARE])
def test_prepare(engines, n, T, B, power):
    eng = engines[n]
    with at_rate(SR[n], n):
        mag = rs.make_mag(np.random.default_rng(T * B), B, T, n)
        bi, vi = rs.guarded(eng, mag.shape, torch.float32, mag)
        bo, vo = rs.guarded(eng, mag.shape, torch.complex64)
        eng.vocoder_stage(0, vi, vo, power=power)
        rs.intact(bi, vi)
        X = rs.intact(bo, vo)
    assert not X.imag.any()
    ratio, raw = rs.check_prepare(X.real, mag, power, TAU[n]["prepare"])
    _record(n, "prepare", raw)
    assert ratio <= 1, (ratio, raw)


@pytest.mark.parametrize("n,hop,win,T,B,seed,_", CASES, ids=IDS)
def test_istft(engines, n, hop, win, T, B, seed, _):
    eng = engines[n]
    with at_rate(SR[n], n):
        X = rs.make_spectrum(np.random.default_rng(seed), B, T, n)
        bi, vi = rs.guarded(eng, X.shape, torch.complex64, X)
        bo, vo = rs.guarded(eng, (B, hop * (T - 1)), torch.float32)
        eng.vocoder_stage(1, vi, vo, hop=hop, win=win)
        assert np.array_equal(rs.intact(bi, vi), X)
        ratio, raw = rs.check_istft(rs.intact(bo, vo), X, hop, win, TAU[n]["istft"])
    _record(n, "istft", raw)
    assert ratio <= 1, (ratio, raw)


@pytest.mark.parametrize("n,hop,win,T,B,_,seed", CASES, ids=IDS)
def test_stft_phase(engines, n, hop, win, T, B, _, seed):
    """T = 2 and 3 put the n_fft / 2 reflect padding past a short signal: np.pad reflects it again and again."""
    eng = engines[n]
    with at_rate(SR[n], n):
        rng = np.random.default_rng(seed)
        Ly = hop * (T - 1)
        y = rs.make_wav(rng, B, Ly)
        S = rng.uniform(0, 2, (B, T, 1 + n // 2)).astype(np.float32) * np.array(rs.LEVELS * B, np.float32)[:B, None, None]
        S[:, :, ::97] = 0.0
        bi, vi = rs.guarded(eng, (B, Ly), torch.float32, y)
        bs, vs = rs.guarded(eng, S.shape, torch.float32, S)
        bo, vo = rs.guarded(eng, S.shape, torch.complex64)
        eng.vocoder_stage(2, vi, vo, S=vs, hop=hop, win=win)
        rs.intact(bi, vi)
        rs.intact(bs, vs)
        ratio, raw = rs.check_stft_phase(rs.intact(bo, vo), y, S, hop, win, TAU[n]["stft"])
    _record(n, "stft", raw)
    assert ratio <= 1, (ratio, raw)


@pytest.mark.parametrize("n,hop,win,T,B,_", TAIL_CASES, ids=TAIL_IDS)
def test_deemph(engines, n, hop, win, T, B, _):
    """The de-emphasis does not depend on n_fft, but it passes the handle's checks at every size."""
    eng = engines[n]
    with at_rate(SR[n], n):
        Ly = hop * (T - 1)
        x = rs.make_deemph_input(np.random.default_rng(Ly), B, Ly)
        bw, vw = rs.guarded(eng, (B, Ly), torch.float32, x)
        eng.vocoder_stage(3, vw, vw, hop=hop, win=win)
        ulps, exact = rs.check_deemph(rs.intact(bw, vw), x)
    _record(n, "deemph_ulps", ulps)
    _record(n, "deemph_inexact", 1 - exact)
    assert ulps <= 1 and exact >= 0.999, (ulps, exact)


@pytest.mark.parametrize("n,hop,win,T,B,quiet_ends", TAIL_CASES, ids=TAIL_IDS)
def test_energies_and_trims(engines, n, hop, win, T, B, quiet_ends):
    """The trim frames stay 2048 / 512 at every rate; the stage passes the handle's checks at every size."""
    eng = engines[n]
    with at_rate(SR[n], n):
        Ly = hop * (T - 1)
        y = rs.make_wav(np.random.default_rng(Ly + 7), B, Ly)
        if quiet_ends:                                       # quiet lead and tail, so that trimming has work to do
            for b in range(B):
                y[b, :Ly // 5] *= 1e-4
                y[b, Ly - Ly // 6:] *= 1e-4
        bi, vi = rs.guarded(eng, (B, Ly), torch.float32, y)
        bo, vo = rs.guarded(eng, (B, 1 + Ly // 512), torch.float32)
        trim = eng.vocoder_stage(4, vi, vo, hop=hop, win=win)
        rs.intact(bi, vi)
        ratio, raw = rs.check_energies(rs.intact(bo, vo), y, TAU[n]["energies"])
    _record(n, "energies", raw)
    assert ratio <= 1, (ratio, raw)
    rs.trims_agree(trim, y)


@pytest.mark.parametrize("T", [2, 3, 60, 513])
def test_spectrogram2wav_without_iterations_is_the_float64_chain(eng, T):
    """prepare -> istft -> de-emphasis in one product call at n_iter = 0: linear and well conditioned, so held to the sum of
    the stage bounds carried through the de-emphasis filter (plus the final float32 rounding)."""
    B, hop, win = 3, hp.hop_length, hp.win_length
    mag = rs.make_mag(np.random.default_rng(T + 11), B, T, 2048)
    wav, trim = eng.spectrogram2wav(mag, n_iter=0)
    wav = wav.cpu().numpy()
    S = rs.ref_prepare(mag, hp.power)
    y, A = rs.ref_istft(S.astype(np.complex128), hop, win)
    ref, bound = rs.ref_deemph(y), rs.ref_deemph((TAU[2048]["istft"] + TAU[2048]["prepare"]) * A)
    err = np.abs(wav - ref)
    ratio = float((err / (bound + 2.0 ** -23 * np.abs(ref) + 1e-37)).max())
    _record(2048, "n_iter0", float((err / (rs.ref_deemph(A) + 1e-37)).max()))
    assert ratio <= 1, ratio
    rs.trims_agree(trim, wav)


ONE_ITERATION = [(2048, 2, 275, 1102), (2048, 3, 275, 1102), (2048, 60, 200, 800), (2048, 513, 275, 1102)] + \
                [(n, T) + RATE_HOP_WIN[n] for T in (2, 3, 60) for n in (1024, 4096)]


@pytest.mark.parametrize("n,T,hop,win", ONE_ITERATION, ids=[_pre(c[0]) + "%d-%d-%d" % c[1:] for c in ONE_ITERATION])
def test_one_iteration_is_the_stages_bit_for_bit(engines, n, T, hop, win):
    """dctts_spectrogram2wav at n_iter = 1 issues exactly the stages' launches: prepare, istft, stft_phase, istft, deemph,
    energies."""
    eng = engines[n]
    with at_rate(SR[n], n):
        B = 3
        mag = torch.from_numpy(rs.make_mag(np.random.default_rng(T), B, T, n)).to(eng.device)
        Ly = hop * (T - 1)
        X = torch.empty(B, T, 1 + n // 2, dtype=torch.complex64, device=eng.device)
        y = torch.empty(B, Ly, device=eng.device)
        mse = torch.empty(B, 1 + Ly // 512, device=eng.device)
        kw = dict(hop=hop, win=win)
        eng.vocoder_stage(0, mag, X, **kw)                   # also sets the handle's vocoder parameters to (hop, win)
        wav = torch.empty(B, Ly, device=eng.device)
        trim = np.zeros((B, 2), np.int32)
        eng._check(eng._lib.dctts_spectrogram2wav(eng._h, mag.data_ptr(), B, T, 1, wav.data_ptr(), trim.ctypes.data,
                                                  eng._stream()), "dctts_spectrogram2wav")
        S = X.real.contiguous()
        eng.vocoder_stage(1, X, y, **kw)
        X2 = torch.empty_like(X)
        eng.vocoder_stage(2, y, X2, S=S, **kw)
        eng.vocoder_stage(1, X2, y, **kw)
        eng.vocoder_stage(3, y, y, **kw)
        trim2 = eng.vocoder_stage(4, y, mse, **kw)
    assert torch.equal(wav, y) and np.array_equal(trim, trim2)


@pytest.mark.parametrize("n", (1024, 4096))
@pytest.mark.parametrize("T,n_iter", [(60, 5), (840, 3)])
def test_spectrogram2wav_vs_the_oracle(engines, n, T, n_iter):
    """The whole chain against ref_vocoder's float32 composition at the size's rate, to 2e-3 of the peak as
    test_vocoder.py holds it at 2048."""
    eng = engines[n]
    with at_rate(SR[n], n) as H:
        mag = np.random.default_rng(T + n).uniform(0.1, 0.95, (2, T, 1 + n // 2)).astype(np.float32)
        mag[1, T // 2:] *= 0.05
        wav, trim = eng.spectrogram2wav(mag, n_iter=n_iter)
        wav = wav.cpu().numpy()
        assert wav.shape == (2, H.hop_length * (T - 1))
        for b in range(2):
            _, se, full = rv.spectrogram2wav(mag[b], n_iter=n_iter)
            scale = np.abs(full).max()
            assert np.abs(wav[b] - full).max() < 2e-3 * scale, (b, np.abs(wav[b] - full).max(), scale)
            assert abs(int(trim[b, 0]) - se[0]) <= 512 and abs(int(trim[b, 1]) - se[1]) <= 512


def test_refusals(eng):
    dev, F = eng.device, 1 + 2048 // 2
    with pytest.raises(DcttsError, match="T >= 2"):
        eng.vocoder_stage(0, torch.zeros(1, 1, F, device=dev), torch.zeros(1, 1, F, dtype=torch.complex64, device=dev))
    with pytest.raises(DcttsError, match="stage 7"):
        eng.vocoder_stage(7, torch.zeros(1, 4, F, device=dev), torch.zeros(1, 4, F, device=dev))
    with pytest.raises(DcttsError, match="shape"):
        eng.vocoder_stage(2, torch.zeros(1, 275 * 3, device=dev), torch.zeros(1, 4, F, dtype=torch.complex64, device=dev),
                          S=torch.zeros(1, 4, F - 1, device=dev))
    y = torch.zeros(2, 275 * 3, device=dev)
    with pytest.raises(DcttsError, match="in place"):
        eng._check(eng._lib.dctts_vocoder_stage(eng._h, 3, 2, 4, y.data_ptr(), None, torch.zeros_like(y).data_ptr(), None,
                                                eng._stream()), "dctts_vocoder_stage")
    mag = np.random.default_rng(0).uniform(0.2, 0.8, (1, 5, F)).astype(np.float32)
    eng.spectrogram2wav(mag, n_iter=1)                  # the handle stays usable


@pytest.mark.parametrize("n_fft", [512, 8192])
def test_unsupported_sizes_are_refused(n_fft):
    from dc_tts_b200.engine import Engine
    with at_rate(48000, n_fft) as H:
        H.win_length = min(H.win_length, n_fft)
        e = Engine(0, hparams=H)
        F = 1 + n_fft // 2
        with pytest.raises(DcttsError, match="supported: 1024, 2048, 4096"):
            e.spectrogram2wav(np.full((1, 5, F), 0.5, np.float32), n_iter=1)
        with pytest.raises(DcttsError, match="supported: 1024, 2048, 4096"):
            e.load_spectrograms_batch([np.zeros(4000, np.float32) + 0.1])
        e.close()


def test_window_longer_than_n_fft_is_refused(engines):
    eng = engines[1024]
    with at_rate(SR[1024], 1024):
        with pytest.raises(DcttsError, match="exceeds n_fft = 1024"):
            eng._check(eng._lib.dctts_set_vocoder_params(eng._h, 200, 1025, 1.5, 100.0, 20.0, 0.97, 1),
                       "dctts_set_vocoder_params")
        # the stock 22.05 kHz window (1102 taps) does not fit a 1024-point frame either
        with pytest.raises(DcttsError, match="exceeds n_fft"):
            eng._check(eng._lib.dctts_set_vocoder_params(eng._h, 275, 1102, 1.5, 100.0, 20.0, 0.97, 1),
                       "dctts_set_vocoder_params")
        mag = np.full((1, 5, 513), 0.5, np.float32)
        wav, _ = eng.spectrogram2wav(mag, n_iter=1)            # the handle stays usable
        assert wav.shape[1] == 200 * 4


# ------------------------------------------------------------------------------------------------ features
@pytest.mark.parametrize("kind", ["int16", "float32"])
def test_short_clip_features_follow_np_pad(eng, kind):
    """Clips shorter than the n_fft / 2 padding (after trimming) are reflected again and again, as librosa's np.pad does."""
    lengths = (2, 3, 100, 275, 276, 300, 413, 414, 550, 551, 552, 600)
    rng = np.random.default_rng(17)
    ys = [np.clip(0.3 * rng.standard_normal(n) + 0.2 * np.sin(np.arange(n) / 7.0), -1, 1).astype(np.float32) for n in lengths]
    if kind == "int16":
        wavs = [np.round(y * 32767).astype(np.int16) for y in ys]
        ys = [w.astype(np.float32) / 32768.0 for w in wavs]
    else:
        wavs = ys
    mels, mags, t, trim = eng.load_spectrograms_batch(wavs)
    mels, mags = mels.cpu().numpy(), mags.cpu().numpy()
    lin = lambda z: 10.0 ** ((z * hp.max_db - hp.max_db + hp.ref_db) / 20.0)
    for b, y in enumerate(ys):
        mel_o, mag_o = rf.load_spectrograms(y)
        assert tuple(trim[b]) == rv.trim_indices(y) and mel_o.shape[0] == t[b], lengths[b]
        mel, mag = mels[b, :t[b]], mags[b, :hp.r * t[b]]
        np.testing.assert_allclose(lin(mag), lin(mag_o), atol=2e-6 * lin(mag_o).max(), rtol=2e-3, err_msg=str(lengths[b]))
        np.testing.assert_allclose(lin(mel), lin(mel_o), atol=2e-6 * lin(mel_o).max(), rtol=2e-3, err_msg=str(lengths[b]))
        assert np.abs(mag - mag_o)[mag_o > 0.35].max(initial=0) < 1e-4, lengths[b]
        assert np.abs(mel - mel_o)[mel_o > 0.35].max(initial=0) < 1e-4, lengths[b]


def _clips(sr, seed=0):
    """Ragged clips from 2 samples to 10 s: speech-like tones with quiet lead and tail."""
    rng = np.random.default_rng(seed)
    lengths = [2, 3, 600, int(0.7 * sr), int(10 * sr)] + [int(sr * rng.uniform(0.3, 10.0)) for _ in range(27)]
    out = []
    for i, n in enumerate(lengths):
        t = np.arange(n) / sr
        y = 0.3 * np.sin(2 * np.pi * (150 + 100 * rng.random()) * t) * (0.5 + 0.5 * np.sin(2 * np.pi * 3 * t))
        y = y + 0.05 * rng.standard_normal(n)
        if n > 8000:
            y[:int(rng.integers(0, 6000))] *= 1e-5
            y[n - int(rng.integers(1, 6000)):] *= 1e-5
        out.append(np.clip(y, -1, 1).astype(np.float32))
    return out


def _check_features(H, ys, mels, mags, t, trim):
    lin = lambda z: 10.0 ** ((z * H.max_db - H.max_db + H.ref_db) / 20.0)
    mels, mags = mels.cpu().numpy(), mags.cpu().numpy()
    for b, y in enumerate(ys):
        mel_o, mag_o = rf.load_spectrograms(y)
        assert mel_o.shape[0] == t[b] and mag_o.shape[1] == 1 + H.n_fft // 2, b
        if tuple(trim[b]) != rv.trim_indices(y):
            # a frame level within 1e-3 dB of the -60 dB threshold may fall on either side in float32
            rs.trims_agree(trim[b:b + 1], y[None])
            continue
        mel, mag = mels[b, :t[b]], mags[b, :H.r * t[b]]
        np.testing.assert_allclose(lin(mag), lin(mag_o), atol=2e-6 * lin(mag_o).max(), rtol=2e-3, err_msg=str(b))
        np.testing.assert_allclose(lin(mel), lin(mel_o), atol=2e-6 * lin(mel_o).max(), rtol=2e-3, err_msg=str(b))
        assert np.abs(mag - mag_o)[mag_o > 0.35].max(initial=0) < 1e-4, b
        assert np.abs(mel - mel_o)[mel_o > 0.35].max(initial=0) < 1e-4, b


@pytest.mark.parametrize("n", (1024, 4096))
@pytest.mark.parametrize("kind", ["int16", "float32"])
@pytest.mark.parametrize("B", [1, 5, 32])
def test_load_spectrograms_batch_vs_oracle(engines, n, kind, B):
    eng = engines[n]
    with at_rate(SR[n], n) as H:
        ys = _clips(H.sr, seed=B)
        ys = [ys[4]] if B == 1 else ys[:B]
        if kind == "int16":
            wavs = [np.round(y * 32767).astype(np.int16) for y in ys]
            ys = [w.astype(np.float32) / 32768.0 for w in wavs]
        else:
            wavs = ys
        mels, mags, t, trim = eng.load_spectrograms_batch(wavs)
        assert tuple(mags.shape) == (B, H.r * int(t.max()), 1 + n // 2)
        _check_features(H, ys, mels, mags, t, trim)


@pytest.mark.parametrize("n", (1024, 4096))
def test_load_spectrograms_batch_resampled_from_22050(engines, n):
    """22.05 kHz clips resampled on the device to hp.sr (librosa.load(sr=hp.sr)) and then featurised: the same features
    as the oracle composition applied to the device's resampled waveform."""
    eng = engines[n]
    with at_rate(SR[n], n) as H:
        ys = _clips(22050, seed=40)[3:8]
        mels, mags, t, trim = eng.load_spectrograms_batch(ys, rates=[22050] * len(ys))
        res = eng.resample_batch(ys, [22050] * len(ys), H.sr)
        res = [r.cpu().numpy() if hasattr(r, "cpu") else np.asarray(r) for r in res]
        _check_features(H, res, mels, mags, t, trim)
