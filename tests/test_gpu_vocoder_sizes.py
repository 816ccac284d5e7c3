"""The Griffin-Lim vocoder and the feature extraction at n_fft 1024 (16 kHz) and 4096 (44.1 / 48 kHz): the STFT kernels'
other two instantiations.

Vocoder stages are held to the float64 references and bound forms of test_gpu_vocoder_stages.py (its helpers read the
module constants N_FFT and F, patched here per size), at the table's (hop, win) plus win = n_fft and n_fft - 1.  Features
are held to the oracle composition with the tolerances of test_gpu_wav_features.py.  Engines are built and run inside
`at_rate` (Hyperparams at that corpus rate)."""
import contextlib

import numpy as np
import pytest
import torch

from dc_tts_b200.engine import DcttsError
from oracle import ref_features as rf
from oracle import ref_vocoder as rv

import test_gpu_vocoder_stages as vs
from sample_rates import at_rate

pytestmark = pytest.mark.gpu
SR = {1024: 16000, 4096: 44100}
HOP_WIN = {1024: [(200, 800), (200, 1024), (200, 1023)],
           4096: [(551, 2205), (600, 2400), (551, 4096), (551, 4095)]}
LENGTHS = (2, 3, 5, 60, 840)
# worst err / bound scale per stage and size over this file's cases on an H100 80GB HBM3 at 700 W (DESIGN.md section 8b):
# n_fft 1024: prepare 7.14e-7, istft 2.87e-7, stft 1.09e-7, energies 1.59e-7; n_fft 4096: prepare 7.14e-7, istft 3.40e-7,
# stft 4.0e-8, energies 1.95e-7.  TAU is about 3x of these; prepare does not depend on n_fft and keeps the 2048 bound.
TAU = {1024: dict(prepare=1.5e-6, istft=9e-7, stft=3.3e-7, energies=4.8e-7),
       4096: dict(prepare=1.5e-6, istft=1.0e-6, stft=1.2e-7, energies=5.9e-7)}
_WORST = {}


def _cases():
    out = []
    for n, hws in HOP_WIN.items():
        for i, ((hop, win), T) in enumerate((hw, T) for hw in hws for T in LENGTHS):
            B = vs.case_batch(i)
            if T * hop > 120000 and B == 32:
                B = 3
            out.append((n, hop, win, T, B))
    return out


CASES = _cases()
IDS = ["n%d-hop%d-win%d-T%d-B%d" % c for c in CASES]


@contextlib.contextmanager
def sized(n):
    """Hyperparams at the size's rate, and the float64 references of test_gpu_vocoder_stages at n_fft = n."""
    old = vs.N_FFT, vs.F
    with at_rate(SR[n], n) as H:
        vs.N_FFT, vs.F = n, 1 + n // 2
        try:
            yield H
        finally:
            vs.N_FFT, vs.F = old


def _record(n, stage, raw):
    _WORST[(n, stage)] = max(_WORST.get((n, stage), 0.0), float(raw))


@pytest.fixture(scope="module")
def engines():
    from dc_tts_b200.engine import Engine
    out = {}
    for n in SR:
        with sized(n) as H:
            out[n] = Engine(0, hparams=H)
    yield out
    print("\nvocoder stages at other n_fft, worst err / bound scale: " +
          ", ".join("n_fft %d %s %.3g" % (k + (v,)) for k, v in sorted(_WORST.items())))
    for e in out.values():
        e.close()


@pytest.mark.parametrize("n", sorted(SR))
@pytest.mark.parametrize("T,B", [(2, 1), (5, 3), (60, 32), (840, 3)])
def test_prepare(engines, n, T, B):
    eng = engines[n]
    with sized(n):
        F = vs.F
        mag = vs.make_mag(np.random.default_rng(T * B), B, T)
        bi, vi = vs._guarded(eng, (B, T, F), torch.float32, mag)
        bo, vo = vs._guarded(eng, (B, T, F), torch.complex64)
        eng.vocoder_stage(0, vi, vo)
        vs._intact(bi, vi)
        X = vs._intact(bo, vo)
        ratio, raw = vs.check_prepare(X.real, mag, 1.5, TAU[n]["prepare"])
    _record(n, "prepare", raw)
    assert ratio <= 1, (ratio, raw)


@pytest.mark.parametrize("n,hop,win,T,B", CASES, ids=IDS)
def test_istft(engines, n, hop, win, T, B):
    eng = engines[n]
    with sized(n):
        F = vs.F
        X = vs.make_spectrum(np.random.default_rng(T + hop + win), B, T)
        bi, vi = vs._guarded(eng, (B, T, F), torch.complex64, X)
        bo, vo = vs._guarded(eng, (B, hop * (T - 1)), torch.float32)
        eng.vocoder_stage(1, vi, vo, hop=hop, win=win)
        assert np.array_equal(vs._intact(bi, vi), X)
        ratio, raw = vs.check_istft(vs._intact(bo, vo), X, hop, win, TAU[n]["istft"])
    _record(n, "istft", raw)
    assert ratio <= 1, (ratio, raw)


@pytest.mark.parametrize("n,hop,win,T,B", CASES, ids=IDS)
def test_stft_phase(engines, n, hop, win, T, B):
    eng = engines[n]
    with sized(n):
        F = vs.F
        rng = np.random.default_rng(T * hop + win)
        Ly = hop * (T - 1)
        y = vs.make_wav(rng, B, Ly)
        S = rng.uniform(0, 2, (B, T, F)).astype(np.float32) * np.array(vs.LEVELS * B, np.float32)[:B, None, None]
        S[:, :, ::97] = 0.0
        bi, vi = vs._guarded(eng, (B, Ly), torch.float32, y)
        bs, vs_ = vs._guarded(eng, (B, T, F), torch.float32, S)
        bo, vo = vs._guarded(eng, (B, T, F), torch.complex64)
        eng.vocoder_stage(2, vi, vo, S=vs_, hop=hop, win=win)
        vs._intact(bi, vi)
        vs._intact(bs, vs_)
        ratio, raw = vs.check_stft_phase(vs._intact(bo, vo), y, S, hop, win, TAU[n]["stft"])
    _record(n, "stft", raw)
    assert ratio <= 1, (ratio, raw)


@pytest.mark.parametrize("n", sorted(SR))
@pytest.mark.parametrize("T,B", [(3, 3), (840, 3), (60, 32)])
def test_deemph_and_energies(engines, n, T, B):
    """Neither stage depends on n_fft (the trim frames stay 2048 / 512 at every rate), but both pass the handle's checks."""
    eng = engines[n]
    with sized(n) as H:
        hop, win = H.hop_length, H.win_length
        Ly = hop * (T - 1)
        x = vs.make_deemph_input(np.random.default_rng(Ly), B, Ly)
        bw, vw = vs._guarded(eng, (B, Ly), torch.float32, x)
        eng.vocoder_stage(3, vw, vw, hop=hop, win=win)
        ulps, exact = vs.check_deemph(vs._intact(bw, vw), x)
        assert ulps <= 1 and exact >= 0.999, (ulps, exact)
        y = vs.make_wav(np.random.default_rng(Ly + 7), B, Ly)
        bi, vi = vs._guarded(eng, (B, Ly), torch.float32, y)
        bo, vo = vs._guarded(eng, (B, 1 + Ly // 512), torch.float32)
        trim = eng.vocoder_stage(4, vi, vo, hop=hop, win=win)
        ratio, raw = vs.check_energies(vs._intact(bo, vo), y, TAU[n]["energies"])
        _record(n, "energies", raw)
        assert ratio <= 1, (ratio, raw)
        vs.trims_agree(trim, y)


@pytest.mark.parametrize("n", sorted(SR))
@pytest.mark.parametrize("T", [2, 3, 60])
def test_one_iteration_is_the_stages_bit_for_bit(engines, n, T):
    eng = engines[n]
    with sized(n) as H:
        B, F, hop, win = 3, vs.F, H.hop_length, H.win_length
        mag = torch.from_numpy(vs.make_mag(np.random.default_rng(T), B, T)).to(eng.device)
        Ly = hop * (T - 1)
        X = torch.empty(B, T, F, dtype=torch.complex64, device=eng.device)
        y = torch.empty(B, Ly, device=eng.device)
        mse = torch.empty(B, 1 + Ly // 512, device=eng.device)
        kw = dict(hop=hop, win=win)
        eng.vocoder_stage(0, mag, X, **kw)
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


@pytest.mark.parametrize("n", sorted(SR))
@pytest.mark.parametrize("T,n_iter", [(60, 5), (840, 3)])
def test_spectrogram2wav_vs_the_oracle(engines, n, T, n_iter):
    """The whole chain against ref_vocoder's float32 composition at the size's rate, to 2e-3 of the peak as
    test_vocoder.py holds it at 2048."""
    eng = engines[n]
    with sized(n) as H:
        mag = np.random.default_rng(T + n).uniform(0.1, 0.95, (2, T, vs.F)).astype(np.float32)
        mag[1, T // 2:] *= 0.05
        wav, trim = eng.spectrogram2wav(mag, n_iter=n_iter)
        wav = wav.cpu().numpy()
        assert wav.shape == (2, H.hop_length * (T - 1))
        for b in range(2):
            _, se, full = rv.spectrogram2wav(mag[b], n_iter=n_iter)
            scale = np.abs(full).max()
            assert np.abs(wav[b] - full).max() < 2e-3 * scale, (b, np.abs(wav[b] - full).max(), scale)
            assert abs(int(trim[b, 0]) - se[0]) <= 512 and abs(int(trim[b, 1]) - se[1]) <= 512


# ------------------------------------------------------------------------------------------------ features
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
            vs.trims_agree(trim[b:b + 1], y[None])
            continue
        mel, mag = mels[b, :t[b]], mags[b, :H.r * t[b]]
        np.testing.assert_allclose(lin(mag), lin(mag_o), atol=2e-6 * lin(mag_o).max(), rtol=2e-3, err_msg=str(b))
        np.testing.assert_allclose(lin(mel), lin(mel_o), atol=2e-6 * lin(mel_o).max(), rtol=2e-3, err_msg=str(b))
        assert np.abs(mag - mag_o)[mag_o > 0.35].max(initial=0) < 1e-4, b
        assert np.abs(mel - mel_o)[mel_o > 0.35].max(initial=0) < 1e-4, b


@pytest.mark.parametrize("n", sorted(SR))
@pytest.mark.parametrize("kind", ["int16", "float32"])
@pytest.mark.parametrize("B", [1, 5, 32])
def test_load_spectrograms_batch_vs_oracle(engines, n, kind, B):
    eng = engines[n]
    with sized(n) as H:
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


@pytest.mark.parametrize("n", sorted(SR))
def test_load_spectrograms_batch_resampled_from_22050(engines, n):
    """22.05 kHz clips resampled on the device to hp.sr (librosa.load(sr=hp.sr)) and then featurised: the same features
    as the oracle composition applied to the device's resampled waveform."""
    eng = engines[n]
    with sized(n) as H:
        ys = _clips(22050, seed=40)[3:8]
        mels, mags, t, trim = eng.load_spectrograms_batch(ys, rates=[22050] * len(ys))
        res = eng.resample_batch(ys, [22050] * len(ys), H.sr)
        res = [r.cpu().numpy() if hasattr(r, "cpu") else np.asarray(r) for r in res]
        _check_features(H, res, mels, mags, t, trim)


# ------------------------------------------------------------------------------------------------ refusals
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
    with sized(1024):
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
