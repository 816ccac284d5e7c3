"""The feature extraction against float64, bin by bin, at every corpus rate of tests/sample_rates.py (n_fft 1024, 2048 and
4096; the hop, window and mel filterbank of each rate).

tests/test_gpu_wav_features.py holds `dctts_load_spectrograms_batch` to the float32 oracle within 1e-4 on the normalised
scale, about 1000x the chain's float32 noise.  This file holds every mag and mel bin to |got - ref| <= tau * S of its
float64 reference (tests/ref_feature_stages.py, pinned on the CPU by tests/test_feature_stages_reference.py), through the
product entry points and through the test aid `dctts_feature_stage` (Engine.feature_stage), whose three stages are the
product's own launches: 0 the trim energies of a packed ragged batch, 1 the spectra of caller-given trimmed segments,
2 the uploaded tables.  When outputs fail, the tables test says whether the tables are to blame.  Outputs lie inside
NaN-guarded allocations; rows the kernels must not write stay NaN (stage 1) or exactly 0 (the product's padding).
Engines are built and run inside `at_rate` (Hyperparams at that corpus rate).
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import ref_features as rf

import ref_feature_stages as fs
from ref_feature_stages import EPS, LEVELS, TAU
from sample_rates import RATES, at_rate

pytestmark = pytest.mark.gpu
KINDS = ("int16", "float32")
INT16_LEVELS = (1.0, 1e-4, 1e-3)               # full scale; a few LSB (quiet passages of 3 LSB); about 33 LSB
_WORST = {}


def _record(sr, what, v):
    _WORST[(sr, what)] = max(_WORST.get((sr, what), 0.0), float(v))


@pytest.fixture(scope="module")
def engines():
    from dc_tts_b200.engine import Engine
    out = {}
    for sr in RATES:
        with at_rate(sr) as H:
            out[sr] = Engine(0, hparams=H)
    yield out
    print("\nfeature stages, worst err / S: " +
          ", ".join("%d %s %.3g" % (k + (v,)) for k, v in sorted(_WORST.items())))
    for e in out.values():
        e.close()


def _level(kind, b):
    return (INT16_LEVELS if kind == "int16" else LEVELS)[b % 3]


def _batch(sr, kind, lengths, seed, lead=3000, tail=2000):
    """Waveforms of the given lengths (samples) at sr, in `kind`, utterance b at level _level(kind, b), with a loud tone
    and a near-silent stretch in every other one."""
    rng = np.random.default_rng(seed)
    out = []
    for b, n in enumerate(lengths):
        y = fs.clip(rng, n, sr, _level(kind, b), lead=min(lead, n // 4), tail=min(tail, n // 4), tone=b % 2 == 0,
                    hush=b % 2 == 1)
        out.append(fs.as_dtype(y, kind))
    return out


def _pack(engine, wavs):
    offsets = np.zeros(len(wavs) + 1, np.int64)
    offsets[1:] = np.cumsum([w.size for w in wavs])
    return torch.from_numpy(np.concatenate(wavs)).to(engine.device), offsets


def _check_utterance(sr, H, y, mag, mel, r, tag):
    """mag (T, F) and the mel rows (ceil(T / r), n_mels) of the trimmed float32 waveform y against float64."""
    tau = TAU[H.n_fft]
    ref = fs.ref_features(y, sr, H.n_fft, H.hop_length, H.win_length)
    T = ref["a"].shape[0]
    assert mag.shape[0] == T and mel.shape[0] == -(-T // r), (tag, mag.shape, mel.shape, T)
    rm, em = fs.check_mag(mag, ref, tau["mag"])
    rl, el = fs.check_mel(mel, ref, tau["mel"], rows=np.arange(0, T, r))
    _record(sr, "mag", em)
    _record(sr, "mel", el)
    assert rm <= 1, ("mag", tag, rm, em)
    assert rl <= 1, ("mel", tag, rl, el)


# ------------------------------------------------------------------------------------------------ stage 2: tables
@pytest.mark.parametrize("sr", list(RATES))
def test_tables(engines, sr):
    e = engines[sr]
    with at_rate(sr) as H:
        F = 1 + H.n_fft // 2
        wbuf, w = fs.guarded(e, (H.n_mels, F), torch.float32)
        hbuf, win = fs.guarded(e, (H.win_length,), torch.float32)
        rng = e.feature_stage(2, w, win)
        w, win = fs.intact(wbuf, w), fs.intact(hbuf, win)
        W = rf.mel_basis(sr, H.n_fft, H.n_mels)
        # a weight below 2^-24 of its filter's peak (3e-18 at the Nyquist bin of the last filter at 44.1 and 48 kHz, where
        # mel_to_hz(hz_to_mel(sr / 2)) rounds a last bit above sr / 2 in numpy's libm) may be 0 on the device
        tiny = EPS * W.max(-1, keepdims=True)
        ulp = lambda x: np.spacing(np.abs(x.astype(np.float32)))
        assert np.all(np.abs(w.astype(np.float64) - W) <= np.maximum(ulp(W), tiny)), "mel weights are not float32 of the float64 basis"
        assert not (w == 0)[W >= tiny].any() and not w[W == 0].any()
        for m in range(H.n_mels):
            nz, sig = np.flatnonzero(w[m]), np.flatnonzero(W[m] >= tiny[m])
            assert tuple(rng[m]) == (nz[0], nz[-1] + 1), (m, tuple(rng[m]), (nz[0], nz[-1] + 1))
            assert rng[m][0] <= sig[0] and rng[m][1] >= sig[-1] + 1, (m, tuple(rng[m]), (sig[0], sig[-1] + 1))
        ref = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(H.win_length) / H.win_length)
        assert np.all(np.abs(win.astype(np.float64) - ref) <= ulp(ref)), "window is not the periodic Hann"


# ------------------------------------------------------------------------------------------------ stage 0: energies
@pytest.mark.parametrize("B", [1, 5, 32])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("sr", list(RATES))
def test_energies_and_trims(engines, sr, kind, B):
    e = engines[sr]
    with at_rate(sr) as H:
        tau = TAU[H.n_fft]["energies"]
        rng = np.random.default_rng(B + sr)
        lengths = [int(sr * 10)] if B == 1 else [int(v) for v in rng.integers(2, int(sr * 3.5), B)]
        lengths[1:3] = [2, 2049][:len(lengths) - 1]
        wavs = _batch(sr, kind, lengths, seed=B * 7 + sr)
        wav, offsets = _pack(e, wavs)
        nfr = 1 + np.diff(offsets) // 512
        buf, out = fs.guarded(e, (int(nfr.sum()),), torch.float32)
        trims = e.feature_stage(0, out, wav=wav, segments=offsets)
        mse = fs.intact(buf, out)
        f0 = np.concatenate([[0], np.cumsum(nfr)])
        checked = 0
        for b, w in enumerate(wavs):
            y = fs.as_float(w)
            ratio, raw = fs.check_energies(mse[f0[b]:f0[b + 1]], y, tau)
            _record(sr, "energies", raw)
            assert ratio <= 1, (b, ratio, raw)
            checked += fs.trims_agree(trims[b], y, tau)
        assert checked >= B - 1


# ------------------------------------------------------------------------------------------------ stage 1: spectra
def _segment_lengths(H, r):
    """Trimmed lengths 2 and 3, n_fft / 2 - 1 .. + 1, hop multiples - 1 .. + 1 giving T % r = 0 .. 3, and 10 s."""
    n2, hop = H.n_fft // 2, H.hop_length
    out = [2, 3, n2 - 1, n2, n2 + 1]
    for k in (37, 38, 39, 40):
        out += [k * hop - 1, k * hop, k * hop + 1]
    out.append(10 * H.sr)
    return out


@pytest.mark.parametrize("r", [4, 1])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("sr", list(RATES))
def test_spectra_stage(engines, sr, kind, r):
    e = engines[sr]
    with at_rate(sr) as H:
        lengths = _segment_lengths(H, r)
        assert {(1 + n // H.hop_length) % 4 for n in lengths} == {0, 1, 2, 3}
        # each segment starts 1000 samples into its waveform: the sample before it is sound, which pre-emphasis must not read
        wavs = _batch(sr, kind, [n + 1500 for n in lengths], seed=sr + r, lead=0, tail=0)
        wav, offsets = _pack(e, wavs)
        seg = np.stack([offsets[:-1] + 1000, lengths], 1)
        B, F = len(lengths), 1 + H.n_fft // 2
        T = 1 + np.asarray(lengths) // H.hop_length
        T_b = int(-(-T.max() // r)) + 1                           # one more row than the longest needs
        mbuf, mag = fs.guarded(e, (B, r * T_b, F), torch.float32)
        lbuf, mel = fs.guarded(e, (B, T_b, H.n_mels), torch.float32)
        e.feature_stage(1, mag, mel, wav=wav, segments=seg, r=r)
        torch.cuda.synchronize()
        for buf, n in ((mbuf, mag.numel()), (lbuf, mel.numel())):
            assert bool(buf[:fs.GUARD].isnan().all()) and bool(buf[fs.GUARD + n:].isnan().all()), "a guard was overwritten"
        mag, mel = mag.cpu().numpy(), mel.cpu().numpy()
        for b, n in enumerate(lengths):
            t_mel = -(-T[b] // r)
            assert np.isnan(mag[b, T[b]:]).all() and np.isnan(mel[b, t_mel:]).all(), (b, "a row past the utterance was written")
            assert not np.isnan(mag[b, :T[b]]).any() and not np.isnan(mel[b, :t_mel]).any(), (b, "a row was not written")
            y = fs.as_float(wavs[b])[1000:1000 + n]
            _check_utterance(sr, H, y, mag[b, :T[b]], mel[b, :t_mel], r, (kind, b, n))


# ------------------------------------------------------------------------------------------------ product entry points
def _raw_batch(engine, wavs, sr, t_capacity):
    """dctts_load_spectrograms_batch on NaN-guarded outputs of B t_capacity rows -> (mel, mag buffers and views, t, trim,
    T_b)."""
    H = engine.hp
    wav, offsets = _pack(engine, wavs)
    dtype = 1 if wav.dtype == torch.int16 else 0
    B, F = len(wavs), engine.F
    lbuf, mel = fs.guarded(engine, (B * t_capacity * H.n_mels,), torch.float32)
    mbuf, mag = fs.guarded(engine, (B * t_capacity * H.r * F,), torch.float32)
    t = np.zeros(B, np.int32)
    trim = np.zeros((B, 2), np.int32)
    T_b = C.c_int32(0)
    p32 = C.POINTER(C.c_int32)
    engine._set_vocoder_params()
    torch.cuda.synchronize()
    rc = engine._lib.dctts_load_spectrograms_batch(
        engine._h, C.c_void_p(wav.data_ptr()), dtype, offsets.ctypes.data_as(C.POINTER(C.c_int64)), B, sr,
        C.c_void_p(mel.data_ptr()), C.c_void_p(mag.data_ptr()), t_capacity, t.ctypes.data_as(p32), trim.ctypes.data_as(p32),
        C.byref(T_b), None)
    torch.cuda.synchronize()
    assert rc == 0, engine._lib.dctts_last_error(engine._h).decode()
    return lbuf, mel, mbuf, mag, t, trim, T_b.value


def _check_batch(engine, sr, H, wavs, ys):
    """The product batch of `wavs` (float32 views `ys`) against float64 on each utterance's own trimmed samples."""
    tau = TAU[H.n_fft]
    cap = max(-(-(1 + y.size // H.hop_length) // H.r) for y in ys) + 2
    lbuf, mel, mbuf, mag, t, trim, T_b = _raw_batch(engine, wavs, sr, cap)
    B, F, r = len(wavs), engine.F, H.r
    torch.cuda.synchronize()
    for buf, view, used in ((lbuf, mel, B * T_b * H.n_mels), (mbuf, mag, B * r * T_b * F)):
        n = view.numel()
        assert bool(buf[:fs.GUARD].isnan().all()) and bool(buf[fs.GUARD + n:].isnan().all()), "a guard was overwritten"
        assert bool(view[used:].isnan().all()), "written past B T_b rows"
    mel = mel[:B * T_b * H.n_mels].view(B, T_b, H.n_mels).cpu().numpy()
    mag = mag[:B * r * T_b * F].view(B, r * T_b, F).cpu().numpy()
    assert T_b == t.max()
    for b, y in enumerate(ys):
        fs.trims_agree(trim[b], y, tau["energies"])
        s, e = trim[b]
        T = 1 + (e - s) // H.hop_length
        assert t[b] == -(-T // r)
        assert not mag[b, T:].any() and not mel[b, t[b]:].any(), (b, "padding is not exactly 0")
        _check_utterance(sr, H, y[s:e], mag[b, :T], mel[b, :t[b]], r, b)


@pytest.mark.parametrize("B", [1, 5, 32])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("sr", list(RATES))
def test_load_spectrograms_batch(engines, sr, kind, B):
    e = engines[sr]
    with at_rate(sr) as H:
        rng = np.random.default_rng(3 * B + sr)
        lengths = [int(sr * 10)] if B == 1 else [int(v) for v in rng.integers(int(0.05 * sr), int(sr * 3.0), B)]
        wavs = _batch(sr, kind, lengths, seed=11 * B + sr)
        _check_batch(e, sr, H, wavs, [fs.as_float(w) for w in wavs])


@pytest.mark.parametrize("sr", list(RATES))
def test_get_spectrograms(engines, sr):
    """dctts_get_spectrograms: one float32 utterance, every frame (r = 1)."""
    e = engines[sr]
    with at_rate(sr) as H:
        y = _batch(sr, "float32", [int(4.2 * sr)], seed=sr)[0]
        mel, mag, (s, t_end) = e.get_spectrograms(y, sr)
        fs.trims_agree((s, t_end), y, TAU[H.n_fft]["energies"])
        _check_utterance(sr, H, y[s:t_end], mag.cpu().numpy(), mel.cpu().numpy(), 1, "single")


@pytest.mark.parametrize("sr", [r for r in RATES if r != 22050])
def test_resampled_on_the_device(engines, sr):
    """22.05 kHz clips resampled to sr inside load_spectrograms_batch, held to float64 on the device's own resampled
    waveform (the same kernel, returned by resample_batch)."""
    e = engines[sr]
    with at_rate(sr) as H:
        lengths = [int(22050 * s) for s in (0.4, 2.3, 6.1)]
        wavs = _batch(22050, "int16", lengths, seed=sr)
        ys = [t.cpu().numpy() for t in e.resample_batch(wavs, [22050] * len(wavs), sr)]
        mels, mags, t, trim = e.load_spectrograms_batch(wavs, rates=[22050] * len(wavs))
        mels, mags = mels.cpu().numpy(), mags.cpu().numpy()
        for b, y in enumerate(ys):
            fs.trims_agree(trim[b], y, TAU[H.n_fft]["energies"])
            s, e_ = trim[b]
            T = 1 + (e_ - s) // H.hop_length
            assert not mags[b, T:].any() and not mels[b, t[b]:].any()
            _check_utterance(sr, H, y[s:e_], mags[b, :T], mels[b, :t[b]], H.r, ("resampled", b))


def test_aid_refuses_bad_calls(engines):
    from dc_tts_b200.engine import DcttsError
    e = engines[22050]
    with at_rate(22050) as H:
        wav = torch.zeros(5000, device=e.device)
        mag = torch.zeros((1, 4 * 2, e.F), device=e.device)
        mel = torch.zeros((1, 2, H.n_mels), device=e.device)
        with pytest.raises(DcttsError, match="T_b"):
            e.feature_stage(1, mag, mel, wav=wav, segments=[[0, 4000]], r=4)       # 15 frames need 4 rows
        with pytest.raises(DcttsError, match="utterance 0"):
            e.feature_stage(1, mag, mel, wav=wav, segments=[[0, 1]], r=4)
        with pytest.raises(DcttsError, match="stage 3"):
            e._check(e._lib.dctts_feature_stage(e._h, 3, 22050, None, 0, None, 1, 1, 1, None, None, None, None),
                     "dctts_feature_stage")
