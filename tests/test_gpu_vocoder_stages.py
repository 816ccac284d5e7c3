"""The Griffin-Lim vocoder one stage at a time (dctts_vocoder_stage), against float64.

`tests/test_vocoder.py` compares whole waveforms with the float32 oracle to 2e-3 of the peak, about 1000x what a float32
implementation of the chain gets wrong; this file holds each stage of `dctts_spectrogram2wav` to its own float64 reference
(built from `oracle/ref_vocoder.py` and `scipy.signal.lfilter`) with a bound that scales with the operation:

  prepare     |got - ref| <= TAU * ref                    ref = (10 ** (m / 20)) ** power in float64
  istft       |got - ref| <= TAU * A + floor              A = the same overlap-add applied to w[m] * sum_k c_k |X_k| / 2048
  stft_phase  |got - ref| <= S * min(2, 2 TAU A_t / max(1e-8, |est|)) + floor     A_t = sum_n |w_n y_pad[n]|
              (a bin whose estimate is small next to A_t has an ill-conditioned phase; the bound says so for that bin alone)
  deemph      within 1 float32 ulp of float32(lfilter_float64(x)), at least 99.9 % of samples bit-exact
  energies    |got - ref| <= TAU * ref per frame; trims equal trim_indices of the GPU's own waveform unless a frame lies
              within 1e-3 dB of the -60 dB threshold

The CPU tests show that a correct float32 chain passes these bounds and that degraded ones (fp16-rounded inputs or
twiddles, de-emphasis in float32) do not.  The GPU tests place every input and output inside a larger allocation with
NaN guards on both sides, and check the guards and the outputs afterwards.
"""
import numpy as np
import pytest
import scipy.fft
import scipy.signal
import torch

from dc_tts_b200.hyperparams import Hyperparams as hp
from oracle import ref_vocoder as rv

N_FFT = 2048
F = 1 + N_FFT // 2
GUARD = 2048                                  # guard elements on each side of every GPU tensor
# worst err / bound scale over every case of this file on an H100 80GB HBM3 at 400 W (DESIGN.md section 8b): prepare
# 7.14e-7, istft 3.92e-7, stft 1.28e-7, energies 2.84e-7.  TAU is about 3x of these; prepare's 2.1x, so that __powf
# (2.35e-6) fails it.
TAU = {"prepare": 1.5e-6, "istft": 1.2e-6, "stft": 3.9e-7, "energies": 8.6e-7}
HOP_WIN = [(275, 1102), (256, 1024), (200, 800), (512, 2048), (275, 1101), (1102, 1102)]
LENGTHS = (2, 3, 4, 5, 8, 60, 513, 840)
_WORST = {}


def _record(stage, raw):
    _WORST[stage] = max(_WORST.get(stage, 0.0), float(raw))


# ------------------------------------------------------------------------------------------------ float64 references
def _window(win, dtype=np.float64):
    return rv.hann_padded(N_FFT, win, dtype)


def _ola(frames, hop, wss):
    """librosa.istft's overlap-add of frames (B, T, n_fft), division by the window sum-square where it exceeds tiny,
    centre trim -> (B, hop (T - 1))."""
    B, T, _ = frames.shape
    n = N_FFT + hop * (T - 1)
    y = np.zeros((B, n), frames.dtype)
    for t in range(T):
        y[:, t * hop:t * hop + N_FFT] += frames[:, t]
    nz = wss > np.finfo(wss.dtype).tiny
    y[:, nz] /= wss[nz]
    return y[:, N_FFT // 2:n - N_FFT // 2]


def ref_prepare(mag, power):
    """utils.py:78-85 with the exponent m * 0.05 formed in float32 as numpy forms it from a float32 mag (the inputs lie on
    a grid where that is exact), then (10 ** e) ** power in float64."""
    m = np.clip(mag, 0, 1).astype(np.float32) * np.float32(hp.max_db) - np.float32(hp.max_db) + np.float32(hp.ref_db)
    e = (m * np.float32(0.05)).astype(np.float64)
    return (10.0 ** e) ** power


def ref_istft(X, hop, win):
    """-> (y, A): float64 librosa.istft of X (B, T, F) and the same map applied to absolute values.  ifft(...).real drops
    the imaginary parts of the DC and Nyquist bins, as librosa's does."""
    X = X.astype(np.complex128)
    X[..., 0] = X[..., 0].real
    X[..., -1] = X[..., -1].real
    w = _window(win)
    wss = rv.window_sumsquare(X.shape[1], N_FFT, hop, win, np.float64)
    y = _ola(np.fft.irfft(X, n=N_FFT, axis=-1) * w, hop, wss)
    c = np.full(F, 2.0); c[0] = c[-1] = 1.0
    a = (np.abs(X) * c).sum(-1) / N_FFT
    A = _ola(w * a[..., None], hop, wss)
    return y, A


def _padded_frames(y, hop, win, T):
    """np.pad(y, n_fft // 2, mode='reflect') framed and windowed: (B, T, n_fft), in y's dtype."""
    yp = np.pad(y, ((0, 0), (N_FFT // 2, N_FFT // 2)), mode="reflect")
    idx = np.arange(N_FFT)[None, :] + hop * np.arange(T)[:, None]
    return yp[:, idx] * _window(win, y.dtype)


def ref_stft(y, hop, win, T):
    """-> (est (B, T, F) complex128, A (B, T)): librosa.stft of y in float64 and A_t = sum_n |w_n y_pad[n]|."""
    fr = _padded_frames(y.astype(np.float64), hop, win, T)
    return np.fft.rfft(fr, axis=-1), np.abs(fr).sum(-1)


def phase_update(S, est, dtype):
    """utils.py:101-104: X = S * est / max(1e-8, |est|)."""
    return S * est / np.maximum(dtype(1e-8), np.abs(est))


def ref_deemph(x):
    return scipy.signal.lfilter([1], [1, -hp.preemphasis], x.astype(np.float64), axis=-1)


def ref_energies(y):
    """librosa.effects.trim's frame energies (rmse ** 2) of y (B, Ly) in float64: (B, 1 + Ly // 512)."""
    yp = np.pad(y.astype(np.float64), ((0, 0), (1024, 1024)), mode="reflect")
    nfr = 1 + y.shape[1] // 512
    idx = np.arange(2048)[None, :] + 512 * np.arange(nfr)[:, None]
    return (yp[:, idx] ** 2).mean(-1)


# ------------------------------------------------------------------------------------------------ the bounds
def check_prepare(got, mag, power, tau=None):
    ref = ref_prepare(mag, power)
    rel = np.abs(got.astype(np.float64) - ref) / ref
    return float(rel.max()) / (tau or TAU["prepare"]), float(rel.max())


def check_istft(got, X, hop, win, tau=None):
    ref, A = ref_istft(X, hop, win)
    err = np.abs(got.astype(np.float64) - ref)
    floor = 1e-37
    pos = A > 0
    raw = float((err[pos] / A[pos]).max()) if pos.any() else 0.0
    return float((err / ((tau or TAU["istft"]) * A + floor)).max()), raw


def check_stft_phase(got, y, S, hop, win, tau=None):
    tau = tau or TAU["stft"]
    T = S.shape[1]
    est, A = ref_stft(y, hop, win, T)
    S = S.astype(np.float64)
    ref = phase_update(S, est, np.float64)
    err = np.abs(got.astype(np.complex128) - ref)
    mag = np.maximum(1e-8, np.abs(est))
    bound = S * np.minimum(2.0, 2.0 * tau * A[..., None] / mag) + 4 * 2.0 ** -24 * S + 1e-37
    good = (np.abs(est) >= 1e-3 * A[..., None]) & (S > 0) & (A[..., None] > 0)    # well-conditioned bins: where the measured ratio comes from
    raw = float((err[good] * mag[good] / (2.0 * S[good] * np.broadcast_to(A[..., None], S.shape)[good])).max()) if good.any() else 0.0
    return float((err / bound).max()), raw


def _ordered(x):
    i = x.astype(np.float32).view(np.int32).astype(np.int64)
    return np.where(i < 0, -(i & 0x7FFFFFFF), i)


def check_deemph(got, x):
    """-> (max float32 ulps from float32(lfilter_float64(x)), fraction bit-exact)."""
    d = np.abs(_ordered(got) - _ordered(ref_deemph(x).astype(np.float32)))
    return int(d.max()), float((d == 0).mean())


def check_energies(got, y, tau=None):
    ref = ref_energies(y)
    err = np.abs(got.astype(np.float64) - ref)
    pos = ref > 0
    raw = float((err[pos] / ref[pos]).max()) if pos.any() else 0.0
    return float((err / ((tau or TAU["energies"]) * ref + 1e-38)).max()), raw


def trims_agree(trim, wav):
    """The product's trims against rv.trim_indices of the same waveform, per utterance, unless a frame's level lies
    within 1e-3 dB of the -60 dB threshold (where float32 and float64 energies may fall on either side)."""
    for b in range(wav.shape[0]):
        mse = ref_energies(wav[b:b + 1])[0]
        db = 10 * np.log10(np.maximum(1e-10, mse)) - 10 * np.log10(np.maximum(1e-10, mse.max()))
        if np.abs(db + 60).min() < 1e-3:
            continue
        assert tuple(trim[b]) == rv.trim_indices(wav[b].astype(np.float64)), (b, tuple(trim[b]), rv.trim_indices(wav[b]))


# ------------------------------------------------------------------------------------------------ inputs
LEVELS = (1.0, 1e-6, 1e-3)                     # utterance b has level LEVELS[b % 3]: a wrong batch stride cannot pass


def make_mag(rng, B, T):
    """Normalised magnitudes on the grid j / 1024 (m * 0.05 exact in float32), below 0 and above 1, exact 0 and 1,
    silent (all-zero) frames, a different level per utterance."""
    mag = rng.integers(-300, 1400, (B, T, F)) / 1024.0
    for b in range(B):
        mag[b] = np.clip(mag[b] - 0.3 * (b % 3), -0.5, 1.5)
        mag[b, 0, :7] = [0, 1, 0, 1, -1, 2, 0.5]
        mag[b, T // 2] = 0.0                                        # a silent frame
    return mag.astype(np.float32)


def make_spectrum(rng, B, T):
    """Random complex X with non-zero imaginary parts at DC and Nyquist; every other utterance is a single bin per
    frame (DC and Nyquist among them); levels 1e6 apart."""
    X = (rng.standard_normal((B, T, F)) + 1j * rng.standard_normal((B, T, F))).astype(np.complex64)
    for b in range(B):
        X[b] *= LEVELS[b % 3]
        if b % 2 == 1:
            keep = rng.integers(0, F, T)
            keep[0], keep[-1] = 0, F - 1
            one = np.zeros((T, F), np.complex64)
            one[np.arange(T), keep] = X[b, np.arange(T), keep]
            X[b] = one
    return X


def make_wav(rng, B, Ly):
    """Noise-like waveforms with a silent stretch (est = 0 there, so X = 0) and a stretch near 1e-9 (|est| about the 1e-8
    phase floor); levels 1e6 apart."""
    y = rng.standard_normal((B, Ly)) * 0.3
    for b in range(B):
        y[b] *= LEVELS[b % 3]
        if Ly >= 8:
            y[b, Ly // 4:Ly // 2] = 0.0
            y[b, Ly // 2:3 * Ly // 4] *= 1e-9 / (0.3 * LEVELS[b % 3])
    return y.astype(np.float32)


def make_deemph_input(rng, B, Ly):
    """A constant DC signal (the largest carry), impulses at samples 512k - 1 and 512k, noise."""
    x = rng.standard_normal((B, Ly)).astype(np.float32) * 0.2
    for b in range(B):
        if b % 3 == 0:
            x[b] = 0.5
        elif b % 3 == 1:
            x[b] = 0.0
            x[b, 511::512] = 1.0
            x[b, 512::512] = -0.75
            x[b, 0] = 0.25
    return x


def case_batch(i):
    return (1, 3, 32)[i % 3]


# ------------------------------------------------------------------------------------------------ CPU: the bounds suit float32
def _fp16(x):
    if np.iscomplexobj(x):
        return (x.real.astype(np.float16) + 1j * x.imag.astype(np.float16)).astype(x.dtype)
    return x.astype(np.float16).astype(x.dtype)


def istft32(X, hop, win, twiddles16=False):
    """A float32 istft: scipy's complex64 inverse FFT (or, with twiddles16, a DFT whose twiddles are rounded to fp16),
    float32 window, overlap-add and window sum-square."""
    X = X.astype(np.complex64).copy()
    X[..., 0] = X[..., 0].real
    X[..., -1] = X[..., -1].real
    if twiddles16:
        k, n = np.arange(F), np.arange(N_FFT)
        W = _fp16(np.exp(2j * np.pi * np.outer(k, n) / N_FFT).astype(np.complex64)).astype(np.complex128)
        c = np.full(F, 2.0); c[0] = c[-1] = 1.0
        frames = ((X.astype(np.complex128) * c) @ W).real.astype(np.float32) / np.float32(N_FFT)
    else:
        frames = scipy.fft.irfft(X, n=N_FFT, axis=-1)
    assert frames.dtype == np.float32
    wss = rv.window_sumsquare(X.shape[1], N_FFT, hop, win, np.float32)
    return _ola(frames * _window(win, np.float32), hop, wss)


@pytest.mark.parametrize("hop,win", HOP_WIN)
def test_float32_istft_passes_and_fp16_fails(hop, win):
    rng = np.random.default_rng(hop + win)
    X = make_spectrum(rng, 3, 8)
    r32, _ = check_istft(istft32(X, hop, win), X, hop, win)
    assert r32 < 0.5, r32
    r_in, _ = check_istft(istft32(_fp16(X), hop, win), X, hop, win)
    r_tw, _ = check_istft(istft32(X, hop, win, twiddles16=True), X, hop, win)
    assert r_in > 1 and r_tw > 1, (r_in, r_tw)


@pytest.mark.parametrize("hop,win", HOP_WIN)
def test_float32_stft_phase_passes_and_fp16_fails(hop, win):
    rng = np.random.default_rng(hop * win)
    T = 8
    y = make_wav(rng, 3, hop * (T - 1))
    S = rng.uniform(0, 2, (3, T, F)).astype(np.float32)
    got = np.stack([phase_update(S[b], rv.stft(y[b], N_FFT, hop, win).T, np.float32) for b in range(3)])
    assert got.dtype == np.complex64
    r32, _ = check_stft_phase(got, y, S, hop, win)
    assert r32 < 0.5, r32
    y16 = _fp16(y)
    bad = np.stack([phase_update(S[b], rv.stft(y16[b], N_FFT, hop, win).T, np.float32) for b in range(3)])
    r16, _ = check_stft_phase(bad, y, S, hop, win)
    assert r16 > 1, r16


@pytest.mark.parametrize("power", [1.5, 1.0])
def test_float32_prepare_passes_and_fp16_fails(power):
    mag = make_mag(np.random.default_rng(3), 3, 5)
    m = np.clip(mag, 0, 1) * np.float32(hp.max_db) - np.float32(hp.max_db) + np.float32(hp.ref_db)
    got = np.power(np.power(np.float32(10), m * np.float32(0.05)), np.float32(power))
    assert got.dtype == np.float32
    assert check_prepare(got, mag, power)[0] < 0.5
    assert check_prepare(_fp16(got), mag, power)[0] > 1


def _deemph_chunked(x, c=hp.preemphasis, lc=512):
    """The GPU's scheme in float64: chunk end states from zero, chained carries, each chunk replayed from its carry."""
    B, Ly = x.shape
    nch = -(-Ly // lc)
    ends = np.zeros((B, nch))
    for j in range(nch):
        ends[:, j] = scipy.signal.lfilter([1], [1, -c], x[:, j * lc:(j + 1) * lc].astype(np.float64), axis=-1)[:, -1]
    carry = np.zeros((B, nch))
    for j in range(1, nch):
        carry[:, j] = ends[:, j - 1] + c ** lc * carry[:, j - 1]
    out = np.empty((B, Ly), np.float32)
    for j in range(nch):
        seg = x[:, j * lc:(j + 1) * lc].astype(np.float64)
        out[:, j * lc:(j + 1) * lc] = scipy.signal.lfilter([1], [1, -c], seg, axis=-1, zi=c * carry[:, j:j + 1])[0]
    return out


@pytest.mark.parametrize("Ly", [275, 512, 1024 + 17, 275 * 512])
def test_chunked_float64_deemph_passes_and_float32_fails(Ly):
    x = make_deemph_input(np.random.default_rng(Ly), 3, Ly)
    ulps, exact = check_deemph(_deemph_chunked(x), x)
    assert ulps <= 1 and exact >= 0.999, (ulps, exact)
    if Ly > 512:
        y32 = scipy.signal.lfilter(np.ones(1, np.float32), np.array([1, -hp.preemphasis], np.float32), x, axis=-1)
        assert y32.dtype == np.float32
        ulps32, exact32 = check_deemph(y32, x)
        assert ulps32 > 1 and exact32 < 0.999, (ulps32, exact32)
        c32 = float(np.float32(hp.preemphasis))             # the float64 filter with a float32-rounded coefficient
        ulps_c, exact_c = check_deemph(_deemph_chunked(x, c32), x)
        assert ulps_c > 1 or exact_c < 0.999, (ulps_c, exact_c)


def energies32(y):
    """Frame energies in float32 in a 256-thread order: each thread fuses 8 squares into its sum (fmaf), the 32 lanes
    of a warp are summed by halving, then the 8 warp sums one after another."""
    yp = np.pad(y, ((0, 0), (1024, 1024)), mode="reflect")
    idx = np.arange(2048)[None, :] + 512 * np.arange(1 + y.shape[1] // 512)[:, None]
    v = yp[:, idx].reshape(y.shape[0], -1, 8, 256).astype(np.float64)
    acc = np.zeros(v.shape[:2] + (256,), np.float32)
    for i in range(8):
        acc = (acc + v[:, :, i] ** 2).astype(np.float32)
    acc = acc.reshape(acc.shape[:2] + (8, 32))
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[..., np.arange(32) ^ o]
    t = np.zeros(acc.shape[:2], np.float32)
    for w in range(8):
        t = t + acc[..., w, 0]
    return t / np.float32(2048)


def test_float32_energies_pass_and_fp16_fail():
    y = make_wav(np.random.default_rng(5), 3, 275 * 59)
    got = energies32(y)
    assert got.dtype == np.float32
    assert check_energies(got, y)[0] < 0.5
    assert check_energies(energies32(_fp16(y)), y)[0] > 1


def test_reference_istft_inverts_reference_stft():
    """The float64 references invert each other (librosa's perfect reconstruction), at every window of the matrix."""
    for hop, win in HOP_WIN[:5]:
        y = np.random.default_rng(win).standard_normal((2, hop * 20))
        est, _ = ref_stft(y, hop, win, 21)
        back, _ = ref_istft(est, hop, win)
        assert np.abs(back - y).max() < 1e-12, (hop, win)


# ------------------------------------------------------------------------------------------------ GPU
def _guarded(engine, shape, dtype, fill=None):
    """(buffer, view): the view lies inside a 1-D allocation with GUARD NaN elements on each side."""
    n = int(np.prod(shape))
    buf = torch.full((n + 2 * GUARD,), complex(np.nan, np.nan) if dtype == torch.complex64 else np.nan, dtype=dtype,
                     device=engine.device)
    view = buf[GUARD:GUARD + n].view(shape)
    if fill is not None:
        view.copy_(torch.from_numpy(np.ascontiguousarray(fill)).to(engine.device))
    return buf, view


def _intact(buf, view):
    """The guards are still NaN and the view holds no NaN; returns the view as numpy."""
    n = view.numel()
    r = torch.view_as_real(buf) if buf.is_complex() else buf
    lo, hi = r[:GUARD], r[GUARD + n:]
    assert bool(lo.isnan().all()) and bool(hi.isnan().all()), "a guard was overwritten"
    out = view.cpu().numpy()
    assert not np.isnan(out.view(np.float32) if np.iscomplexobj(out) else out).any(), "NaN in the output (a read outside the input?)"
    return out


def _matrix():
    cases = []
    for i, (hw, T) in enumerate((hw, T) for hw in HOP_WIN for T in LENGTHS):
        B = case_batch(i)
        if T * hw[0] > 120000 and B == 32:
            B = 3
        cases.append((hw[0], hw[1], T, B))
    return cases


CASES = _matrix()
_ids = ["hop%d-win%d-T%d-B%d" % c for c in CASES]


@pytest.fixture(scope="module")
def eng():
    from dc_tts_b200.engine import Engine
    e = Engine(0)
    yield e
    print("\nvocoder stages, worst err / bound scale: " + ", ".join("%s %.3g" % kv for kv in sorted(_WORST.items())))
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("power", [1.5, 1.0])
@pytest.mark.parametrize("T,B", [(2, 1), (3, 3), (60, 32), (513, 3), (840, 32)])
def test_prepare(eng, T, B, power):
    mag = make_mag(np.random.default_rng(T * B), B, T)
    bi, vi = _guarded(eng, (B, T, F), torch.float32, mag)
    bo, vo = _guarded(eng, (B, T, F), torch.complex64)
    eng.vocoder_stage(0, vi, vo, power=power)
    _intact(bi, vi)
    X = _intact(bo, vo)
    assert not X.imag.any()
    ratio, raw = check_prepare(X.real, mag, power)
    _record("prepare", raw)
    assert ratio <= 1, (ratio, raw)


@pytest.mark.gpu
@pytest.mark.parametrize("hop,win,T,B", CASES, ids=_ids)
def test_istft(eng, hop, win, T, B):
    X = make_spectrum(np.random.default_rng(T + hop), B, T)
    Ly = hop * (T - 1)
    bi, vi = _guarded(eng, (B, T, F), torch.complex64, X)
    bo, vo = _guarded(eng, (B, Ly), torch.float32)
    eng.vocoder_stage(1, vi, vo, hop=hop, win=win)
    assert np.array_equal(_intact(bi, vi), X)
    ratio, raw = check_istft(_intact(bo, vo), X, hop, win)
    _record("istft", raw)
    assert ratio <= 1, (ratio, raw)


@pytest.mark.gpu
@pytest.mark.parametrize("hop,win,T,B", CASES, ids=_ids)
def test_stft_phase(eng, hop, win, T, B):
    """T = 2 and 3 put the n_fft / 2 reflect padding past a short signal: np.pad reflects it again and again."""
    rng = np.random.default_rng(T * hop + 1)
    Ly = hop * (T - 1)
    y = make_wav(rng, B, Ly)
    S = rng.uniform(0, 2, (B, T, F)).astype(np.float32) * np.array(LEVELS * B, np.float32)[:B, None, None]
    S[:, :, ::97] = 0.0
    bi, vi = _guarded(eng, (B, Ly), torch.float32, y)
    bs, vs = _guarded(eng, (B, T, F), torch.float32, S)
    bo, vo = _guarded(eng, (B, T, F), torch.complex64)
    eng.vocoder_stage(2, vi, vo, S=vs, hop=hop, win=win)
    _intact(bi, vi)
    _intact(bs, vs)
    ratio, raw = check_stft_phase(_intact(bo, vo), y, S, hop, win)
    _record("stft", raw)
    assert ratio <= 1, (ratio, raw)


@pytest.mark.gpu
@pytest.mark.parametrize("hop,win,T,B", CASES, ids=_ids)
def test_deemph(eng, hop, win, T, B):
    Ly = hop * (T - 1)
    x = make_deemph_input(np.random.default_rng(Ly), B, Ly)
    bw, vw = _guarded(eng, (B, Ly), torch.float32, x)
    eng.vocoder_stage(3, vw, vw, hop=hop, win=win)
    ulps, exact = check_deemph(_intact(bw, vw), x)
    _WORST["deemph_ulps"] = max(_WORST.get("deemph_ulps", 0), ulps)
    _WORST["deemph_inexact"] = max(_WORST.get("deemph_inexact", 0.0), 1 - exact)
    assert ulps <= 1 and exact >= 0.999, (ulps, exact)


@pytest.mark.gpu
@pytest.mark.parametrize("hop,win,T,B", CASES, ids=_ids)
def test_energies_and_trims(eng, hop, win, T, B):
    Ly = hop * (T - 1)
    rng = np.random.default_rng(Ly + 7)
    y = make_wav(rng, B, Ly)
    for b in range(B):                                   # quiet lead and tail, so that trimming has work to do
        y[b, :Ly // 5] *= 1e-4
        y[b, Ly - Ly // 6:] *= 1e-4
    nfr = 1 + Ly // 512
    bi, vi = _guarded(eng, (B, Ly), torch.float32, y)
    bo, vo = _guarded(eng, (B, nfr), torch.float32)
    trim = eng.vocoder_stage(4, vi, vo, hop=hop, win=win)
    _intact(bi, vi)
    ratio, raw = check_energies(_intact(bo, vo), y)
    _record("energies", raw)
    assert ratio <= 1, (ratio, raw)
    trims_agree(trim, y)


@pytest.mark.gpu
@pytest.mark.parametrize("T", [2, 3, 60, 513])
def test_spectrogram2wav_without_iterations_is_the_float64_chain(eng, T):
    """prepare -> istft -> de-emphasis in one product call at n_iter = 0: linear and well conditioned, so held to the sum of
    the stage bounds carried through the de-emphasis filter (plus the final float32 rounding)."""
    B, hop, win = 3, hp.hop_length, hp.win_length
    mag = make_mag(np.random.default_rng(T + 11), B, T)
    wav, trim = eng.spectrogram2wav(mag, n_iter=0)
    wav = wav.cpu().numpy()
    S = ref_prepare(mag, hp.power)
    y, A = ref_istft(S.astype(np.complex128), hop, win)
    ref, bound = ref_deemph(y), ref_deemph((TAU["istft"] + TAU["prepare"]) * A)
    err = np.abs(wav - ref)
    ratio = float((err / (bound + 2.0 ** -23 * np.abs(ref) + 1e-37)).max())
    _record("n_iter0", float((err / (ref_deemph(A) + 1e-37)).max()))
    assert ratio <= 1, ratio
    trims_agree(trim, wav)


@pytest.mark.gpu
@pytest.mark.parametrize("T,hop,win", [(2, 275, 1102), (3, 275, 1102), (60, 200, 800), (513, 275, 1102)])
def test_one_iteration_is_the_stages_bit_for_bit(eng, T, hop, win):
    """dctts_spectrogram2wav at n_iter = 1 issues exactly the stages' launches: prepare, istft, stft_phase, istft, deemph,
    energies."""
    B = 3
    mag = torch.from_numpy(make_mag(np.random.default_rng(T), B, T)).to(eng.device)
    Ly = hop * (T - 1)
    X = torch.empty(B, T, F, dtype=torch.complex64, device=eng.device)
    y = torch.empty(B, Ly, device=eng.device)
    mse = torch.empty(B, 1 + Ly // 512, device=eng.device)
    kw = dict(hop=hop, win=win)
    eng.vocoder_stage(0, mag, X, **kw)                   # also sets the handle's vocoder parameters to (hop, win)
    wav = torch.empty(B, Ly, device=eng.device)
    trim = np.zeros((B, 2), np.int32)
    eng._check(eng._lib.dctts_spectrogram2wav(eng._h, mag.data_ptr(), B, T, 1, wav.data_ptr(), trim.ctypes.data, eng._stream()),
               "dctts_spectrogram2wav")
    S = X.real.contiguous()
    eng.vocoder_stage(1, X, y, **kw)
    X2 = torch.empty_like(X)
    eng.vocoder_stage(2, y, X2, S=S, **kw)
    eng.vocoder_stage(1, X2, y, **kw)
    eng.vocoder_stage(3, y, y, **kw)
    trim2 = eng.vocoder_stage(4, y, mse, **kw)
    assert torch.equal(wav, y) and np.array_equal(trim, trim2)


@pytest.mark.gpu
def test_refusals(eng):
    from dc_tts_b200.engine import DcttsError
    dev = eng.device
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


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["int16", "float32"])
def test_short_clip_features_follow_np_pad(eng, kind):
    """Clips shorter than the n_fft / 2 padding (after trimming) are reflected again and again, as librosa's np.pad does."""
    from oracle import ref_features as rf
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
