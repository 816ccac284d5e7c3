"""ORACLE (test infrastructure) -- float64 references and bounds for each stage of the Griffin-Lim vocoder, the inputs
the vocoder suites feed it, and the signals of the fast Griffin-Lim tests.

Every function that depends on n_fft takes it as an argument or reads it from an input's last axis (n_fft = 2 (F - 1)).
The bounds, with A the stage's absolute-value map of the same input:

  prepare     |got - ref| <= TAU * ref                    ref = (10 ** (m / 20)) ** power in float64
  istft       |got - ref| <= TAU * A + floor              A = the same overlap-add applied to w[m] * sum_k c_k |X_k| / n_fft
  stft_phase  |got - ref| <= S * min(2, 2 TAU A_t / max(1e-8, |c|)) + floor     c = est - alpha E_prev,
              A_t = sum_n |w_n y_pad[n]| + alpha |E_prev|  (alpha = 0 and E_prev = 0 for plain Griffin-Lim; a bin whose
              c is small next to A_t has an ill-conditioned phase, and the bound says so for that bin alone)
  deemph      within 1 float32 ulp of float32(lfilter_float64(x)), at least 99.9 % of samples bit-exact
  energies    |got - ref| <= TAU * ref per frame; trims equal trim_indices of the GPU's own waveform unless a frame lies
              within 1e-3 dB of the -60 dB threshold
"""
import numpy as np
import scipy.fft
import scipy.signal
import torch

from dc_tts_b200.hyperparams import Hyperparams as hp
from oracle import ref_features as rf
from oracle import ref_vocoder as rv

GUARD = 2048                                  # guard elements on each side of every GPU tensor
# worst err / bound scale per stage on an H100 80GB HBM3 (DESIGN.md section 8b), at 400 W for n_fft 2048: prepare 7.14e-7,
# istft 3.92e-7, stft 1.28e-7, energies 2.84e-7; at 700 W for n_fft 1024: prepare 7.14e-7, istft 2.87e-7, stft 1.09e-7,
# energies 1.59e-7, and n_fft 4096: prepare 7.14e-7, istft 3.40e-7, stft 4.0e-8, energies 1.95e-7.  TAU is about 3x of
# these; prepare's 2.1x, so that __powf (2.35e-6) fails it, and it does not depend on n_fft.
TAU = {1024: dict(prepare=1.5e-6, istft=9e-7, stft=3.3e-7, energies=4.8e-7),
       2048: dict(prepare=1.5e-6, istft=1.2e-6, stft=3.9e-7, energies=8.6e-7),
       4096: dict(prepare=1.5e-6, istft=1.0e-6, stft=1.2e-7, energies=5.9e-7)}


# ------------------------------------------------------------------------------------------------ float64 references
def window(n_fft, win, dtype=np.float64):
    return rv.hann_padded(n_fft, win, dtype)


def _ola(frames, hop, wss):
    """librosa.istft's overlap-add of frames (B, T, n_fft), division by the window sum-square where it exceeds tiny,
    centre trim -> (B, hop (T - 1))."""
    B, T, n_fft = frames.shape
    n = n_fft + hop * (T - 1)
    y = np.zeros((B, n), frames.dtype)
    for t in range(T):
        y[:, t * hop:t * hop + n_fft] += frames[:, t]
    nz = wss > np.finfo(wss.dtype).tiny
    y[:, nz] /= wss[nz]
    return y[:, n_fft // 2:n - n_fft // 2]


def ref_prepare(mag, power):
    """utils.py:78-85 with the exponent m * 0.05 formed in float32 as numpy forms it from a float32 mag (the inputs lie on
    a grid where that is exact), then (10 ** e) ** power in float64."""
    m = np.clip(mag, 0, 1).astype(np.float32) * np.float32(hp.max_db) - np.float32(hp.max_db) + np.float32(hp.ref_db)
    e = (m * np.float32(0.05)).astype(np.float64)
    return (10.0 ** e) ** power


def ref_istft(X, hop, win):
    """-> (y, A): float64 librosa.istft of X (B, T, F) and the same map applied to absolute values.  ifft(...).real drops
    the imaginary parts of the DC and Nyquist bins, as librosa's does."""
    n_fft = 2 * (X.shape[-1] - 1)
    X = X.astype(np.complex128)
    X[..., 0] = X[..., 0].real
    X[..., -1] = X[..., -1].real
    w = window(n_fft, win)
    wss = rv.window_sumsquare(X.shape[1], n_fft, hop, win, np.float64)
    y = _ola(np.fft.irfft(X, n=n_fft, axis=-1) * w, hop, wss)
    c = np.full(X.shape[-1], 2.0); c[0] = c[-1] = 1.0
    a = (np.abs(X) * c).sum(-1) / n_fft
    A = _ola(w * a[..., None], hop, wss)
    return y, A


def _padded_frames(y, n_fft, hop, win, T):
    """np.pad(y, n_fft // 2, mode='reflect') framed and windowed: (B, T, n_fft), in y's dtype."""
    yp = np.pad(y, ((0, 0), (n_fft // 2, n_fft // 2)), mode="reflect")
    idx = np.arange(n_fft)[None, :] + hop * np.arange(T)[:, None]
    return yp[:, idx] * window(n_fft, win, y.dtype)


def ref_stft(y, n_fft, hop, win, T):
    """-> (est (B, T, F) complex128, A (B, T)): librosa.stft of y in float64 and A_t = sum_n |w_n y_pad[n]|."""
    fr = _padded_frames(y.astype(np.float64), n_fft, hop, win, T)
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
def check_prepare(got, mag, power, tau):
    ref = ref_prepare(mag, power)
    rel = np.abs(got.astype(np.float64) - ref) / ref
    return float(rel.max()) / tau, float(rel.max())


def check_istft(got, X, hop, win, tau):
    ref, A = ref_istft(X, hop, win)
    err = np.abs(got.astype(np.float64) - ref)
    floor = 1e-37
    pos = A > 0
    raw = float((err[pos] / A[pos]).max()) if pos.any() else 0.0
    return float((err / (tau * A + floor)).max()), raw


def check_phase(got, est, A, S, E_prev, alpha, tau):
    """The stft_phase bound of X = S c / max(1e-8, |c|), c = est - alpha E_prev, against float64 est (B, T, F) and
    A (B, T) from ref_stft -> (ratio, raw)."""
    S = S.astype(np.float64)
    Ep = np.asarray(E_prev).astype(np.complex128)
    c = est - float(alpha) * Ep
    mag = np.maximum(1e-8, np.abs(c))
    ref = S * c / mag
    A_ext = np.broadcast_to(A[..., None] + float(alpha) * np.abs(Ep), S.shape)
    err = np.abs(got.astype(np.complex128) - ref)
    bound = S * np.minimum(2.0, 2.0 * tau * A_ext / mag) + 4 * 2.0 ** -24 * S + 1e-37
    good = (np.abs(c) >= 1e-3 * A_ext) & (S > 0) & (A_ext > 0)      # well-conditioned bins: where the measured ratio comes from
    raw = float((err[good] * mag[good] / (2.0 * S[good] * A_ext[good])).max()) if good.any() else 0.0
    return float((err / bound).max()), raw


def check_stft_phase(got, y, S, hop, win, tau):
    """Plain Griffin-Lim's phase step (alpha = 0, E_prev = 0) of y (B, Ly) against S (B, T, F)."""
    est, A = ref_stft(y, 2 * (S.shape[-1] - 1), hop, win, S.shape[1])
    return check_phase(got, est, A, S, 0.0, 0.0, tau)


def _ordered(x):
    i = x.astype(np.float32).view(np.int32).astype(np.int64)
    return np.where(i < 0, -(i & 0x7FFFFFFF), i)


def check_deemph(got, x):
    """-> (max float32 ulps from float32(lfilter_float64(x)), fraction bit-exact)."""
    d = np.abs(_ordered(got) - _ordered(ref_deemph(x).astype(np.float32)))
    return int(d.max()), float((d == 0).mean())


def check_energies(got, y, tau):
    ref = ref_energies(y)
    err = np.abs(got.astype(np.float64) - ref)
    pos = ref > 0
    raw = float((err[pos] / ref[pos]).max()) if pos.any() else 0.0
    return float((err / (tau * ref + 1e-38)).max()), raw


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
# (hop, win) of the stage cases at each n_fft, the rates' own windows and win = n_fft and n_fft - 1 among them
HOP_WIN = {2048: [(275, 1102), (256, 1024), (200, 800), (512, 2048), (275, 1101), (1102, 1102)],
           1024: [(200, 800), (200, 1024), (200, 1023)],
           4096: [(551, 2205), (600, 2400), (551, 4096), (551, 4095)]}
LEVELS = (1.0, 1e-6, 1e-3)                     # utterance b has level LEVELS[b % 3]: a wrong batch stride cannot pass


def make_mag(rng, B, T, n_fft):
    """Normalised magnitudes on the grid j / 1024 (m * 0.05 exact in float32), below 0 and above 1, exact 0 and 1,
    silent (all-zero) frames, a different level per utterance."""
    mag = rng.integers(-300, 1400, (B, T, 1 + n_fft // 2)) / 1024.0
    for b in range(B):
        mag[b] = np.clip(mag[b] - 0.3 * (b % 3), -0.5, 1.5)
        mag[b, 0, :7] = [0, 1, 0, 1, -1, 2, 0.5]
        mag[b, T // 2] = 0.0                                        # a silent frame
    return mag.astype(np.float32)


def make_spectrum(rng, B, T, n_fft):
    """Random complex X with non-zero imaginary parts at DC and Nyquist; every other utterance is a single bin per
    frame (DC and Nyquist among them); levels 1e6 apart."""
    F = 1 + n_fft // 2
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


# ------------------------------------------------------------------------------------------------ float32 and degraded chains
def fp16(x):
    if np.iscomplexobj(x):
        return (x.real.astype(np.float16) + 1j * x.imag.astype(np.float16)).astype(x.dtype)
    return x.astype(np.float16).astype(x.dtype)


def istft32(X, hop, win, twiddles16=False):
    """A float32 istft: scipy's complex64 inverse FFT (or, with twiddles16, a DFT whose twiddles are rounded to fp16),
    float32 window, overlap-add and window sum-square."""
    F = X.shape[-1]
    n_fft = 2 * (F - 1)
    X = X.astype(np.complex64).copy()
    X[..., 0] = X[..., 0].real
    X[..., -1] = X[..., -1].real
    if twiddles16:
        k, n = np.arange(F), np.arange(n_fft)
        W = fp16(np.exp(2j * np.pi * np.outer(k, n) / n_fft).astype(np.complex64)).astype(np.complex128)
        c = np.full(F, 2.0); c[0] = c[-1] = 1.0
        frames = ((X.astype(np.complex128) * c) @ W).real.astype(np.float32) / np.float32(n_fft)
    else:
        frames = scipy.fft.irfft(X, n=n_fft, axis=-1)
    assert frames.dtype == np.float32
    wss = rv.window_sumsquare(X.shape[1], n_fft, hop, win, np.float32)
    return _ola(frames * window(n_fft, win, np.float32), hop, wss)


def deemph_chunked(x, c=hp.preemphasis, lc=512):
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


# ------------------------------------------------------------------------------------------------ GPU buffers
def guarded(engine, shape, dtype, fill=None):
    """(buffer, view): the view lies inside a 1-D allocation with GUARD NaN elements on each side."""
    n = int(np.prod(shape))
    buf = torch.full((n + 2 * GUARD,), complex(np.nan, np.nan) if dtype == torch.complex64 else np.nan, dtype=dtype,
                     device=engine.device)
    view = buf[GUARD:GUARD + n].view(shape)
    if fill is not None:
        view.copy_(torch.from_numpy(np.ascontiguousarray(fill)).to(engine.device))
    return buf, view


def intact(buf, view):
    """The guards are still NaN and the view holds no NaN; returns the view as numpy."""
    n = view.numel()
    r = torch.view_as_real(buf) if buf.is_complex() else buf
    lo, hi = r[:GUARD], r[GUARD + n:]
    assert bool(lo.isnan().all()) and bool(hi.isnan().all()), "a guard was overwritten"
    out = view.cpu().numpy()
    assert not np.isnan(out.view(np.float32) if np.iscomplexobj(out) else out).any(), "NaN in the output (a read outside the input?)"
    return out


# ------------------------------------------------------------------------------------------------ fast Griffin-Lim signals
SIGNALS = ("vibrato", "chirp", "bursts")
POWERS = (1.0, 1.5)


def signal(kind, seconds=1.0, seed=0):
    """Seeded synthetic waveforms at hp.sr: a harmonic tone with vibrato, a linear chirp, noise bursts."""
    rng = np.random.default_rng(seed)
    n = int(seconds * hp.sr)
    t = np.arange(n) / hp.sr
    if kind == "vibrato":
        f0 = 140.0 + 8.0 * np.sin(2 * np.pi * 5.5 * t)
        ph = 2 * np.pi * np.cumsum(f0) / hp.sr
        y = sum(0.3 / h * np.sin(h * ph) for h in range(1, 9)) * (0.6 + 0.4 * np.sin(2 * np.pi * 2 * t))
    elif kind == "chirp":
        y = 0.5 * np.sin(2 * np.pi * (200.0 * t + 0.5 * 3000.0 * t * t / seconds))
    else:
        y = 0.02 * rng.standard_normal(n)
        for start in rng.uniform(0, seconds - 0.12, 6):
            i = int(start * hp.sr)
            m = int(0.1 * hp.sr)
            y[i:i + m] += 0.4 * rng.standard_normal(m) * np.hanning(m)
    return np.clip(y, -1, 1).astype(np.float32)


def magnitude(kind):
    """The normalised linear magnitude (T, 1 + n_fft / 2) of signal `kind`, as the reference's get_spectrograms gives it."""
    return rf.get_spectrograms(signal(kind))[1]


def amplitude(mag, power, dtype=np.float32):
    """utils.py:78-85 at `power`: (F, T) amplitude target S of a (T, F) normalised magnitude."""
    m = (np.clip(mag.T, 0, 1) * hp.max_db) - hp.max_db + hp.ref_db
    return (np.power(10.0, m * 0.05) ** power).astype(dtype)
