"""Vocoder half of the reference's utils.py (/root/reference/utils.py:67-114) with the same names:
`spectrogram2wav(mag)`, `griffin_lim(spectrogram)`, `invert_spectrogram(spectrogram)`.

The reference runs librosa's stft / istft on the CPU, 50 + 51 times per utterance; here the whole
Griffin-Lim loop runs on the GPU (csrc/kernels_vocoder.cu: one CTA per STFT frame, an n_fft-point FFT
in shared memory, n_fft 1024, 2048 or 4096) behind `dctts_spectrogram2wav`.  This is the first "next" row of SURVEY.md 8(f), not part
of the Text2Mel + SSRN hot path.  Feature extraction (`get_spectrograms`, `load_spectrograms`,
utils.py:20-65,147-162) runs on the GPU too (`dctts_get_spectrograms` / `dctts_load_spectrograms_batch`: trim,
pre-emphasis, STFT, mel filterbank, dB, normalisation in two kernels per call, for one utterance or a whole bucket);
`librosa.load` is replaced by scipy's WAV reader,
and with `resample=True` a file at another sample rate is resampled to hp.sr on the GPU as librosa.load(fpath, sr=hp.sr)
does (`dctts_resample_batch`: librosa 0.6 / resampy 'kaiser_best'); without it such a file is refused, so a corpus at an
unexpected rate is never converted silently.  `plot_alignment` writes its PNG without matplotlib (no title, axes or
colorbar).  Other file formats and the remaining training helpers of the reference's utils.py stay out of scope.
"""
import os

import numpy as np

from .engine import get_engine
from .hyperparams import Hyperparams as hp


def stretch_path(path, lengths, factor, steps=None):
    """Speaking rate: the attention-window path of each utterance slowed down (factor > 1) or sped up (factor < 1).
    path (B, S) integers, lengths (B,) frames per utterance (numpy, or tensors that are copied to the host).  Utterance
    b gets n'_b = max(1, round(factor * n_b)) frames (Python's round: halves go to the even integer), with
    P'[j] = P[min(n_b - 1, floor(j / factor))].  Returns (path' (B, max n') int32 padded with each row's last window,
    n' (B,) int32).  A stretched length above `steps` (default hp.max_T) is refused."""
    P = np.asarray(path.cpu() if hasattr(path, "cpu") else path)
    n = np.asarray(lengths.cpu() if hasattr(lengths, "cpu") else lengths).reshape(-1).astype(np.int64)
    factor = float(factor)
    if not factor > 0:
        raise ValueError("stretch_path: factor must be > 0, got %r" % factor)
    if P.ndim != 2 or P.shape[0] != n.shape[0]:
        raise ValueError("stretch_path: path must be (B, S) for %d lengths, got %s" % (n.shape[0], P.shape))
    steps = hp.max_T if steps is None else int(steps)
    bad = np.flatnonzero((n < 1) | (n > P.shape[1]))
    if bad.size:
        raise ValueError("stretch_path: utterance %d has length %d outside [1, %d]" % (bad[0], n[bad[0]], P.shape[1]))
    m = np.array([max(1, int(round(factor * int(nb)))) for nb in n], np.int64)
    over = np.flatnonzero(m > steps)
    if over.size:
        b = over[0]
        raise ValueError("stretch_path: utterance %d stretched from %d to %d frames, more than %d"
                         % (b, n[b], m[b], steps))
    out = np.empty((n.shape[0], int(m.max())), np.int32)
    for b in range(n.shape[0]):
        src = np.minimum(n[b] - 1, np.floor(np.arange(m[b]) / factor).astype(np.int64))
        out[b, :m[b]] = P[b, src]
        out[b, m[b]:] = out[b, m[b] - 1]
    return out, m.astype(np.int32)


def spectrogram2wav(mag, momentum=0.0):
    """utils.py:67-94.  mag: (T, 1+n_fft//2) normalised magnitudes -> trimmed float32 wav (numpy).  `momentum`: the
    fast Griffin-Lim update (librosa's griffinlim(momentum=...)); 0 is the reference's plain Griffin-Lim."""
    wav, trim = get_engine().spectrogram2wav(np.asarray(mag, np.float32)[None], momentum=momentum)
    s, e = int(trim[0, 0]), int(trim[0, 1])
    return wav[0, s:e].cpu().numpy().astype(np.float32)


def spectrograms2wavs(mags, lengths=None, momentum=0.0, engine=None):
    """Batched form: (B, T, F) -> list of trimmed wavs (one device pass for the whole batch).  `lengths`: optional (B,)
    magnitude frames per utterance; wav b is then spectrogram2wav(mags[b, :lengths[b]]), bit for bit.  `momentum` as
    for spectrogram2wav.  `engine`: the Engine to run on (default: the process-wide one)."""
    wav, trim = (engine or get_engine()).spectrogram2wav(mags, lengths=lengths, momentum=momentum)
    wav = wav.cpu().numpy()
    return [wav[b, int(trim[b, 0]):int(trim[b, 1])].astype(np.float32) for b in range(wav.shape[0])]


def _vocode_amplitude(S, n_iter, clip):
    """The device vocoder on an amplitude S (t, 1+n_fft//2), already ** hp.power, without its de-emphasis.  `clip`:
    clip the normalised magnitude to [0, 1], else refuse one outside it."""
    # undo the de-normalisation the device entry point applies: S = (10 ^ ((z*max_db - max_db + ref_db)/20)) ^ power
    z = (20.0 * np.log10(np.maximum(S, 1e-30) ** (1.0 / hp.power)) + hp.max_db - hp.ref_db) / hp.max_db
    if not clip and (z.min() < 0 or z.max() > 1):
        raise ValueError("griffin_lim: amplitude outside the range spectrogram2wav can produce")
    wav, _ = get_engine().spectrogram2wav(np.clip(z, 0, 1)[None].astype(np.float32), n_iter=n_iter)
    # spectrogram2wav also de-pre-emphasises; Griffin-Lim alone does not: invert y[n] = x[n] + c y[n-1]
    y = wav[0].cpu().numpy().astype(np.float64)
    x = y.copy()
    x[1:] -= hp.preemphasis * y[:-1]
    return x.astype(np.float32)


def griffin_lim(spectrogram):
    """utils.py:96-107.  spectrogram: (1+n_fft//2, t) amplitude (already ** hp.power) -> waveform."""
    return _vocode_amplitude(np.asarray(spectrogram, np.float32).T, -1, clip=False)


def invert_spectrogram(spectrogram):
    """utils.py:109-114: one inverse STFT (librosa.istft conventions) = Griffin-Lim with zero iterations."""
    S = np.asarray(spectrogram)
    if np.iscomplexobj(S):
        raise NotImplementedError("invert_spectrogram: only zero-phase (real) input is exposed; the complex "
                                  "iterations run inside dctts_spectrogram2wav")
    return _vocode_amplitude(S.T, 0, clip=True)


def _read_wav(fpath):
    """The samples of a WAV file at hp.sr as scipy reads them (raises for another sample rate)."""
    y, sr = _read_raw(fpath)
    if sr != hp.sr:
        raise ValueError("%s: sample rate %d != hp.sr %d (this reader does not resample; _read_pcm returns the native rate)"
                         % (fpath, sr, hp.sr))
    return y


def _read_raw(fpath):
    from scipy.io import wavfile
    sr, y = wavfile.read(fpath)
    return y, int(sr)


def _read_pcm(fpath):
    """(samples, native sample rate) of a WAV file for the batched feature path: mono int16 stays int16 (the device
    divides by 32768, exactly as `_load_wav` does); every other format is converted on the host by `_load_wav`'s rules."""
    y, sr = _read_raw(fpath)
    return (y if (y.ndim == 1 and y.dtype == np.int16) else _load_wav_samples(y)), sr


def _read_pcm_for(fpath, resample):
    """`_read_pcm`, refusing a file at another rate than hp.sr unless the caller asked to `resample` it."""
    y, sr = _read_pcm(fpath)
    if sr != hp.sr and not resample:
        raise ValueError("%s: sample rate %d != hp.sr %d (pass resample=True to resample it to hp.sr)" % (fpath, sr, hp.sr))
    return y, sr


def _load_pcm(fpath):
    """`_read_pcm` for a file that must already be at hp.sr (raises for another sample rate)."""
    return _read_pcm_for(fpath, False)[0]


def _load_wav(fpath):
    """What `librosa.load(fpath, sr=hp.sr)` returns for a mono PCM / float WAV that already has hp.sr."""
    return _load_wav_samples(_read_wav(fpath))


def _load_wav_samples(y):
    """librosa's buf_to_float then to_mono: each channel is scaled to float32 first, then the channels are averaged."""
    if y.dtype == np.int16:
        y = y.astype(np.float32) / 32768.0
    elif y.dtype == np.int32:
        y = y.astype(np.float32) / 2147483648.0
    elif y.dtype == np.uint8:
        y = (y.astype(np.float32) - 128.0) / 128.0
    y = np.asarray(y, np.float32)
    if y.ndim > 1:
        y = y.mean(axis=1)
    return np.ascontiguousarray(y, np.float32)


def _path(fpath):
    return isinstance(fpath, (str, bytes, os.PathLike))


def get_spectrograms(fpath, resample=False):
    """utils.py:20-65.  `fpath`: a WAV file path at hp.sr -- or at any rate with `resample=True`, resampled to hp.sr on
    the device first as librosa.load(fpath, sr=hp.sr) does -- or the already loaded waveform (1-D float array at hp.sr).
    Returns normalised mel (T, n_mels) and linear magnitude (T, 1+n_fft/2), float32 numpy."""
    e = get_engine()
    if _path(fpath):
        y, sr = _read_pcm_for(fpath, resample)
        y = e.resample_batch([y], [sr])[0] if sr != hp.sr else _load_wav_samples(y)
    else:
        y = np.asarray(fpath, np.float32)
    mel, mag, _ = e.get_spectrograms(y)
    return mel.cpu().numpy(), mag.cpu().numpy()


def load_spectrograms(fpath, resample=False):
    """utils.py:147-162: pads T to a multiple of hp.r and keeps every r-th mel frame (`resample`: see get_spectrograms)."""
    fname = os.path.basename(fpath) if _path(fpath) else None
    mel, mag = get_spectrograms(fpath, resample)
    t = mel.shape[0]
    num_paddings = hp.r - (t % hp.r) if t % hp.r != 0 else 0
    mel = np.pad(mel, [[0, num_paddings], [0, 0]], mode="constant")
    mag = np.pad(mag, [[0, num_paddings], [0, 0]], mode="constant")
    mel = mel[::hp.r, :]
    return fname, mel, mag


def load_spectrograms_batch(fpaths, engine=None, resample=False):
    """`load_spectrograms` for several WAV files in one device call (`Engine.load_spectrograms_batch`), padded with zeros
    as one bucketed batch; with `resample=True` the files may be at any sample rates and are resampled to hp.sr first.
    Returns (fnames, mels (B, T_b, n_mels), mags (B, r T_b, F), t): CUDA tensors, and the reduced rows t (B,) of each
    utterance -- utterance b is mels[b, :t[b]], mags[b, :r t[b]], bit for bit what `load_spectrograms` returns for it."""
    pcms, rates = zip(*[_read_pcm_for(p, resample) for p in fpaths])
    mels, mags, t, _ = (engine or get_engine()).load_spectrograms_batch(list(pcms), rates=list(rates))
    return [os.path.basename(p) for p in fpaths], mels, mags, t


def guided_attention(g=0.2):
    """utils.py:134-140: W[n, t] = 1 - exp(-(t/max_T - n/max_N)^2 / (2 g^2)), shape (max_N, max_T) float32 (the device
    training step builds the same table itself: dctts_train_init)."""
    n = np.arange(hp.max_N, dtype=np.float64)[:, None] / float(hp.max_N)
    t = np.arange(hp.max_T, dtype=np.float64)[None, :] / float(hp.max_T)
    return (1.0 - np.exp(-(t - n) ** 2 / (2.0 * g * g))).astype(np.float32)


# 256-entry viridis table from a published degree-6 polynomial fit of matplotlib's viridis (per channel, t in [0, 1])
_VIRIDIS_FIT = np.array([[0.2777273272234177, 0.005407344544966578, 0.3340998053353061],
                         [0.1050930431085774, 1.404613529898575, 1.384590162594685],
                         [-0.3308618287255563, 0.214847559468213, 0.09509516302823659],
                         [-4.634230498983486, -5.799100973351585, -19.33244095627987],
                         [6.228269936347081, 14.17993336680509, 56.69055260068105],
                         [4.776384997670288, -13.74514537774601, -65.35303263337234],
                         [-5.435455855934631, 4.645852612178535, 26.3124352495832]])


def _viridis():
    t = np.linspace(0.0, 1.0, 256)[:, None]
    rgb = sum(c[None, :] * t ** k for k, c in enumerate(_VIRIDIS_FIT))
    return np.round(np.clip(rgb, 0, 1) * 255).astype(np.uint8)


def plot_alignment(alignment, gs, dir=hp.logdir):
    """utils.py:116-132: writes `{dir}/alignment_{gs}.png` of an (N, T) alignment -- N rows, T columns, row 0 at the top
    as imshow draws it, scaled from its min to its max through a 256-entry viridis table and enlarged by an integer factor
    (at least 400 pixels on the shorter side, at most 4 times).  No title, axes or colorbar (matplotlib is not used).
    Returns the path."""
    from .summary import png
    os.makedirs(dir, exist_ok=True)
    a = np.asarray(alignment, np.float64)
    if a.ndim != 2:
        raise ValueError("plot_alignment: alignment must be (N, T), got shape %s" % (a.shape,))
    lo, hi = np.nanmin(a), np.nanmax(a)
    idx = np.zeros(a.shape, np.int64) if not hi > lo else np.clip(np.floor((a - lo) / (hi - lo) * 255.0 + 0.5), 0, 255).astype(np.int64)
    k = max(1, min(4, -(-400 // max(1, min(a.shape)))))
    px = np.repeat(np.repeat(_viridis()[idx], k, axis=0), k, axis=1)
    path = os.path.join(dir, "alignment_{}.png".format(gs))
    with open(path, "wb") as f:
        f.write(png(px))
    return path


def learning_rate_decay(init_lr, global_step, warmup_steps=4000.):
    """utils.py:142-145, the Noam scheme: step = global_step + 1; lr * warmup^0.5 * min(step * warmup^-1.5, step^-0.5)."""
    step = float(global_step + 1)
    return float(init_lr) * warmup_steps ** 0.5 * min(step * warmup_steps ** -1.5, step ** -0.5)
