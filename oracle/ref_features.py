"""ORACLE (test infrastructure, not product) -- numpy restatement of the reference's feature extraction
`get_spectrograms` / `load_spectrograms` (/root/reference/utils.py:20-65, 147-162) from a waveform array on
(file decoding and resampling, `librosa.load`, are outside: LJ Speech is already 22050 Hz PCM).

Third-party pieces restated from librosa 0.6 (absent offline; pinned by independent librosa-compatible implementations:
torch.stft for the STFT, transformers.audio_utils.mel_filter_bank(slaney) for the filterbank -- equal to 1e-16 -- and by
the reference's own get_spectrograms / load_spectrograms executed with these primitives, tests/test_reference_shim.py):
  effects.trim        ref_vocoder.trim_indices
  core.stft           ref_vocoder.stft
  filters.mel(sr, n_fft, n_mels)   Slaney scale (htk=False), fmin 0, fmax sr/2, area normalisation (norm=1):
      mel(f) = f / (200/3) below 1 kHz, 15 + ln(f/1000) / (ln(6.4)/27) above; n_mels + 2 points equally spaced
      in mel; triangular weights max(0, min((f - f[i]) / (f[i+1]-f[i]), (f[i+2] - f) / (f[i+2]-f[i+1]))) on the
      FFT bin frequencies linspace(0, sr/2, 1 + n_fft/2), each row scaled by 2 / (f[i+2] - f[i]).
"""
import numpy as np

from dc_tts_b200.hyperparams import Hyperparams as hp

from . import ref_vocoder as rv


def hz_to_mel(f):
    f = np.asarray(f, np.float64)
    f_sp = 200.0 / 3
    mels = f / f_sp
    min_log_hz, min_log_mel, logstep = 1000.0, 1000.0 / f_sp, np.log(6.4) / 27.0
    return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-300) / min_log_hz) / logstep, mels)


def mel_to_hz(m):
    m = np.asarray(m, np.float64)
    f_sp = 200.0 / 3
    min_log_hz, min_log_mel, logstep = 1000.0, 1000.0 / f_sp, np.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)


def mel_basis(sr=None, n_fft=None, n_mels=None):
    """librosa.filters.mel(sr, n_fft, n_mels) -> (n_mels, 1 + n_fft//2) float64."""
    sr = sr or hp.sr; n_fft = n_fft or hp.n_fft; n_mels = n_mels or hp.n_mels
    fftfreqs = np.linspace(0, sr / 2.0, 1 + n_fft // 2)
    mel_f = mel_to_hz(np.linspace(hz_to_mel(0.0), hz_to_mel(sr / 2.0), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - fftfreqs[None, :]
    w = np.zeros((n_mels, 1 + n_fft // 2))
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        w[i] = np.maximum(0, np.minimum(lower, upper))
    return w * (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None]


def get_spectrograms(y, dtype=np.float32):
    """utils.py:33-65 from the loaded waveform `y` (float32, hp.sr) -> (mel (T, n_mels), mag (T, 1+n_fft/2)).
    dtype=np.float64 runs everything after the (float32) trim and pre-emphasis in float64."""
    y = np.asarray(y, np.float32)
    s, e = rv.trim_indices(y)                                             # :36
    y = y[s:e]
    y = np.append(y[0], y[1:] - hp.preemphasis * y[:-1]).astype(np.float32)   # :39 (float32 in, float32 out)
    linear = rv.stft(y.astype(dtype))                                     # :42-45  (F, T) complex64
    mag = np.abs(linear)                                                  # :48
    mel = np.dot(mel_basis(), mag)                                        # :51-52
    mel = 20 * np.log10(np.maximum(1e-5, mel))                            # :55-56
    mag = 20 * np.log10(np.maximum(1e-5, mag))
    mel = np.clip((mel - hp.ref_db + hp.max_db) / hp.max_db, 1e-8, 1)     # :59-60
    mag = np.clip((mag - hp.ref_db + hp.max_db) / hp.max_db, 1e-8, 1)
    return mel.T.astype(dtype), mag.T.astype(dtype)


def load_spectrograms(y, dtype=np.float32):
    """utils.py:147-162 (without the file name): pad T to a multiple of hp.r, keep every r-th mel frame."""
    mel, mag = get_spectrograms(y, dtype)
    t = mel.shape[0]
    num_paddings = hp.r - (t % hp.r) if t % hp.r != 0 else 0
    mel = np.pad(mel, [[0, num_paddings], [0, 0]], mode="constant")
    mag = np.pad(mag, [[0, num_paddings], [0, 0]], mode="constant")
    return mel[::hp.r, :], mag
