"""ORACLE (test infrastructure) -- the fast Griffin-Lim algorithm (Perraudin, Balazs and Sondergaard 2013) on top of
oracle/ref_vocoder.py's stft / istft, in float32 or float64, with the spectral convergence of every iteration.

The update is librosa's griffinlim(momentum=...) as recalled, UNPINNED (librosa is absent offline), with the reference's
zero initial phase and its max(1e-8, .) normaliser where librosa divides by |c| + eps (DESIGN.md section 8b):
alpha = momentum / (1 + momentum) in float64, rounded to the spectrogram's precision as numpy does for
complex64 * Python float; est_i = stft(istft(X_i)), est_{-1} = 0, c = est_i - alpha est_{i-1},
X_{i+1} = S c / max(1e-8, |c|).  alpha = 0 skips the subtraction: ref_vocoder.griffin_lim, bit for bit."""
import numpy as np

from dc_tts_b200.hyperparams import Hyperparams as hp
from oracle import ref_vocoder as rv


def spectral_convergence(S, est):
    """||S - |est||| / ||S|| (Frobenius norms), in float64."""
    S = np.asarray(S, np.float64)
    return float(np.linalg.norm(S - np.abs(est).astype(np.float64)) / np.linalg.norm(S))


def fast_griffin_lim(spectrogram, n_iter=None, momentum=0.0, convergence=False):
    """spectrogram: (F, T) amplitude.  Returns the waveform, and with `convergence` also the n_iter + 1 spectral
    convergences of est_0 .. est_{n_iter} (the last from one more stft of the waveform)."""
    n_iter = hp.n_iter if n_iter is None else n_iter
    S = spectrogram
    alpha = np.float32(momentum / (1.0 + momentum)) if S.dtype in (np.float32, np.complex64) else momentum / (1.0 + momentum)
    X_best = S.copy()
    prev = None
    hist = []
    for _ in range(n_iter):
        est = rv.stft(rv.istft(X_best))
        if convergence:
            hist.append(spectral_convergence(S, est))
        c = est if alpha == 0 else est - alpha * (prev if prev is not None else np.zeros_like(est))
        prev = est
        X_best = S * (c / np.maximum(1e-8, np.abs(c)))
    y = np.real(rv.istft(X_best))
    if convergence:
        hist.append(spectral_convergence(S, rv.stft(y)))
        return y, np.array(hist)
    return y
