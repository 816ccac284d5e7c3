"""ORACLE (test infrastructure, not product) -- numpy restatement of the resampling inside `librosa.load(fpath, sr=hp.sr)`
(/root/reference/utils.py:32): librosa 0.6 core.resample(y, orig_sr, target_sr, res_type='kaiser_best', fix=True), which
calls resampy 0.2 resample / resample_f with the 'kaiser_best' filter.

librosa and resampy are absent offline.  The filter constants (beta, rolloff, 64 zero crossings, precision 9) are
resampy's documented 'kaiser_best' values as recalled, not checked against resampy's shipped table: parity unpinned.
What is pinned here is the arithmetic of resample_f given the table:
  - the time register is the literal sequential float64 sum 0, inc, inc + inc, ... (np.cumsum is sequential);
  - per output, n = int(reg), frac = scale (reg - n), offset = int(512 frac), eta = 512 frac - offset, the left wing on
    x[n - i], then frac = scale - frac and the right wing on x[n + k + 1];
  - the accumulator is float32 and every tap rounds float32(double(y) + weight * double(x)) (numba, float32 y),
    vectorised over the outputs with one tap per iteration, in resample_f's tap order.
"""
import numpy as np
import scipy.signal

ZEROS = 64
PRECISION = 9
BETA = 14.769656459379492
ROLLOFF = 0.9475937167399596


def kaiser(M, beta):
    """scipy.signal.kaiser(M, beta) (symmetric), the window resampy's filters were built with."""
    return scipy.signal.windows.kaiser(M, beta, sym=True)


def sinc_window(num_zeros=ZEROS, precision=PRECISION, beta=BETA, rolloff=ROLLOFF):
    """resampy.filters.sinc_window with a Kaiser taper: (interp_win (num_zeros 2^precision + 1,), 2^precision, rolloff)."""
    num_bits = 2 ** precision
    n = num_bits * num_zeros
    sinc_win = rolloff * np.sinc(rolloff * np.linspace(0, num_zeros, num=n + 1, endpoint=True))
    taper = kaiser(2 * n + 1, beta)[n:]
    return taper * sinc_win, num_bits, rolloff


def time_register(n_out, sample_ratio):
    """resample_f's `time_register` before each output: 0, then `time_register += time_increment` in float64."""
    reg = np.zeros(n_out, np.float64)
    if n_out > 1:
        reg[1:] = np.cumsum(np.full(n_out - 1, 1. / sample_ratio))
    return reg


def resample_f(x, n_out, sample_ratio, interp_win, interp_delta, num_table):
    x = np.asarray(x, np.float32)
    scale = min(1.0, sample_ratio)
    index_step = int(scale * num_table)
    nwin, n_orig = interp_win.shape[0], x.shape[0]
    xd = x.astype(np.float64)
    reg = time_register(n_out, sample_ratio)
    n = reg.astype(np.int64)
    frac = scale * (reg - n)
    y = np.zeros(n_out, np.float32)

    def wing(frac, count, src):
        index_frac = frac * num_table
        offset = index_frac.astype(np.int64)
        eta = index_frac - offset
        count = np.minimum(count, (nwin - offset) // index_step)
        for i in range(int(count.max(initial=0))):
            m = i < count
            j = offset[m] + i * index_step
            w = interp_win[j] + eta[m] * interp_delta[j]
            y[m] = (y[m].astype(np.float64) + w * xd[src(n[m], i)]).astype(np.float32)

    wing(frac, n + 1, lambda n, i: n - i)                       # left wing
    wing(scale - frac, n_orig - n - 1, lambda n, k: n + k + 1)  # right wing
    return y


def resample(x, sr_orig, sr_new):
    """resampy.resample(x, sr_orig, sr_new, filter='kaiser_best') for a 1-D float32 signal: int(n ratio) samples."""
    sample_ratio = float(sr_new) / sr_orig
    n_out = int(x.shape[-1] * sample_ratio)
    if n_out < 1:
        raise ValueError("Input signal length=%d is too small to resample from %d->%d" % (x.shape[-1], sr_orig, sr_new))
    interp_win, precision, _ = sinc_window()
    if sample_ratio < 1:
        interp_win *= sample_ratio
    interp_delta = np.zeros_like(interp_win)
    interp_delta[:-1] = np.diff(interp_win)
    return resample_f(x, n_out, sample_ratio, interp_win, interp_delta, precision)


def librosa_resample(y, orig_sr, target_sr):
    """librosa.core.resample(y, orig_sr, target_sr, res_type='kaiser_best', fix=True): y itself at equal rates, else
    resampy's output zero-padded to ceil(n ratio) (util.fix_length), float32."""
    y = np.asarray(y, np.float32)
    if orig_sr == target_sr:
        return y
    ratio = float(target_sr) / orig_sr
    n_samples = int(np.ceil(y.shape[-1] * ratio))
    y_hat = resample(y, orig_sr, target_sr)
    out = np.zeros(n_samples, np.float32)
    out[:y_hat.size] = y_hat
    return out


def load(pcm, sr_native, sr):
    """librosa.load(fpath, sr=sr) after decoding: int16 PCM as value / 32768 (float32), then resampled to sr."""
    y = pcm.astype(np.float32) / np.float32(32768.0) if pcm.dtype == np.int16 else np.asarray(pcm, np.float32)
    return librosa_resample(y, sr_native, sr)
