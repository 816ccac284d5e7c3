"""Hyperparameters at another corpus rate, as a user sets them in hyperparams.py: `sr`, and with it `hop_length` and
`win_length` (12.5 ms and 50 ms of samples), and `n_fft`.  Tests build engines and run the oracles inside `at_rate`,
which patches the Hyperparams class (read by the engine, the oracles and the Python layers) and restores it."""
import contextlib

from dc_tts_b200.hyperparams import Hyperparams

# (sr, n_fft): the smallest power-of-two n_fft of at least win_length at each rate
RATES = {16000: 1024, 22050: 2048, 24000: 2048, 32000: 2048, 44100: 4096, 48000: 4096}


def rate_values(sr, n_fft=None):
    n_fft = n_fft or RATES[sr]
    return dict(sr=sr, n_fft=n_fft, hop_length=int(sr * Hyperparams.frame_shift),
                win_length=int(sr * Hyperparams.frame_length))


@contextlib.contextmanager
def at_rate(sr, n_fft=None):
    vals = rate_values(sr, n_fft)
    old = {k: getattr(Hyperparams, k) for k in vals}
    for k, v in vals.items():
        setattr(Hyperparams, k, v)
    try:
        yield Hyperparams
    finally:
        for k, v in old.items():
            setattr(Hyperparams, k, v)
