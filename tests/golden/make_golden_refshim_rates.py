"""Generates refshim_sample_rates.npz: the reference's own utils.spectrogram2wav (3 iterations), get_spectrograms and
load_spectrograms at (sr, n_fft) = (16000, 1024), (44100, 4096) and (48000, 4096), executed under the TensorFlow API
stand-in of tf_shim.py with the restated librosa primitives (oracle/ref_vocoder.py, ref_features.py) standing in for the
absent librosa.  The reference's Hyperparams computes hop_length and win_length from sr when its class is created, so
all of sr, n_fft, hop_length and win_length are set.  tests/test_reference_shim_rates.py checks the fixture against the
oracle's composition, and runs `reference_outputs` live where the reference is present.  Run from the repo root:
    python tests/golden/make_golden_refshim_rates.py
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

RATES = ((16000, 1024), (44100, 4096), (48000, 4096))


def rate_inputs(sr, n_fft):
    """(magnitudes (12, F), 0.25 s waveform with a quiet lead) from a seed per rate."""
    rng = np.random.default_rng(sr)
    mag = rng.uniform(0.2, 0.8, (12, 1 + n_fft // 2)).astype(np.float32)
    t = np.arange(int(sr * 0.25)) / sr
    y = (0.2 * np.sin(2 * np.pi * 300 * t) + 0.02 * rng.standard_normal(t.size)).astype(np.float32)
    y[:t.size // 4] *= 1e-5
    return mag, y


def reference_outputs():
    """{key: array} of the reference's utils at every rate of RATES (needs the reference at tf_shim.REFERENCE)."""
    import tf_shim
    from oracle import ref_features as rf
    from oracle import ref_vocoder as rv
    tf_shim.install(tf_shim.Store({}))
    import hyperparams as ref_hp
    import utils as ref_utils
    H = ref_hp.Hyperparams
    wavs = {}
    old_lib = getattr(ref_utils, "librosa", None)
    ref_utils.librosa = types.SimpleNamespace(
        stft=lambda y, n_fft=None, hop_length=None, win_length=None: rv.stft(np.asarray(y, np.float32), n_fft, hop_length, win_length),
        istft=lambda S, hop_length=None, win_length=None, window="hann": rv.istft(S, hop_length, win_length),
        effects=types.SimpleNamespace(trim=lambda y: (lambda se: (y[se[0]:se[1]], se))(rv.trim_indices(np.asarray(y)))),
        filters=types.SimpleNamespace(mel=lambda sr, n_fft, n_mels: rf.mel_basis(sr, n_fft, n_mels)),
        load=lambda fpath, sr=None: (wavs[fpath], sr))
    keys = ("sr", "n_fft", "hop_length", "win_length", "n_iter")
    old = {k: getattr(H, k) for k in keys}
    out = {}
    try:
        for sr, n_fft in RATES:
            H.sr, H.n_fft, H.n_iter = sr, n_fft, 3
            H.hop_length, H.win_length = int(sr * H.frame_shift), int(sr * H.frame_length)
            mag, y = rate_inputs(sr, n_fft)
            out["wav_%d" % sr] = ref_utils.spectrogram2wav(mag)
            wavs["LJ001-0001.wav"] = y
            mel, mg = ref_utils.get_spectrograms("LJ001-0001.wav")
            out["get_mel_%d" % sr] = mel                    # get_mag is load_mag before the padding to a multiple of r
            out["get_frames_%d" % sr] = np.array(len(mg))
            fname, mel, mg = ref_utils.load_spectrograms("LJ001-0001.wav")
            assert fname == "LJ001-0001.wav"
            out["load_mel_%d" % sr], out["load_mag_%d" % sr] = mel, mg
    finally:
        for k, v in old.items():
            setattr(H, k, v)
        ref_utils.librosa = old_lib
    return out


if __name__ == "__main__":
    np.savez_compressed(os.path.join(HERE, "refshim_sample_rates.npz"), **reference_outputs())
    print("refshim_sample_rates.npz written to %s" % HERE)
