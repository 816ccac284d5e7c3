"""Configuration surface of the DC-TTS synthesis path.

Mirror of the reference's `Hyperparams` class (/root/reference/hyperparams.py:7-47):
same attribute names, same values, imported everywhere as `hp`.  The north star
requires this surface to stay drop-in, so every attribute the reference defines is
kept -- including the ones only the out-of-scope trainer/DSP code reads -- but the
kernels only specialise on the "model" and "data" groups below.

Note (reference hyperparams.py:17): hop_length evaluates to int(22050*0.0125) = 275,
not the 276 its comment claims; win_length = 1102.
"""


class Hyperparams:
    # --- pipeline -----------------------------------------------------------
    prepro = True            # False: trainer.bucketed_batches computes the features from the wavs on the device

    # --- signal processing (only used by the out-of-scope vocoder/feature code)
    sr = 22050
    n_fft = 2048
    frame_shift = 0.0125
    frame_length = 0.05
    hop_length = int(sr * frame_shift)      # 275 samples
    win_length = int(sr * frame_length)     # 1102 samples
    n_mels = 80
    power = 1.5
    n_iter = 50
    preemphasis = .97
    max_db = 100
    ref_db = 20

    # --- model --------------------------------------------------------------
    r = 4                    # reduction factor (fixed by the architecture)
    dropout_rate = 0.05
    e = 128                  # embedding width
    d = 256                  # Text2Mel hidden units
    c = 512                  # SSRN hidden units
    attention_win_size = 3

    # --- data ---------------------------------------------------------------
    data = "/data/private/voice/LJSpeech-1.0"
    test_data = 'harvard_sentences.txt'
    vocab = "PE abcdefghijklmnopqrstuvwxyz'.?"   # P: padding (id 0), E: end of sentence (id 1)
    max_N = 180              # characters per utterance
    max_T = 210              # reduced mel frames per utterance

    # --- training scheme (trainer is out of scope; kept for API parity) -------
    lr = 0.001
    logdir = "logdir/LJ01"
    sampledir = 'samples'
    B = 32
    num_iterations = 2000000


# Derived constants used by the synthesis path and the benchmark.
def n_mags(hp=Hyperparams):
    """Linear-spectrogram bins F = 1 + n_fft/2 (reference networks.py:269)."""
    return 1 + hp.n_fft // 2


def seconds_per_mel_frame(hp=Hyperparams):
    """Audio seconds covered by one reduced mel frame: r * hop / sr (SURVEY.md 8d)."""
    return hp.r * hp.hop_length / float(hp.sr)
