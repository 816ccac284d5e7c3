"""End to end at 44.1 kHz with n_fft = 4096 (F = 2049): synthesize() from a text file to wav files, and SSRN training
straight from a small wav corpus (hp.prepro = False).  Hyperparams are patched for the module (`at_rate`) and restored."""
import numpy as np
import pytest

from dc_tts_b200 import trainer
from dc_tts_b200.params import init_params

from sample_rates import at_rate

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def hp441():
    with at_rate(44100) as H:
        yield H


@pytest.fixture(scope="module")
def eng441(hp441):
    from dc_tts_b200.engine import Engine
    e = Engine(0, hparams=hp441)
    yield e
    e.close()


def test_synthesize_writes_441_khz_wavs(hp441, eng441, tmp_path, monkeypatch):
    from scipy.io.wavfile import read as read_wav
    from dc_tts_b200 import synthesize as syn
    from dc_tts_b200.engine import get_engine, set_engine
    path = tmp_path / "s.txt"
    path.write_text("header\n1. The birch canoe slid on the smooth planks.\n2. Glue the sheet to the dark blue background.\n")
    monkeypatch.chdir(tmp_path)
    prev = get_engine()
    set_engine(eng441)
    try:
        Y, Z = syn.synthesize(params=init_params(0), sentences=str(path), fast=True, write=True)
    finally:
        set_engine(prev)
    Z = np.asarray(Z.cpu().numpy() if hasattr(Z, "cpu") else Z)
    assert Z.shape == (2, 4 * hp441.max_T, 2049) and np.isfinite(Z).all()
    wav, trim = eng441.spectrogram2wav(Z)
    assert wav.shape == (2, 551 * (840 - 1))                     # untrimmed: hop (T - 1) at 44.1 kHz
    for i in range(2):
        sr, w = read_wav(tmp_path / "samples" / ("%d.wav" % (i + 1)))
        assert sr == 44100 and w.dtype == np.float32 and np.isfinite(w).all()
        assert len(w) == trim[i, 1] - trim[i, 0] and 0 < len(w) <= 551 * 839


def test_ssrn_training_from_441_khz_wavs(hp441, tmp_path):
    from dc_tts_b200.engine import Engine
    from test_gpu_wav_features import _wav_corpus
    d = _wav_corpus(tmp_path, n=10, seed=2)                      # int16 wavs written at hp.sr = 44100
    fpaths, lens, texts = trainer.load_train_data(d)
    eng = Engine(0, hparams=hp441)
    eng.load_params(init_params(1))
    losses, log = [], []
    step = eng.train_step_ssrn

    def recording(*a, **k):
        out = step(*a, **k)
        losses.append(out["loss"])
        return out
    eng.train_step_ssrn = recording
    batches = trainer.bucketed_batches(fpaths, lens, texts, B=4, seed=0, prepro=False, engine=eng)
    gs = trainer.train(2, eng, batches, num_iterations=5, logdir=str(tmp_path / "log"), global_step=0, save_every=10 ** 9,
                       log=log.append)
    assert gs == 6 and len(losses) == 6 and np.isfinite(losses).all(), (gs, losses, log)
    assert eng.train_tensor("SSRN/C_16/conv1d/bias", "param").shape == (2049,)
    eng.close()
