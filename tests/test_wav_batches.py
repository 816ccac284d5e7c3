"""The wav route of trainer.bucketed_batches (hp.prepro = False, data_load.py:104-113): the buckets collect the samples of
the wav files and a full bucket gets its features from one batched call.  On the CPU the feature call is the oracle
(oracle/ref_features.load_spectrograms, padded per batch), so these tests check that routing, sharding and padding do
not depend on the route."""
import os

import numpy as np
import pytest

from dc_tts_b200 import trainer
from dc_tts_b200.hyperparams import Hyperparams as hp
from oracle import ref_features as rf


def _clip(rng, seconds):
    n = int(hp.sr * seconds)
    t = np.arange(n) / hp.sr
    f0 = rng.uniform(120, 300)
    y = 0.3 * np.sin(2 * np.pi * f0 * t) * (0.5 + 0.5 * np.sin(2 * np.pi * 3 * t)) + 0.03 * rng.standard_normal(n)
    lead, tail = int(rng.integers(800, 3000)), int(rng.integers(800, 3000))
    y[:lead] *= 1e-4
    y[n - tail:] *= 1e-4
    return np.round(np.clip(y, -1, 1) * 32767).astype(np.int16)


def _corpus(root, n=14, seed=0):
    """LJ-shaped: transcript.csv, wavs/*.wav (int16, hp.sr), and mels/ mags/ written from the oracle as prepo.py would."""
    from scipy.io import wavfile
    rng = np.random.default_rng(seed)
    d = root / "LJSpeech-1.0"
    (d / "wavs").mkdir(parents=True)
    (root / "mels").mkdir(); (root / "mags").mkdir()
    lines = []
    for i in range(n):
        name = "LJ%03d" % i
        lines.append("%s|raw|%s" % (name, "".join(rng.choice(list("abcdefghijklmnopqrstuvwxyz '"), int(rng.integers(10, 90))))))
        pcm = _clip(rng, float(rng.uniform(0.25, 0.8)))
        wavfile.write(str(d / "wavs" / (name + ".wav")), hp.sr, pcm)
        mel, mag = rf.load_spectrograms(pcm.astype(np.float32) / 32768.0)
        np.save(root / "mels" / (name + ".npy"), mel); np.save(root / "mags" / (name + ".npy"), mag)
    (d / "transcript.csv").write_text("\n".join(lines) + "\n", encoding="utf-8")
    return str(d)


def oracle_features(pcms):
    """What the batched device call returns, from the oracle: each utterance's load_spectrograms, zero-padded."""
    out = [rf.load_spectrograms(p.astype(np.float32) / 32768.0 if p.dtype == np.int16 else p) for p in pcms]
    T_b = max(m.shape[0] for m, _ in out)
    mels = np.zeros((len(out), T_b, hp.n_mels), np.float32)
    mags = np.zeros((len(out), hp.r * T_b, 1 + hp.n_fft // 2), np.float32)
    for b, (m, g) in enumerate(out):
        mels[b, :m.shape[0]] = m; mags[b, :g.shape[0]] = g
    return mels, mags


@pytest.mark.parametrize("rank,world", [(0, 1), (0, 2), (1, 2)])
def test_wav_route_yields_the_npy_routes_batches(tmp_path, rank, world):
    d = _corpus(tmp_path)
    fpaths, lens, texts = trainer.load_train_data(d)
    loader = lambda p: trainer._load_spectrograms_npy(p, str(tmp_path / "mels"), str(tmp_path / "mags"))
    kw = dict(B=2, seed=5, epochs=2, rank=rank, world=world)
    npy = list(trainer.bucketed_batches(fpaths, lens, texts, loader=loader, prepro=True, **kw))
    wav = list(trainer.bucketed_batches(fpaths, lens, texts, loader=None, prepro=False, features=oracle_features, **kw))
    assert len(npy) == len(wav) > 2
    for (L0, m0, g0, n0, k0), (L1, m1, g1, n1, k1) in zip(npy, wav):
        assert n0 == n1 and k0 == k1 and np.array_equal(L0, L1)
        assert m0.shape == m1.shape and g0.shape == g1.shape
        assert np.array_equal(m0, m1) and np.array_equal(g0, g1)


def test_default_route_is_the_npy_loader(tmp_path):
    assert hp.prepro is True
    d = _corpus(tmp_path, n=6)
    fpaths, lens, texts = trainer.load_train_data(d)
    read = []

    def loader(p):
        read.append(os.path.basename(p))
        return trainer._load_spectrograms_npy(p, str(tmp_path / "mels"), str(tmp_path / "mags"))

    def features(pcms):
        raise AssertionError("the npy route must not compute features")

    batches = list(trainer.bucketed_batches(fpaths, lens, texts, B=1, seed=0, loader=loader, epochs=1, features=features))
    assert len(batches) == 6 and sorted(read) == sorted(os.path.basename(p) for p in fpaths)
    assert all(isinstance(b[1], np.ndarray) for b in batches)


def test_wav_route_reads_files_like_load_wav(tmp_path):
    """Mono int16 goes to the feature call as int16; other formats arrive converted by utils._load_wav's rules."""
    from scipy.io import wavfile
    from dc_tts_b200 import utils
    rng = np.random.default_rng(3)
    pcm = _clip(rng, 0.3)
    wavfile.write(str(tmp_path / "a.wav"), hp.sr, pcm)
    wavfile.write(str(tmp_path / "b.wav"), hp.sr, np.stack([pcm, pcm // 2], 1))
    wavfile.write(str(tmp_path / "c.wav"), hp.sr, pcm.astype(np.float32) / 32768.0)
    a = utils._load_pcm(str(tmp_path / "a.wav"))
    assert a.dtype == np.int16 and np.array_equal(a, pcm)
    for name in ("b.wav", "c.wav"):
        got = utils._load_pcm(str(tmp_path / name))
        assert got.dtype == np.float32 and np.array_equal(got, utils._load_wav(str(tmp_path / name)))
    wavfile.write(str(tmp_path / "d.wav"), 16000, pcm)
    with pytest.raises(ValueError, match="sample rate"):
        utils._load_pcm(str(tmp_path / "d.wav"))
