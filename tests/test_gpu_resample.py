"""Resampling on the device (`dctts_resample_batch`, Engine.resample_batch) and feature extraction from files at any
sample rate (Engine.load_spectrograms_batch(..., rates=...), utils.load_spectrograms, the wav route of the trainer)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from dc_tts_b200 import prepo as prepo_mod
from dc_tts_b200 import trainer, utils
from dc_tts_b200.engine import DcttsError, Engine
from dc_tts_b200.hyperparams import Hyperparams as hp
from dc_tts_b200.params import init_params
from oracle import ref_features as rf
from oracle import ref_resample as rr

pytestmark = pytest.mark.gpu
RATES = [8000, 11025, 16000, 24000, 32000, 44100, 48000, 96000]


def _pcm(seed, sr, n, lead=0, tail=0):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / sr
    y = 0.3 * np.sin(2 * np.pi * rng.uniform(120, 300) * t) * (0.5 + 0.5 * np.sin(2 * np.pi * 3 * t))
    y += 0.1 * np.sin(2 * np.pi * rng.uniform(2000, 0.45 * sr) * t) + 0.03 * rng.standard_normal(n)
    y[:lead] *= 1e-4
    if tail:
        y[n - tail:] *= 1e-4
    return np.round(np.clip(y, -1, 1) * 32767).astype(np.int16)


@pytest.fixture(scope="module")
def pool():
    """32 int16 clips cycling through RATES: 600 samples, 12 s, and 0.1-2.5 s; with the oracle's result for each."""
    rng = np.random.default_rng(7)
    clips = []
    for i in range(32):
        sr = RATES[i % len(RATES)]
        n = 600 if i < 8 else int(12 * sr) if i in (13, 22) else int(sr * rng.uniform(0.1, 2.5))
        clips.append((_pcm(i, sr, n), sr))
    return [(p, sr, rr.load(p, sr, hp.sr)) for p, sr in clips]


def _within_one_ulp(got, want):
    return np.abs(got - want) <= np.spacing(np.maximum(np.abs(got), np.abs(want)).astype(np.float32))


@pytest.mark.parametrize("kind", ["int16", "float32"])
@pytest.mark.parametrize("B", [1, 7, 32])
def test_resample_batch_against_the_oracle(engine, pool, B, kind):
    items = [pool[13]] if B == 1 else pool[:B]
    wavs = [p if kind == "int16" else p.astype(np.float32) / np.float32(32768.0) for p, _, _ in items]
    outs = engine.resample_batch(wavs, [sr for _, sr, _ in items])
    exact = total = 0
    for (p, sr, want), got in zip(items, outs):
        got = got.cpu().numpy()
        assert got.dtype == np.float32 and got.shape == want.shape, (sr, p.size)
        assert _within_one_ulp(got, want).all(), (sr, p.size)
        exact += int((got == want).sum())
        total += got.size
    assert exact >= 0.999 * total                       # the filter table is built in C++, the oracle's by numpy


def _files(tmp_path, specs, seed=0):
    from scipy.io import wavfile
    paths = []
    for i, (sr, seconds) in enumerate(specs):
        n = int(sr * seconds)
        p = _pcm(seed + i, sr, n, lead=int(0.1 * sr), tail=int(0.15 * sr))
        path = str(tmp_path / ("u%02d.wav" % i))
        wavfile.write(path, sr, p)
        paths.append(path)
    return paths


def _trim_margin_db(y, top_db=60):
    """How far (dB) the frame energy nearest the -60 dB threshold of librosa.effects.trim lies from it."""
    yp = np.pad(y, 1024, mode="reflect")
    n_frames = 1 + (len(yp) - 2048) // 512
    idx = np.arange(2048)[:, None] + 512 * np.arange(n_frames)[None, :]
    mse = np.mean(np.abs(yp[idx].astype(np.float64)) ** 2, axis=0)
    db = 10 * np.log10(np.maximum(1e-10, mse)) - 10 * np.log10(np.maximum(1e-10, mse.max()))
    return np.abs(db + top_db).min()


def test_mixed_rate_bucket(engine, tmp_path):
    from dc_tts_b200.engine import set_engine
    set_engine(engine)
    specs = [(22050, 1.3), (16000, 2.1), (44100, 0.9), (48000, 3.2), (44100, 2.6), (16000, 0.7), (22050, 1.8), (48000, 1.1)]
    paths = _files(tmp_path, specs)
    with pytest.raises(ValueError, match="resample=True"):
        utils.load_spectrograms_batch(paths, engine)          # other rates are refused unless asked for
    _, mels, mags, t = utils.load_spectrograms_batch(paths, engine, resample=True)
    mels, mags = mels.cpu().numpy(), mags.cpu().numpy()
    lin = lambda z: 10.0 ** ((z * hp.max_db - hp.max_db + hp.ref_db) / 20.0)
    trims_checked = 0
    for b, path in enumerate(paths):
        _, mel, mag = utils.load_spectrograms(path, resample=True)
        assert t[b] == mel.shape[0] and np.array_equal(mels[b, :t[b]], mel) and np.array_equal(mags[b, :hp.r * t[b]], mag), b
        assert not mels[b, t[b]:].any() and not mags[b, hp.r * t[b]:].any()
        pcm, sr = utils._read_pcm(path)
        y = rr.load(pcm, sr, hp.sr)
        mel_o, mag_o = rf.load_spectrograms(y)
        if _trim_margin_db(y) > 1e-3:                   # the oracle's trim is not a float32 near-tie
            _, _, tr = engine.get_spectrograms(engine.resample_batch([pcm], [sr])[0])
            from oracle import ref_vocoder as rv
            assert tr == rv.trim_indices(y), b
            assert mel_o.shape[0] == t[b]
            np.testing.assert_allclose(lin(mag), lin(mag_o), atol=2e-6 * lin(mag_o).max(), rtol=2e-3)
            np.testing.assert_allclose(lin(mel), lin(mel_o), atol=2e-6 * lin(mel_o).max(), rtol=2e-3)
            assert np.abs(mag - mag_o)[mag_o > 0.35].max() < 1e-4
            assert np.abs(mel - mel_o)[mel_o > 0.35].max() < 1e-4
            trims_checked += 1
    assert trims_checked >= 6


def test_launches_and_the_all_native_batch(engine, pool):
    native = [_pcm(40 + i, hp.sr, int(hp.sr * (0.5 + 0.3 * i))) for i in range(5)]
    n0 = engine.launch_count()
    m0, g0, t0, r0 = engine.load_spectrograms_batch(native)
    n1 = engine.launch_count()
    m1, g1, t1, r1 = engine.load_spectrograms_batch(native, rates=[hp.sr] * 5)
    n2 = engine.launch_count()
    assert n1 - n0 == n2 - n1 == 2                      # no resampling kernel when every rate is hp.sr
    assert torch.equal(m0, m1) and torch.equal(g0, g1) and np.array_equal(t0, t1) and np.array_equal(r0, r1)
    mixed = [p for p, _, _ in pool]
    rates = [sr for _, sr, _ in pool]
    engine.load_spectrograms_batch(mixed[1:2], rates=rates[1:2])
    n3 = engine.launch_count()
    engine.load_spectrograms_batch(mixed, rates=rates)
    n4 = engine.launch_count()
    assert n3 - n2 == n4 - n3 == 3


def _raw_resample(engine, wavs, rates, capacity):
    lib = engine._lib
    offsets = np.zeros(len(wavs) + 1, np.int64)
    offsets[1:] = np.cumsum([w.size for w in wavs])
    wav = torch.from_numpy(np.concatenate(wavs)).to(engine.device)
    out = torch.full((max(capacity, 1),), 7.0, device=engine.device)
    sr = np.asarray(rates, np.int32)
    oo = np.full(len(wavs) + 1, -5, np.int64)
    torch.cuda.synchronize()
    n0 = engine.launch_count()
    rc = lib.dctts_resample_batch(engine._h, C.c_void_p(wav.data_ptr()), 1, offsets.ctypes.data_as(C.POINTER(C.c_int64)),
                                  sr.ctypes.data_as(C.POINTER(C.c_int32)), len(wavs), hp.sr, C.c_void_p(out.data_ptr()), capacity,
                                  oo.ctypes.data_as(C.POINTER(C.c_int64)), None)
    torch.cuda.synchronize()
    return rc, lib.dctts_last_error(engine._h).decode(), out, oo, engine.launch_count() - n0


def test_error_paths_name_the_utterance_and_write_nothing(engine, pool):
    wavs = [p for p, _, _ in pool[8:12]]
    rates = [sr for _, sr, _ in pool[8:12]]
    need = sum(int(np.ceil(w.size * (hp.sr / float(r)))) if r != hp.sr else w.size for w, r in zip(wavs, rates))
    for bad_wavs, bad_rates, cap, text in [
            (wavs, rates[:2] + [0] + rates[3:], need, "utterance 2 has sample rate 0"),
            (wavs[:1] + [np.ones(1, np.int16)] + wavs[1:], rates[:1] + [44100] + rates[1:], need + 1, "utterance 1: 1 samples"),
            (wavs, rates, need - 1, "utterance 3 ends at output sample")]:
        rc, err, out, oo, launched = _raw_resample(engine, bad_wavs, bad_rates, cap)
        assert rc != 0 and text in err, err
        assert bool((out == 7).all()) and (oo == -5).all() and launched == 0
    with pytest.raises(DcttsError, match="utterance 1"):
        engine.load_spectrograms_batch(wavs[:1] + [np.ones(1, np.int16)], rates=[rates[0], 44100])
    rc, err, out, oo, launched = _raw_resample(engine, wavs, rates, need)
    assert rc == 0 and oo[-1] == need and launched == 1


# ------------------------------------------------------------------------------------------- training from a 44.1 kHz corpus
def _corpus_44k(root, n=20, seed=0):
    from scipy.io import wavfile
    rng = np.random.default_rng(seed)
    d = root / "LJSpeech-1.0"
    (d / "wavs").mkdir(parents=True)
    lines = []
    for i in range(n):
        lines.append("LJ%03d|raw|%s" % (i, "".join(rng.choice(list("abcdefghijklmnopqrstuvwxyz '"), int(rng.integers(10, 120))))))
        sr = 44100
        m = int(sr * float(rng.uniform(0.5, 3.0)))
        wavfile.write(str(d / "wavs" / ("LJ%03d.wav" % i)), sr, _pcm(200 + i, sr, m, lead=int(rng.integers(500, 4000)) * 2,
                                                                    tail=int(rng.integers(500, 4000)) * 2))
    (d / "transcript.csv").write_text("\n".join(lines) + "\n", encoding="utf-8")
    return str(d)


def _train(num, P, batches, logdir):
    eng = Engine(0)
    eng.load_params(P)
    gs = trainer.train(num, eng, batches, num_iterations=19, logdir=logdir, global_step=0, save_every=10 ** 9, log=lambda *_: None)
    eng.close()
    return gs


def test_training_and_prepo_from_a_44k_corpus(engine, tmp_path):
    from dc_tts_b200.engine import set_engine
    set_engine(engine)
    d = _corpus_44k(tmp_path)
    fpaths, lens, texts = trainer.load_train_data(d)
    kw = dict(B=4, seed=0)
    P = init_params(1)
    for num in (1, 2):
        assert _train(num, P, trainer.bucketed_batches(fpaths, lens, texts, prepro=False, resample=True, **kw), str(tmp_path / ("w%d" % num))) == 20
    out = tmp_path / "prep"
    assert prepo_mod.prepo(d, str(out / "batched"), batch_size=4, engine=engine, resample=True) == len(fpaths)
    prepo_mod.prepo(d, str(out / "single"), load_spectrograms=lambda p: utils.load_spectrograms(p, resample=True))
    for sub in ("mels", "mags"):
        names = sorted(os.listdir(out / "single" / sub))
        assert names == sorted(os.listdir(out / "batched" / sub)) and len(names) == len(fpaths)
        for nm in names:
            assert (out / "single" / sub / nm).read_bytes() == (out / "batched" / sub / nm).read_bytes(), (sub, nm)
    loader = lambda p: trainer._load_spectrograms_npy(p, str(out / "batched" / "mels"), str(out / "batched" / "mags"))
    npy = list(trainer.bucketed_batches(fpaths, lens, texts, epochs=1, loader=loader, **kw))
    wav = list(trainer.bucketed_batches(fpaths, lens, texts, epochs=1, prepro=False, engine=engine, resample=True, **kw))
    assert len(npy) == len(wav) >= 2
    for (L0, m0, g0, n0, _), (L1, m1, g1, n1, _) in zip(npy, wav):
        assert n0 == n1 and np.array_equal(L0, L1)
        assert torch.equal(torch.from_numpy(m0), m1.cpu()) and torch.equal(torch.from_numpy(g0), g1.cpu())


def test_load_spectrograms_resamples_a_16k_file_on_request(engine, tmp_path):
    """utils.load_spectrograms on a file at hp.sr against the oracle; the same samples written at 16 kHz are refused by
    default and, with resample=True, resampled first as librosa.load(fpath, sr=hp.sr) does."""
    from scipy.io import wavfile
    from dc_tts_b200.engine import set_engine
    set_engine(engine)
    rng = np.random.default_rng(3)
    t = np.arange(int(hp.sr * 1.5)) / hp.sr
    y = 0.3 * np.sin(2 * np.pi * 180 * t) * (0.5 + 0.5 * np.sin(2 * np.pi * 3 * t)) + 0.05 * rng.standard_normal(t.size)
    y[:3000] *= 1e-5
    pcm = np.round(np.clip(y, -1, 1) * 32767).astype(np.int16)
    path = str(tmp_path / "LJ001-0001.wav")
    wavfile.write(path, hp.sr, pcm)
    fname, mel, mag = utils.load_spectrograms(path)
    m_o, g_o = rf.load_spectrograms(pcm.astype(np.float32) / 32768.0)
    assert fname == "LJ001-0001.wav" and mel.shape == m_o.shape and mag.shape == g_o.shape
    assert np.abs(mag - g_o)[g_o > 0.35].max() < 1e-4 and np.abs(mel - m_o)[m_o > 0.35].max() < 1e-4
    wavfile.write(path, 16000, pcm)
    with pytest.raises(ValueError, match="sample rate 16000"):
        utils.load_spectrograms(path)
    _, mel16, mag16 = utils.load_spectrograms(path, resample=True)
    m_o, g_o = rf.load_spectrograms(rr.load(pcm, 16000, hp.sr))
    assert mel16.shape == m_o.shape and np.abs(mel16 - m_o)[m_o > 0.35].max() < 1e-4
    assert np.abs(mag16 - g_o)[g_o > 0.35].max() < 1e-4
