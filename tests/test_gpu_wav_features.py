"""Batched feature extraction (`dctts_load_spectrograms_batch`, Engine.load_spectrograms_batch) and training straight from
the wav files (trainer.bucketed_batches(..., prepro=False), data_load.py:104-113) on the GPU."""
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
from oracle import ref_vocoder as rv

pytestmark = pytest.mark.gpu
F = 1 + hp.n_fft // 2


def _speechlike(seed, n, lead, tail, quiet=1e-5):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / hp.sr
    f0 = 150 + 100 * rng.random()
    y = 0.3 * np.sin(2 * np.pi * f0 * t) * (0.5 + 0.5 * np.sin(2 * np.pi * 3 * t)) + 0.05 * rng.standard_normal(n)
    y[:lead] *= quiet
    if tail:
        y[n - tail:] *= quiet
    return np.clip(y, -1, 1).astype(np.float32)


def _frames(y):
    s, e = rv.trim_indices(y)
    return 1 + (e - s) // hp.hop_length


def _with_frames(seed, seconds, want_multiple):
    """A clip whose trimmed frame count is (or is not) a multiple of r, found by moving the silent tail."""
    n = int(hp.sr * seconds)
    for j in range(16):
        y = _speechlike(seed, n, 3000, 2000 + 512 * j)
        if (_frames(y) % hp.r == 0) == want_multiple:
            return y
    raise AssertionError("no tail length gives the wanted frame count")


@pytest.fixture(scope="module")
def pool():
    """Float32 clips: ~600 samples (shorter than n_fft / 2: reflect padding clamps), 0.7 s, 2 s, 5.3 s, 10 s with silent
    lead and tail, then 27 more of 0.3-10 s."""
    ys = [_speechlike(0, 600, 0, 0),
          _with_frames(1, 0.7, False),
          _with_frames(2, 2.0, True),
          _with_frames(3, 5.3, False),
          _speechlike(4, int(10 * hp.sr), 4000, 6000)]
    rng = np.random.default_rng(9)
    for i in range(27):
        n = int(hp.sr * rng.uniform(0.3, 10.0))
        ys.append(_speechlike(10 + i, n, int(rng.integers(0, 6000)), int(rng.integers(0, 6000))))
    fr = [_frames(y) % hp.r for y in ys[1:4]]
    assert 0 in fr and any(f != 0 for f in fr)
    return ys


def _as(y, kind):
    return np.round(y * 32767).astype(np.int16) if kind == "int16" else y


def _single(engine, w):
    """What `utils.load_spectrograms` gives for one utterance (int16 as utils._load_wav converts it), plus the trim."""
    y = w.astype(np.float32) / 32768.0 if w.dtype == np.int16 else w
    _, mel, mag = utils.load_spectrograms(y)
    _, _, trim = engine.get_spectrograms(y)
    return mel, mag, trim


@pytest.mark.parametrize("kind", ["int16", "float32"])
@pytest.mark.parametrize("B", [1, 5, 32])
def test_ragged_batch_is_bitwise_the_single_call(engine, pool, B, kind):
    wavs = [_as(y, kind) for y in (pool[4:5] if B == 1 else pool[:B])]
    mels, mags, t, trim = engine.load_spectrograms_batch(wavs)
    assert mels.is_cuda and mels.is_contiguous() and mags.is_contiguous()
    T_b = int(t.max())
    assert tuple(mels.shape) == (B, T_b, hp.n_mels) and tuple(mags.shape) == (B, hp.r * T_b, F)
    mels, mags = mels.cpu().numpy(), mags.cpu().numpy()
    for b, w in enumerate(wavs):
        mel, mag, tr = _single(engine, w)
        assert t[b] == mel.shape[0] and mag.shape[0] == hp.r * t[b] and tuple(trim[b]) == tr
        assert np.array_equal(mels[b, :t[b]], mel) and np.array_equal(mags[b, :hp.r * t[b]], mag), b
        assert not mels[b, t[b]:].any() and not mags[b, hp.r * t[b]:].any()


def test_batch_against_the_oracle(engine, pool):
    ys = pool[:5]
    mels, mags, t, trim = engine.load_spectrograms_batch(ys)
    mels, mags = mels.cpu().numpy(), mags.cpu().numpy()
    lin = lambda z: 10.0 ** ((z * hp.max_db - hp.max_db + hp.ref_db) / 20.0)
    for b, y in enumerate(ys):
        mel_o, mag_o = rf.load_spectrograms(y)
        assert tuple(trim[b]) == rv.trim_indices(y) and mel_o.shape[0] == t[b]
        mel, mag = mels[b, :t[b]], mags[b, :hp.r * t[b]]
        np.testing.assert_allclose(lin(mag), lin(mag_o), atol=2e-6 * lin(mag_o).max(), rtol=2e-3)
        np.testing.assert_allclose(lin(mel), lin(mel_o), atol=2e-6 * lin(mel_o).max(), rtol=2e-3)
        assert np.abs(mag - mag_o)[mag_o > 0.35].max() < 1e-4
        assert np.abs(mel - mel_o)[mel_o > 0.35].max() < 1e-4


def test_launches_do_not_depend_on_the_batch(engine, pool):
    n0 = engine.launch_count()
    engine.load_spectrograms_batch(pool[:1])
    n1 = engine.launch_count()
    engine.load_spectrograms_batch(pool[:32])
    n32 = engine.launch_count()
    assert n1 - n0 == n32 - n1 == 2


def _raw_call(engine, wavs, t_capacity):
    """The C-ABI call on output buffers pre-filled with 7: returns (rc, error text, mel, mag)."""
    lib = engine._lib
    offsets = np.zeros(len(wavs) + 1, np.int64)
    offsets[1:] = np.cumsum([w.size for w in wavs])
    wav = torch.from_numpy(np.concatenate(wavs)).to(engine.device)
    mel = torch.full((len(wavs) * t_capacity * hp.n_mels,), 7.0, device=engine.device)
    mag = torch.full((len(wavs) * t_capacity * hp.r * F,), 7.0, device=engine.device)
    t = np.zeros(len(wavs), np.int32)
    trim = np.zeros(2 * len(wavs), np.int32)
    T_b = C.c_int32(0)
    p32 = C.POINTER(C.c_int32)
    torch.cuda.synchronize()
    rc = lib.dctts_load_spectrograms_batch(engine._h, C.c_void_p(wav.data_ptr()), 1, offsets.ctypes.data_as(C.POINTER(C.c_int64)),
                                           len(wavs), hp.sr, C.c_void_p(mel.data_ptr()), C.c_void_p(mag.data_ptr()), t_capacity,
                                           t.ctypes.data_as(p32), trim.ctypes.data_as(p32), C.byref(T_b), None)
    torch.cuda.synchronize()
    return rc, lib.dctts_last_error(engine._h).decode(), mel, mag


def test_error_paths_name_the_utterance_and_write_nothing(engine, pool):
    wavs = [_as(y, "int16") for y in pool[:5]]
    # an utterance with nothing left to frame (a single sample) fails the call, naming its index
    rc, err, mel, mag = _raw_call(engine, wavs[:2] + [np.zeros(1, np.int16)] + wavs[2:], 800)
    assert rc != 0 and "utterance 2" in err
    assert bool((mel == 7).all()) and bool((mag == 7).all())
    with pytest.raises(DcttsError, match="utterance 2"):
        engine.load_spectrograms_batch(wavs[:2] + [np.zeros(1, np.int16)])
    # outputs too small for the longest member (the 10 s clip, index 4)
    _, _, t, _ = engine.load_spectrograms_batch(wavs)
    rc, err, mel, mag = _raw_call(engine, wavs, int(t.max()) - 1)
    assert rc != 0 and "utterance 4" in err and "t_capacity" in err
    assert bool((mel == 7).all()) and bool((mag == 7).all())
    with pytest.raises(DcttsError, match="t_capacity"):
        engine.load_spectrograms_batch(wavs, t_capacity=int(t.max()) - 1)
    # the handle stays usable
    mels, _, t2, _ = engine.load_spectrograms_batch(wavs)
    assert np.array_equal(t2, t) and mels.shape[1] == t.max()


def test_all_zero_utterance_is_kept_like_the_single_call(engine, pool):
    """librosa.effects.trim keeps every frame of an all-zero signal (each is 0 dB below the loudest), so a silent
    utterance yields the clip floor, exactly as the single-utterance call does."""
    z = np.zeros(5000, np.int16)
    mels, mags, t, trim = engine.load_spectrograms_batch([_as(pool[1], "int16"), z])
    mel, mag, tr = _single(engine, z)
    assert tuple(trim[1]) == tr == (0, 5000)
    assert np.array_equal(mels[1, :t[1]].cpu().numpy(), mel) and np.array_equal(mags[1, :hp.r * t[1]].cpu().numpy(), mag)


# ------------------------------------------------------------------------------------------- training from wavs
def _wav_corpus(root, n=24, seed=0):
    """LJ-shaped corpus of int16 wavs with transcripts; LJ007 is 11 s of sound, over capacity after trimming."""
    from scipy.io import wavfile
    rng = np.random.default_rng(seed)
    d = root / "LJSpeech-1.0"
    (d / "wavs").mkdir(parents=True)
    lines = []
    for i in range(n):
        nchar = int(rng.integers(10, 120))
        lines.append("LJ%03d|raw|%s" % (i, "".join(rng.choice(list("abcdefghijklmnopqrstuvwxyz '"), nchar))))
        seconds = 11.0 if i == 7 else float(rng.uniform(0.5, 3.0))
        y = _speechlike(100 + i, int(seconds * hp.sr), int(rng.integers(500, 4000)), int(rng.integers(500, 4000)))
        wavfile.write(str(d / "wavs" / ("LJ%03d.wav" % i)), hp.sr, _as(y, "int16"))
    (d / "transcript.csv").write_text("\n".join(lines) + "\n", encoding="utf-8")
    return str(d)


def _run(num, P, batches, logdir):
    eng = Engine(0)
    eng.load_params(P)
    losses, log = [], []
    step = eng.train_step if num == 1 else eng.train_step_ssrn

    def recording(*a, **k):
        out = step(*a, **k)
        losses.append(out["loss"])
        return out
    if num == 1:
        eng.train_step = recording
    else:
        eng.train_step_ssrn = recording
    gs = trainer.train(num, eng, batches, num_iterations=19, logdir=logdir, global_step=0, save_every=10 ** 9, log=log.append)
    eng.close()
    return gs, np.array(losses, np.float64), sum(s.startswith("skipped") for s in log)


def test_training_from_wavs_matches_the_npy_route(engine, tmp_path):
    d = _wav_corpus(tmp_path)
    fpaths, lens, texts = trainer.load_train_data(d)
    out = tmp_path / "prep"
    kw = dict(B=4, seed=0)
    wav_epoch = list(trainer.bucketed_batches(fpaths, lens, texts, epochs=1, prepro=False, engine=engine, **kw))
    assert not (out / "mels").exists()
    P = init_params(1)
    wav_runs = {num: _run(num, P, trainer.bucketed_batches(fpaths, lens, texts, prepro=False, **kw), str(tmp_path / ("w%d" % num)))
                for num in (1, 2)}
    assert prepo_mod.prepo(d, str(out), engine=engine) == len(fpaths)
    loader = lambda p: trainer._load_spectrograms_npy(p, str(out / "mels"), str(out / "mags"))
    npy_epoch = list(trainer.bucketed_batches(fpaths, lens, texts, epochs=1, loader=loader, **kw))
    assert len(npy_epoch) == len(wav_epoch) > 2
    for (L0, m0, g0, n0, k0), (L1, m1, g1, n1, k1) in zip(npy_epoch, wav_epoch):
        assert n0 == n1 and k0 == k1 and np.array_equal(L0, L1) and m1.is_cuda and g1.is_cuda
        assert torch.equal(torch.from_numpy(m0), m1.cpu()) and torch.equal(torch.from_numpy(g0), g1.cpu())
    for num in (1, 2):
        gs_w, loss_w, skip_w = wav_runs[num]
        gs_n, loss_n, skip_n = _run(num, P, trainer.bucketed_batches(fpaths, lens, texts, loader=loader, **kw), str(tmp_path / ("n%d" % num)))
        assert gs_w == gs_n == 20 and len(loss_w) == len(loss_n) == 20
        assert skip_w == skip_n >= 1
        np.testing.assert_allclose(loss_w[:3], loss_n[:3], rtol=1e-4)
        np.testing.assert_allclose(loss_w, loss_n, rtol=5e-3)


def test_batched_prepo_writes_the_per_file_bytes(engine, tmp_path):
    from dc_tts_b200.engine import set_engine
    set_engine(engine)
    d = _wav_corpus(tmp_path, n=11, seed=3)
    prepo_mod.prepo(d, str(tmp_path / "batched"), batch_size=4, engine=engine)
    prepo_mod.prepo(d, str(tmp_path / "single"), load_spectrograms=utils.load_spectrograms)
    for sub in ("mels", "mags"):
        names = sorted(os.listdir(tmp_path / "single" / sub))
        assert names == sorted(os.listdir(tmp_path / "batched" / sub)) and len(names) == 11
        for nm in names:
            assert (tmp_path / "single" / sub / nm).read_bytes() == (tmp_path / "batched" / sub / nm).read_bytes(), (sub, nm)
