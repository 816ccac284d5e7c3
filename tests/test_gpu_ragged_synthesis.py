"""SSRN with a length per utterance (Engine.ssrn(lengths=...), include/dctts.h: dctts_ssrn_ragged) and the synthesis
entry point that ends each utterance at its text (synthesize(until_eos=True)).

Per utterance, rows below 4 x its length must be those of SSRN on that utterance alone at its own length, bit for bit,
on the same kernel set, and the rows past them exactly 0.  Mel rows past a length hold NaN, then 1e4: they must never
be read, nor enter the per-utterance input scale.  The lengths sit at the 128-row tile edges of the three time levels
(L, 2L, 4L) and at both ends of the range."""
import os

import numpy as np
import pytest
import torch

from dc_tts_b200.engine import DcttsError
from dc_tts_b200.hyperparams import Hyperparams as hp
from dc_tts_b200.params import init_params

from sample_rates import at_rate

pytestmark = pytest.mark.gpu

T = hp.max_T
LENS = [1, 2, 3, 31, 32, 33, 127, 128, 129, 209, 210, 64, 17, 100]
SENTINEL = -123.25


@pytest.fixture(scope="module")
def eng():
    from dc_tts_b200.engine import Engine
    e = Engine(0)
    e.load_params(init_params(0, "perturbed"))
    yield e
    e.close()


@pytest.fixture(scope="module")
def mels():
    return torch.from_numpy(np.random.default_rng(11).uniform(0, 1, (40, T, hp.n_mels)).astype(np.float32))


_SINGLE = {}


def _single(e, path, Y, b, n):
    """SSRN of utterance b alone at its own length (cached per engine and kernel set; the key holds the engine itself, as
    an engine built after another was closed may get its id)."""
    key = (e, path, b, n)
    if key not in _SINGLE:
        lg, Z = e.ssrn(Y[b:b + 1, :n])
        _SINGLE[key] = (lg[0].cpu(), Z[0].cpu())
    return _SINGLE[key]


def _ragged(e, Y, n, fill):
    """Engine.ssrn with lengths n; the mel rows past each length hold `fill`, the outputs start as a sentinel."""
    Yr = Y.clone()
    for b, k in enumerate(n):
        Yr[b, k:] = fill
    B = len(n)
    Z = torch.full((B, hp.r * Y.shape[1], e.F), SENTINEL, device=e.device)
    lg, Z = e.ssrn(Yr, out=Z, lengths=torch.as_tensor(n, dtype=torch.int32, device=e.device))
    return lg.cpu(), Z.cpu()


def _check(e, path, Y, n, lg, Z):
    for b, k in enumerate(n):
        lg1, Z1 = _single(e, path, Y, b, k)
        assert torch.equal(Z[b, :hp.r * k], Z1), (path, b, k)
        assert torch.equal(lg[b, :hp.r * k], lg1), (path, b, k)
        assert not Z[b, hp.r * k:].any() and not lg[b, hp.r * k:].any(), (path, b, k)


@pytest.mark.parametrize("path", [1, 0], ids=["tensorpath", "fp32path"])
@pytest.mark.parametrize("B", [1, 3, 32, 40])
def test_ssrn_ragged_equals_each_utterance_alone(eng, mels, path, B):
    eng.set_tensor_path(path)
    try:
        n = [LENS[(b * 5 + B) % len(LENS)] for b in range(B)]
        Y = mels[:B].to(eng.device)
        for fill in (float("nan"), 1e4):
            lg, Z = _ragged(eng, Y, n, fill)
            _check(eng, path, Y, n, lg, Z)
        # every utterance at full length.  On the wgmma path that is the batch call itself.  The fp32 path's GEMM
        # schedule follows the launch's row count, so there a batch call differs from its utterances' own calls in the
        # last bits and the ragged call keeps to the latter.
        lg, Z = _ragged(eng, Y, [T] * B, 0.0)
        if path == 1 or B == 1:
            lg0, Z0 = eng.ssrn(Y)
            assert torch.equal(Z, Z0.cpu()) and torch.equal(lg, lg0.cpu())
        else:
            _check(eng, path, Y, [T] * B, lg, Z)
    finally:
        eng.set_tensor_path(1)


@pytest.mark.parametrize("path", [1, 0], ids=["tensorpath", "fp32path"])
def test_ssrn_ragged_at_a_shorter_call_length(eng, mels, path):
    """T below max_T (the batch's longest length, as synthesize(until_eos=True) calls it), without logits."""
    eng.set_tensor_path(path)
    try:
        n = [40, 7, 64, 1]
        Y = mels[:4, :64].to(eng.device)
        Yr = Y.clone()
        for b, k in enumerate(n):
            Yr[b, k:] = float("nan")
        lg, Z = eng.ssrn(Yr, want_logits=False, lengths=n)
        assert lg is None and tuple(Z.shape) == (4, 256, eng.F)
        for b, k in enumerate(n):
            assert torch.equal(Z[b, :4 * k].cpu(), eng.ssrn(Y[b:b + 1, :k])[1][0].cpu()), (path, b, k)
            assert not Z[b, 4 * k:].any()
    finally:
        eng.set_tensor_path(1)


@pytest.mark.parametrize("sr", [16000, 44100], ids=["F513", "F2049"])
@pytest.mark.parametrize("path", [1, 0], ids=["tensorpath", "fp32path"])
def test_ssrn_ragged_other_widths(sr, path):
    from dc_tts_b200.engine import Engine
    with at_rate(sr) as H:
        e = Engine(0, hparams=H)
        try:
            e.load_params(init_params(0, "perturbed"))
            e.set_tensor_path(path)
            n = [129, 1, 33]
            Y = torch.from_numpy(np.random.default_rng(sr).uniform(0, 1, (3, T, hp.n_mels)).astype(np.float32)).to(e.device)
            lg, Z = _ragged(e, Y, n, float("nan"))
            _check(e, path, Y, n, lg, Z)
        finally:
            e.close()


@pytest.mark.parametrize("path", [1, 0], ids=["tensorpath", "fp32path"])
def test_ssrn_ragged_refuses_lengths_outside_the_range(eng, mels, path):
    eng.set_tensor_path(path)
    try:
        Y = mels[:3].to(eng.device)
        for bad in ([5, 0, 7], [5, 7, T + 1]):
            with pytest.raises(DcttsError, match="utterance %d" % (1 if bad[1] == 0 else 2)):
                eng.ssrn(Y, lengths=bad)
        with pytest.raises(DcttsError, match="3 lengths for 2"):
            eng.ssrn(Y[:2], lengths=[1, 2, 3])
    finally:
        eng.set_tensor_path(1)


def test_ssrn_ragged_fp32_entry_point_refuses_without_writing(eng, mels):
    """The fp32 path reads the lengths back: a length outside [1, T] fails the call before any launch."""
    from dc_tts_b200.engine import _ptr
    eng.set_tensor_path(0)
    try:
        Y = mels[:2].to(eng.device)
        n = torch.tensor([4, T + 1], dtype=torch.int32, device=eng.device)
        Z = torch.full((2, hp.r * T, eng.F), SENTINEL, device=eng.device)
        rc = eng._lib.dctts_ssrn_ragged(eng._h, _ptr(Y), 2, T, _ptr(n), _ptr(None), _ptr(Z), eng._stream())
        assert rc != 0 and b"utterance 1" in eng._lib.dctts_last_error(eng._h)
        assert bool((Z == SENTINEL).all())
    finally:
        eng.set_tensor_path(1)


def test_synthesize_until_eos_writes_each_utterance_to_its_end(tmp_path, monkeypatch):
    """synthesize(until_eos=True) with seeded weights: every wav is the utterance-by-utterance chain
    spectrogram2wav(SSRN(Y_b[:len_b])) trimmed, bit for bit."""
    from scipy.io.wavfile import read as read_wav
    from dc_tts_b200 import engine as engine_mod
    from dc_tts_b200.engine import Engine
    from dc_tts_b200.synthesize import synthesize
    from dc_tts_b200.train import Graph
    from dc_tts_b200.utils import spectrogram2wav

    texts = ["a cat", "the dog ran", "hello", "a short one", "it is"]
    sent = tmp_path / "sentences.txt"
    sent.write_text("header\n" + "".join("%d. %s\n" % (i + 1, t) for i, t in enumerate(texts)))
    out = tmp_path / "samples"
    monkeypatch.setattr(hp, "sampledir", str(out))
    prev = engine_mod._default
    e = Engine(0)
    engine_mod.set_engine(e)
    try:
        Y, Z = synthesize(params=init_params(0), sentences=str(sent), write=True, until_eos=True)
        from dc_tts_b200.data_load import load_data
        Yd, _, n = Graph(mode="synthesize").generate_until_eos(load_data("synthesize", str(sent)))
        n = n.cpu().numpy()
        assert (n < T).any(), n
        assert np.array_equal(Y, Yd.cpu().numpy())
        for b, k in enumerate(n):
            assert not Y[b, k:].any() and not Z[b, hp.r * k:].any()
            _, Zb = e.ssrn(Yd[b:b + 1, :k])
            assert np.array_equal(Z[b, :hp.r * k], Zb[0].cpu().numpy()), b
            sr, wav = read_wav(os.path.join(str(out), "%d.wav" % (b + 1)))
            assert sr == hp.sr and wav.dtype == np.float32
            assert np.array_equal(wav, spectrogram2wav(Zb[0].cpu().numpy())), b
    finally:
        engine_mod.set_engine(prev)
        e.close()


# ---------------------------------------------------------------------------------------- Griffin-Lim
def _chunk_edges(hop, T_max, chunk=512):
    """Frame counts whose hop (T_b - 1) samples lie just past and just short of a multiple of the de-emphasis chunk."""
    ms = range(2, T_max)
    past = min(ms, key=lambda m: (hop * (m - 1)) % chunk)
    short = max(ms, key=lambda m: (hop * (m - 1)) % chunk)
    return [past, short]


_VSINGLE = {}


def _voc_single(e, mags, b, k, n_iter):
    key = (e, b, k, n_iter)                 # the engine itself, as for _single
    if key not in _VSINGLE:
        wav, trim = e.spectrogram2wav(mags[b:b + 1, :k], n_iter=n_iter)
        _VSINGLE[key] = (wav[0].cpu(), trim[0].copy())
    return _VSINGLE[key]


def _voc_check(e, mags, n, n_iter):
    """The ragged call (mag rows past each count NaN) against each utterance's own call."""
    B, T = len(n), mags.shape[1]
    m = mags[:B].clone()
    for b, k in enumerate(n):
        m[b, k:] = float("nan")
    wav, trim = e.spectrogram2wav(m, n_iter=n_iter, lengths=n)
    wav = wav.cpu()
    assert tuple(wav.shape) == (B, e.hp.hop_length * (T - 1))
    for b, k in enumerate(n):
        w1, t1 = _voc_single(e, mags, b, k, n_iter)
        Ly = e.hp.hop_length * (k - 1)
        assert torch.equal(wav[b, :Ly], w1), (b, k, n_iter)
        assert not wav[b, Ly:].any(), (b, k, n_iter)
        assert np.array_equal(trim[b], t1), (b, k, n_iter, trim[b], t1)


@pytest.fixture(scope="module")
def mags(eng):
    T = hp.r * hp.max_T
    return torch.from_numpy(np.random.default_rng(21).uniform(0, 1, (32, T, eng.F)).astype(np.float32)).to(eng.device)


@pytest.mark.parametrize("n_iter", [0, 1, -1], ids=["iter0", "iter1", "default"])
@pytest.mark.parametrize("B", [1, 3, 32])
def test_vocoder_ragged_equals_each_utterance_alone(eng, mags, B, n_iter):
    T = mags.shape[1]
    counts = [2, 3, 4, 5, 60, T] + _chunk_edges(hp.hop_length, T)
    n = [counts[(b + B) % len(counts)] for b in range(B)]
    if B == 3:
        n = [counts[-2], 2, counts[-1]]
    _voc_check(eng, mags, n, n_iter)


def test_vocoder_ragged_at_a_shorter_call_length(eng, mags):
    """T below r max_T (the batch's longest count, as synthesize(until_eos=True) calls it)."""
    _voc_check(eng, mags[:, :100], [100, 37, 2, 64], -1)


@pytest.mark.parametrize("sr", [16000, 44100], ids=["F513", "F2049"])
def test_vocoder_ragged_other_widths(sr):
    from dc_tts_b200.engine import Engine
    with at_rate(sr) as H:
        e = Engine(0, hparams=H)
        try:
            m = torch.from_numpy(np.random.default_rng(sr).uniform(0, 1, (3, 240, e.F)).astype(np.float32)).to(e.device)
            _voc_check(e, m, [240, 2] + _chunk_edges(H.hop_length, 240)[:1], 3)
        finally:
            e.close()


def test_vocoder_ragged_refuses_counts_outside_the_range(eng, mags):
    from dc_tts_b200.engine import _ptr
    m = mags[:3, :50].contiguous()
    for bad, who in (([5, 1, 7], 1), ([5, 7, 51], 2)):
        with pytest.raises(DcttsError, match="utterance %d" % who):
            eng.spectrogram2wav(m, lengths=bad)
    with pytest.raises(DcttsError, match="2 lengths for 3"):
        eng.spectrogram2wav(m, lengths=[4, 5])
    wav = torch.full((3, hp.hop_length * 49), SENTINEL, device=eng.device)
    n = np.array([5, 0, 7], np.int32)
    trim = np.full((3, 2), -7, np.int32)
    import ctypes as C
    rc = eng._lib.dctts_spectrogram2wav_ragged(eng._h, _ptr(m), 3, 50, n.ctypes.data_as(C.c_void_p), -1, _ptr(wav),
                                               trim.ctypes.data_as(C.c_void_p), eng._stream())
    assert rc != 0 and b"utterance 1" in eng._lib.dctts_last_error(eng._h)
    torch.cuda.synchronize()
    assert bool((wav == SENTINEL).all()) and bool((trim == -7).all())
