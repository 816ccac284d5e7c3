"""Streaming synthesis from text on the GPU (dctts_synth_stream_*, Engine.synthesis_stream).

  * Decode: the stream's Y and lengths equal text2mel_generate_until's bit for bit (B = 1, 5, 7, 32; tail 0 and 3; a mix
    of stop positions), and the library's halos equal the CPU ones (tests/ref_synth_stream.py).
  * SSRN: the committed magnitudes equal ssrn(Y, lengths) bit for bit, on inputs whose Y abs-max lies in [0.5, 1) (the
    windows' fixed input scale); the windowed SSRN on quiet inputs (Y x 1e-3) matches the float64 oracle within the
    SSRN tests' tolerance, at n_fft 1024, 2048 and 4096.
  * Timing independence: a stream polled as fast as it goes and one polled only after its decode ended give the same
    samples, lengths and trims.
  * Offline replay: ssrn(Y, lengths) pushed to Engine.vocoder_stream on the same grid gives the stream's samples bit for
    bit, plain and with momentum 0.99; with chunk >= max_T the samples and trims are spectrogram2wav's.
  * Streaming happens: a full-length utterance's first chunk is pushed before its decode has ended.
  * The frames a poll reports as published never decrease, and end at or past each utterance's length.
  * The measurement switches: decode_group changes no output, decode_timing reports the decode's GPU time.
  * Refusals (TextEnc, the generations, workspace growth and training while a stream is open; a handle whose decode
    packing is stale after training), and an engine closed while a stream is open."""
import numpy as np
import pytest
import torch

import ref_synth_stream as rs
from dc_tts_b200.engine import DcttsError
from dc_tts_b200.hyperparams import Hyperparams as hp
from dc_tts_b200.params import init_params, synthetic_text
from oracle import ref_numpy as rn
from sample_rates import at_rate

pytestmark = pytest.mark.gpu
NET_TOL = 1e-3                 # tests/test_gpu_ssrn_sizes.py
TARGETS = [1, 40, 120, None, 210, 7, 90]


@pytest.fixture
def eng(engine):
    engine.set_tensor_path(1)
    if not engine.get_option("decode_available"):
        pytest.skip("no persistent decode on this device")
    return engine


def _texts(B, seed=0):
    return np.concatenate([synthetic_text(1, 20 + (37 * i) % 150, seed=seed + i) for i in range(B)])


def _stops(eng, L):
    """A mix of stop positions from a full-length run's windows: ends near the TARGETS frames, and never (-1)."""
    _, P, _, _ = eng.text2mel_generate(L)
    P = P.cpu().numpy()
    return np.array([-1 if t is None else int(P[b, min(t, hp.max_T - 1)]) for b, t in
                     zip(range(len(L)), TARGETS * len(L))], np.int64)


def _run(eng, L, sp, tail, chunk, momentum=0.0, late=False):
    """Opens a stream, polls it (right away, or after its decode ended) -> (per-utterance samples, lengths, trims, Y, Z,
    first frames)."""
    ss = eng.synthesis_stream(L, stop_pos=sp, tail=tail, chunk=chunk, momentum=momentum)
    if late:
        torch.cuda.synchronize()
    pieces = [[] for _ in range(len(L))]
    for out in ss:
        for b, w in enumerate(out):
            pieces[b].append(w)
    n, trim, Y, Z = ss.close(outputs=True)
    return [np.concatenate(p) for p in pieces], n, trim, Y, Z, ss.first_frames


def _replay(eng, Z, n, chunk, momentum):
    """ssrn's rows pushed to one vocoder stream per utterance on the stream's grid -> samples per utterance, trims."""
    wavs, trims = [], []
    for b in range(len(n)):
        vs = eng.vocoder_stream(1, n_iter=-1, momentum=momentum)
        got = []
        for a, e, _, _, fin in rs.chunks(int(n[b]), chunk, 0, 0):
            got += vs.push(Z[b:b + 1, 4 * a:4 * e], [4 * (e - a)], fin)
        wavs.append(np.concatenate(got))
        trims.append(vs.close()[0])
    return wavs, np.array(trims)


def test_halo(eng):
    assert eng.ssrn_halo() == rs.halo()


@pytest.mark.parametrize("tail", [0, 3])
@pytest.mark.parametrize("B", [1, 5, 7, 32])
def test_stream_matches_the_one_shot_chain(eng, B, tail):
    L = _texts(B, seed=10 * B + tail)
    sp = _stops(eng, L)
    chunk = 16
    wav, n, trim, Y, Z, _ = _run(eng, L, sp, tail, chunk)
    Yu, _, nu = eng.text2mel_generate_until(L, stop_pos=sp, tail=tail)
    assert np.array_equal(n, nu.cpu().numpy())
    assert torch.equal(Y, Yu)
    amax = np.array([Y[b, :n[b]].abs().max().item() for b in range(B)])
    assert ((amax >= 0.5) & (amax < 1)).all(), amax
    _, Zr = eng.ssrn(Y, lengths=n)
    assert torch.equal(Z, Zr)
    # the same texts polled only after the decode ended: identical samples, lengths and trims
    wav2, n2, trim2, _, _, _ = _run(eng, L, sp, tail, chunk, late=True)
    assert np.array_equal(n2, n) and np.array_equal(trim2, trim)
    assert all(np.array_equal(a, b) for a, b in zip(wav, wav2))
    # offline replay of ssrn(Y, lengths) on the same grid
    rw, rt = _replay(eng, Zr, n, chunk, 0.0)
    assert all(np.array_equal(a, b) for a, b in zip(wav, rw))
    assert np.array_equal(rt, trim)
    assert all(w.size == hp.hop_length * (4 * int(k) - 1) for w, k in zip(wav, n))


def test_momentum_replay(eng):
    L = _texts(5, seed=77)
    sp = _stops(eng, L)
    wav, n, trim, _, Z, _ = _run(eng, L, sp, 0, 7, momentum=0.99)
    rw, rt = _replay(eng, Z, n, 7, 0.99)
    assert all(np.array_equal(a, b) for a, b in zip(wav, rw))
    assert np.array_equal(rt, trim)


def test_whole_utterance_chunk(eng):
    L = _texts(5, seed=91)
    sp = _stops(eng, L)
    wav, n, trim, Y, Z, _ = _run(eng, L, sp, 3, hp.max_T)
    _, Zr = eng.ssrn(Y, lengths=n)
    w, t = eng.spectrogram2wav(Zr, lengths=4 * n)
    w = w.cpu().numpy()
    for b in range(5):
        assert np.array_equal(wav[b], w[b, :hp.hop_length * (4 * int(n[b]) - 1)]), b
    assert np.array_equal(trim, t)


def test_streaming_happens(eng):
    L = _texts(1, seed=5)
    _, n, _, _, _, first = _run(eng, L, [-1], 0, 16)
    assert n[0] == hp.max_T
    print("first push at %d published frames" % first[0])
    assert 0 < first[0] < hp.max_T


def test_quiet_windows_match_the_float64_oracle(eng, params):
    rng = np.random.default_rng(3)
    T, n = 60, [60, 33]
    Y = (rng.uniform(0, 1, (2, T, hp.n_mels)) * 1e-3).astype(np.float32)
    Z = eng.ssrn_windows(Y, [0, 20], [60, 13], n).cpu().numpy()
    for b, (a, c) in enumerate(((0, 60), (20, 13))):
        ref = rn.SSRN(params, Y[b:b + 1, :n[b]].astype(np.float64))[1][0, 4 * a:4 * (a + c)]
        assert np.abs(Z[b, :4 * c] - ref).max() <= NET_TOL


@pytest.mark.parametrize("n_fft,sr", [(1024, 16000), (4096, 44100)])
def test_windows_at_other_rates(n_fft, sr):
    from dc_tts_b200.engine import Engine
    with at_rate(sr, n_fft) as H:
        P = init_params(0, "perturbed")
        e = Engine(0, hparams=H)
        try:
            e.load_params(P)
            Y = np.random.default_rng(4).uniform(0, 0.99, (1, 40, H.n_mels)).astype(np.float32)
            Z = e.ssrn_windows(Y, [16], [8], [40]).cpu().numpy()
            _, Zw = e.ssrn(Y, lengths=[40])
            assert Z.shape == (1, 32, 1 + n_fft // 2)
            assert np.array_equal(Z[0], Zw.cpu().numpy()[0, 64:96])
        finally:
            e.close()


def test_refusals(eng):
    L = _texts(2, seed=1)
    with pytest.raises(DcttsError, match="chunk must be >= 1"):
        eng.synthesis_stream(L, chunk=0)
    ss = eng.synthesis_stream(L, stop_pos=[-1, 5], chunk=32)
    try:
        with pytest.raises(DcttsError, match="already open"):
            eng.synthesis_stream(L)
        with pytest.raises(DcttsError, match="synthesis stream is open"):
            eng.text2mel_generate_until(L)
        with pytest.raises(DcttsError, match="synthesis stream is open"):
            eng.text2mel_generate(L)
        with pytest.raises(DcttsError, match="dctts_textenc: a synthesis stream is open"):
            eng.textenc(L)
        with pytest.raises(DcttsError, match="dctts_reserve_frames: a synthesis stream is open"):
            eng._check(eng._lib.dctts_reserve_frames(eng._h, 64, 4000, None), "dctts_reserve_frames")   # far past any growth
        with pytest.raises(DcttsError, match="synthesis stream is open"):
            eng._check(eng._lib.dctts_reserve(eng._h, 64), "dctts_reserve")
        with pytest.raises(DcttsError, match="dctts_train_init: a synthesis stream is open"):
            eng.train_init(1)
    finally:
        n, trim = ss.close()
    assert n[0] == hp.max_T and trim.shape == (2, 2)
    eng.text2mel_generate_until(L)                                # the handle is usable again


def test_refusals_without_decode_or_tensor_path(eng):
    L = _texts(1, seed=2)
    eng.set_option("decode_mode", 0)
    try:
        with pytest.raises(DcttsError, match="persistent decode"):
            eng.synthesis_stream(L)
    finally:
        eng.set_option("decode_mode", 1)
    eng.set_tensor_path(0)
    try:
        with pytest.raises(DcttsError, match="no tensor-core chain"):
            eng.synthesis_stream(L)
    finally:
        eng.set_tensor_path(1)


def test_engine_close_frees_an_open_stream(params):
    from dc_tts_b200.engine import Engine
    e = Engine(0)
    e.load_params(params)
    ss = e.synthesis_stream(_texts(3, seed=4), chunk=8)
    ss.poll()
    e.close()
    with pytest.raises(DcttsError, match="the stream is closed"):
        ss.poll()


def test_published_frames_never_decrease(eng):
    L = _texts(5, seed=33)
    sp = _stops(eng, L)
    ss = eng.synthesis_stream(L, stop_pos=sp, chunk=8)
    seen = [ss.frames.copy()]
    for _ in ss:
        seen.append(ss.frames.copy())
    n, _ = ss.close()
    seen = np.array(seen)
    assert (np.diff(seen, axis=0) >= 0).all()
    assert (seen[-1] >= n).all() and (seen[-1] <= hp.max_T).all()


def test_measurement_switches(eng):
    L = _texts(7, seed=44)
    sp = _stops(eng, L)
    Y0, _, n0 = eng.text2mel_generate_until(L, stop_pos=sp)
    try:
        eng.set_option("decode_timing", 1)
        for G in (1, 2, 5):
            eng.set_option("decode_group", G)
            Y, _, n = eng.text2mel_generate_until(L, stop_pos=sp)
            assert torch.equal(Y, Y0) and torch.equal(n, n0), G
            assert eng.get_option("decode_last_us") > 0
            ss = eng.synthesis_stream(L, stop_pos=sp, chunk=16)
            n2, _, Y2, _ = ss.close(outputs=True)
            assert torch.equal(Y2, Y0) and np.array_equal(n2, n0.cpu().numpy()), G
            assert eng.get_option("decode_last_us") > 0
    finally:
        eng.set_option("decode_group", 0)
        eng.set_option("decode_timing", 0)


def test_refusal_after_training(params):
    """train_init leaves the packed decode stream stale: the stream repeats why and points to refresh_synthesis()."""
    from dc_tts_b200.engine import Engine
    e = Engine(0)
    try:
        e.load_params(params)
        e.train_init(1)
        with pytest.raises(DcttsError, match="has been trained.*refresh_synthesis"):
            e.synthesis_stream(_texts(1, seed=6))
        e.refresh_synthesis()
        n, _ = e.synthesis_stream(_texts(1, seed=6), stop_pos=[3], chunk=16).close()
        assert n[0] >= 1
    finally:
        e.close()
