"""The decode along a caller's attention windows (Engine.text2mel_generate_path) on both decode paths.

Replaying the window history of a free run reproduces that run bit for bit: the path decode is the free decode with
the next window read instead of taken from the argmax, and every other step (the recompute trigger on a window move,
the packed recompute, the stream bound) is the same code.  Arbitrary paths are held to the step-wise loop fed the same
windows (full recompute per frame) and to the CPU oracle."""
import os

import numpy as np
import pytest
import torch

from dc_tts_b200.engine import DcttsError
from dc_tts_b200.hyperparams import Hyperparams as hp
from dc_tts_b200.params import init_params, synthetic_text
from dc_tts_b200.utils import stretch_path

pytestmark = pytest.mark.gpu

T, N, WIN = hp.max_T, hp.max_N, hp.attention_win_size


@pytest.fixture
def path_engine(engine):
    engine.set_tensor_path(1)
    yield engine
    engine.set_option("decode_force_prepass", 0)
    engine.set_option("decode_mode", 1)


def _mode(e, mode):
    if mode == 1 and not e.get_option("decode_available"):
        pytest.skip("no persistent decode on this device")
    e.set_option("decode_mode", mode)


def _texts(B, seed):
    return np.concatenate([synthetic_text(1, 20 + (37 * i) % 150, seed=seed + i) for i in range(B)])


def _cluster_frames(e, n):
    """Frames the persistent path decode executes: per cluster (consecutive utterances in length order), its longest."""
    B, mc = len(n), max(1, e.get_option("decode_max_clusters"))
    G = 1
    while G < 5 and -(-B // G) > mc:
        G += 1
    order = np.argsort(n, kind="stable")
    return sum(int(n[order[c * G:(c + 1) * G]].max()) for c in range(-(-B // G)))


def _check_tail(Y, P, M, n):
    for b, k in enumerate(n):
        assert not Y[b, k:].any() and bool((P[b, k:] == -1).all()) and bool((M[b, k:] == -1).all()), (b, k)


@pytest.mark.parametrize("mode", [1, 0], ids=["persistent", "graph"])
@pytest.mark.parametrize("B", [1, 5, 6, 23, 40])
def test_replay_is_exact(path_engine, B, mode):
    """Free run and until-EOS run fed back as the path: Y and the window history bit-identical, and the argmax history
    is the next frame's window."""
    e = path_engine
    _mode(e, mode)
    L = _texts(B, 300)
    for force in ((0, 1) if mode == 1 else (0,)):
        e.set_option("decode_force_prepass", force)
        Yf, Pf, _, _ = e.text2mel_generate(L)
        Y, P, M = e.text2mel_generate_path(L, Pf)
        assert torch.equal(Y, Yf) and torch.equal(P, Pf), force
        assert torch.equal(M[:, :-1], Pf[:, 1:]), force
        assert e.get_option("decode_last_frames") == (_cluster_frames(e, np.full(B, T)) if mode == 1 else T)

        sp = np.array([int(Pf[b].max()) if b % 3 else int(Pf[b, T // 2]) for b in range(B)])
        Yu, Pu, nu = e.text2mel_generate_until(L, stop_pos=sp, tail=3)
        n = nu.cpu().numpy()
        Y, P, M = e.text2mel_generate_path(L, Pu, nu)
        assert torch.equal(Y, Yu) and torch.equal(P, Pu), force
        for b, k in enumerate(n):
            assert torch.equal(M[b, :k - 1], Pu[b, 1:k]), (force, b, k)
        _check_tail(Y, P, M, n)
        assert e.get_option("decode_last_frames") == (_cluster_frames(e, n) if mode == 1 else T), force


def _arbitrary_paths(Pf, steps):
    """Stretched by 0.7 and 1.5, backward moves and long jumps, and windows at the end of the text."""
    B = Pf.shape[0]
    n0 = np.full(B, steps)
    p07, n07 = stretch_path(Pf[:, :steps], n0, 0.7, steps=steps)
    p15, n15 = stretch_path(Pf[:, :steps], np.full(B, steps * 2 // 3), 1.5, steps=steps)
    rng = np.random.default_rng(5)
    jumps = np.zeros((B, steps), np.int64)
    for b in range(B):
        w = 0
        for j in range(steps):
            jumps[b, j] = w
            w = int(np.clip(w + rng.choice([-7, -1, 0, 0, 1, 2, 25, 60]), 0, N - 1))
    tail = N - WIN + rng.integers(0, WIN, size=(B, steps))
    out = []
    for p, n in ((p07, n07), (p15, n15), (jumps, n0), (tail, n0)):
        full = np.zeros((B, steps), np.int64)
        full[:, :p.shape[1]] = p[:, :steps]
        out.append((full, np.asarray(n)))
    return out


@pytest.mark.parametrize("mode", [1, 0], ids=["persistent", "graph"])
def test_arbitrary_paths_match_the_stepwise_loop(path_engine, mode):
    e = path_engine
    _mode(e, mode)
    B, steps = 3, 40
    L = _texts(B, 700)
    _, Pf, _, _ = e.text2mel_generate(L, steps=steps)
    for i, (path, n) in enumerate(_arbitrary_paths(Pf.cpu().numpy(), steps)):
        Y, P, M = e.text2mel_generate_path(L, path, n)
        # the step-wise loop (one full-recompute sess.run per frame) fed the same windows
        Ys = torch.zeros((B, T, hp.n_mels), device=e.device)
        for j in range(steps):
            pma = torch.as_tensor(path[:, j], dtype=torch.int32, device=e.device)
            _Y, _, _ = e.text2mel_forward(L, Ys, pma, want_alignments=False)
            Ys[:, j] = _Y[:, j]
        for b, k in enumerate(n):
            Ys[b, k:] = 0
            assert torch.equal(P[b, :k].cpu(), torch.as_tensor(path[b, :k], dtype=torch.int32)), (i, b)
        assert (Y - Ys).abs().max().item() < 1e-5, i
        _check_tail(Y, P, M, n)
        # a permuted batch gives the permuted result, bit for bit
        perm = [2, 0, 1]
        Yp, Pp, Mp = e.text2mel_generate_path(L[perm], path[perm], n[perm])
        assert torch.equal(Yp, Y[perm]) and torch.equal(Pp, P[perm]) and torch.equal(Mp, M[perm]), i


@pytest.fixture(scope="module")
def oracle_case(params):
    """Three utterances, 24 frames: backward moves, long jumps, windows at the end of the text, and a stretched run; the
    CPU oracle's synthesize graph (full recompute per frame, float32) fed those windows, computed once."""
    import ref_window_path as rw
    L = np.concatenate([synthetic_text(1, n, seed=11 + n) for n in (60, 120, 175)])
    path = np.array([[0, 0, 3, 3, 1, 9, 9, 2, 40, 40, 41, 0, 0, 1, 1, 1, 2, 2, 30, 31, 31, 31, 32, 33],
                     [N - WIN, N - 1, N - 3, 5, 5, 5, 6, 0, 0, 0, 17, 17, N - 2, N - 2, 4, 4, 4, 90, 90, 91, 91, 92, 0, 0],
                     [0, 0, 0, 1, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4, 4, 5, 5, 5, 6, 6, 6, 7, 7, 7]])
    lengths = np.array([24, 19, 24])
    return L, path, lengths, rw.forced_path(params, L, path)


@pytest.mark.parametrize("mode", [1, 0], ids=["persistent", "graph"])
def test_forced_path_matches_the_oracle(path_engine, oracle_case, mode):
    """Y within the suite's 1e-3 of the oracle below each length, and the argmax inside the forced window equal to the
    oracle's on every row.  The case is chosen free of near-ties: every row's top-2 probability gap is above 1e-3, ten
    times the suite's near-tie margin, so no row is skipped."""
    e = path_engine
    _mode(e, mode)
    L, path, n, r = oracle_case
    Yt, P, Mt = e.text2mel_generate_path(L, path, n)
    _check_tail(Yt, P, Mt, n)
    Y, M = Yt.cpu().numpy(), Mt.cpu().numpy()
    for b, k in enumerate(n):
        assert np.abs(Y[b, :k] - r["Y"][b, :k]).max() < 1e-3, b
        assert (r["margin"][b, :k] > 1e-3).all(), (b, r["margin"][b, :k])
        assert np.array_equal(M[b, :k], r["argmax"][b, :k]), b


def test_refusals_launch_nothing(path_engine):
    import ctypes as C
    from dc_tts_b200.engine import _ptr
    e = path_engine
    L = synthetic_text(3, 30, seed=1)
    ok = np.zeros((3, 20), np.int64)
    cases = [
        (dict(path=np.where(np.arange(20) == 7, N, 0)[None].repeat(3, 0)), "utterance 0 has window %d at frame 7" % N),
        (dict(path=ok - (np.arange(3) == 2)[:, None]), "utterance 2 has window -1 at frame 0"),
        (dict(path=ok, lengths=[5, 0, 5]), "utterance 1 has length 0"),
        (dict(path=ok, lengths=[5, 5, 21]), "utterance 2 has length 21"),
    ]
    before = e.launch_count()
    for kw, msg in cases:
        with pytest.raises(DcttsError, match=msg):
            e.text2mel_generate_path(L, **kw)
    # both C entry points (device and host arrays) check on their own, before any launch
    Ld = e._i32(L)
    Y, P, M = e._empty(3, T, hp.n_mels), e._empty(3, T, dtype=torch.int32), e._empty(3, T, dtype=torch.int32)
    for path, n, msg in ((ok + (np.arange(20) == 19) * N, [20, 20, 20], b"utterance 0 has window"),
                         (ok, [20, 21, 20], b"utterance 1 has length 21")):
        p, nn = e._i32(path), e._i32(np.asarray(n))
        rc = e._lib.dctts_text2mel_generate_path(e._h, _ptr(Ld), 3, 20, _ptr(p), _ptr(nn), _ptr(Y), _ptr(P), _ptr(M),
                                                 C.c_void_p(0))
        assert rc != 0 and msg in e._lib.dctts_last_error(e._h)
        ph, nh = np.ascontiguousarray(path, np.int32), np.asarray(n, np.int32)
        rc = e._lib.dctts_text2mel_generate_path_host(e._h, _ptr(Ld), 3, 20, C.c_void_p(ph.ctypes.data),
                                                      C.c_void_p(nh.ctypes.data), _ptr(Y), _ptr(P), _ptr(M), C.c_void_p(0))
        assert rc != 0 and msg in e._lib.dctts_last_error(e._h)
    assert e.launch_count() == before
    # a window past a length is never read, so it is not checked
    e.text2mel_generate_path(L, ok + (np.arange(20) >= 10) * 10 * N, lengths=[10, 10, 10])
    assert e.launch_count() > before


@pytest.mark.parametrize("mode", [1, 0], ids=["persistent", "graph"])
def test_device_and_host_entry_points_agree(path_engine, mode):
    """dctts_text2mel_generate_path (device arrays, read back) and _host (what the Engine calls) give the same bits."""
    import ctypes as C
    from dc_tts_b200.engine import _ptr
    e = path_engine
    _mode(e, mode)
    B, steps = 4, 50
    L = _texts(B, 40)
    rng = np.random.default_rng(3)
    path = np.clip(np.cumsum(rng.integers(-1, 4, size=(B, steps)), axis=1), 0, N - 1).astype(np.int32)
    n = np.array([50, 1, 33, 49], np.int32)
    Ld = e._i32(L)
    out = []
    for host in (False, True):
        Y, P, M = e._empty(B, T, hp.n_mels), e._empty(B, T, dtype=torch.int32), e._empty(B, T, dtype=torch.int32)
        if host:
            rc = e._lib.dctts_text2mel_generate_path_host(e._h, _ptr(Ld), B, steps, C.c_void_p(path.ctypes.data),
                                                          C.c_void_p(n.ctypes.data), _ptr(Y), _ptr(P), _ptr(M),
                                                          C.c_void_p(0))
        else:
            p, nn = e._i32(path), e._i32(n)
            rc = e._lib.dctts_text2mel_generate_path(e._h, _ptr(Ld), B, steps, _ptr(p), _ptr(nn), _ptr(Y), _ptr(P),
                                                     _ptr(M), C.c_void_p(0))
        assert rc == 0, e._lib.dctts_last_error(e._h)
        torch.cuda.synchronize()
        out.append((Y, P, M))
    for a, b in zip(*out):
        assert torch.equal(a, b)
    _check_tail(*out[0], n)


@pytest.mark.parametrize("scale", [1.25, 0.8])
def test_synthesize_duration_scale(tmp_path, monkeypatch, scale):
    """synthesize(duration_scale=...): each length is the stretched EOS length, Y is the decode along the stretched
    path, and each wav is the ragged vocoder's output at r times that length.  At 1.0 it is synthesize() itself."""
    from scipy.io.wavfile import read as read_wav
    from dc_tts_b200 import engine as engine_mod
    from dc_tts_b200.data_load import load_data
    from dc_tts_b200.engine import Engine
    from dc_tts_b200.synthesize import synthesize
    from dc_tts_b200.train import Graph
    from dc_tts_b200.utils import spectrograms2wavs

    texts = ["a cat", "the dog ran far away", "hello", "it is"]
    sent = tmp_path / "sentences.txt"
    sent.write_text("header\n" + "".join("%d. %s\n" % (i + 1, t) for i, t in enumerate(texts)))
    out = tmp_path / "samples"
    monkeypatch.setattr(hp, "sampledir", str(out))
    prev = engine_mod._default
    e = Engine(0)
    engine_mod.set_engine(e)
    try:
        Y1, Z1 = synthesize(params=init_params(0), sentences=str(sent), write=False)
        # the later calls use the parameters this one committed
        Yd, Zd = synthesize(sentences=str(sent), write=False, duration_scale=1.0)
        assert np.array_equal(Y1, Yd) and np.array_equal(Z1, Zd)

        Y, Z = synthesize(sentences=str(sent), write=True, duration_scale=scale)
        L = load_data("synthesize", str(sent))
        g = Graph(mode="synthesize")
        _, Pu, nu = g.generate_until_eos(L)
        path, n = stretch_path(Pu, nu, scale)
        nu = nu.cpu().numpy()
        for b in range(len(texts)):
            assert n[b] == max(1, round(scale * int(nu[b]))), (b, n[b], nu[b])
        Ya, _, _ = g.generate_along(L, path, n)
        assert np.array_equal(Y, Ya.cpu().numpy())
        wavs = spectrograms2wavs(Z[:, :hp.r * int(n.max())], lengths=hp.r * n)
        for b, k in enumerate(n):
            assert not Y[b, k:].any() and not Z[b, hp.r * k:].any()
            sr, wav = read_wav(os.path.join(str(out), "%d.wav" % (b + 1)))
            assert np.array_equal(wav, wavs[b]), b
    finally:
        engine_mod.set_engine(prev)
        e.close()
