"""Aligning recorded speech to its text on the GPU (Engine.text2mel_align, Engine.align_search, Graph.align and
synthesize(timing_from=...)), on both tensor paths.

The teacher-forced alignments are held to the float64 oracle (ref_torch composed as the dense forward); the search to
the float64 restatement tests/ref_align.py, exactly on synthetic alignments and wherever the reference reports no
near-tie on the GPU's own.  On the wgmma path an utterance aligned alone equals the same utterance in a batch, bit for
bit."""
import numpy as np
import pytest
import torch

from dc_tts_b200.engine import DcttsError, Engine
from dc_tts_b200.hyperparams import Hyperparams
from dc_tts_b200.params import synthetic_text
from oracle import ref_torch as rt
from ref_align import admissible, path_score, search_batch

pytestmark = pytest.mark.gpu

EOS = Hyperparams.vocab.index("E")
# alignments against the float64 oracle, by tensor path: about 3x the worst measured (3.7e-7 on the wgmma kernels, 1.1e-7
# on the fp32 ones; DESIGN.md section 4d)
ATOL = {1: 1.2e-6, 0: 3.5e-7}
NEAR_TIE = 1e-9


@pytest.fixture
def side_engine(params):
    made = []

    def make(H=Hyperparams, P=None):
        e = Engine(0, hparams=H)
        e.load_params(params if P is None else P)
        made.append(e)
        return e
    yield make
    for e in made:
        e.close()


@pytest.fixture
def tp_engine(engine):
    yield engine
    engine.set_tensor_path(1)


def _noise_wav(seconds, seed, sr=Hyperparams.sr):
    """Noise bursts with silences between them, int16."""
    rng = np.random.default_rng(seed)
    n = int(seconds * sr)
    env = np.repeat(rng.random(n // 2205 + 1) < 0.6, 2205)[:n] * rng.uniform(0.05, 0.5)
    return np.clip(rng.standard_normal(n) * env * 32767 * 0.3, -32768, 32767).astype(np.int16)


def _batch(e, B, seed, wav_mel=None):
    """B utterances with ragged frame counts (utterance 0 at the full T): U(0, 1) mels, an all-zero recording at b = 1,
    and feature-scale mels from a synthetic wav at b = 2; texts as long as the window size lets each recording reach."""
    h = e.hp
    rng = np.random.default_rng(seed)
    T = h.max_T
    n = rng.integers(max(1, T // 4), T + 1, B)
    n[0] = T
    mels = np.zeros((B, T, h.n_mels), np.float32)
    for b in range(B):
        if b != 1:
            mels[b, :n[b]] = rng.random((n[b], h.n_mels))
    if wav_mel is not None and B > 2:
        k = min(T, len(wav_mel))
        n[2] = k
        mels[2] = 0
        mels[2, :k] = wav_mel[:k]
    L = np.zeros((B, h.max_N), np.int32)
    for b in range(B):
        c = int(rng.integers(1, min(h.max_N - 1, (h.attention_win_size - 1) * n[b]) + 1))
        L[b, :c] = rng.integers(2, 32, c)
        L[b, c] = EOS
    return L, mels, n


def _wav_mel(e):
    mel, _, t, _ = e.load_spectrograms_batch([_noise_wav(2.5, 11)])
    return mel[0, :int(t[0])].cpu().numpy()


@torch.no_grad()
def _oracle(P, L, mels):
    m = torch.as_tensor(mels, dtype=torch.float64)
    S = torch.cat((torch.zeros_like(m[:, :1]), m[:, :-1]), 1)
    K, _ = rt.TextEnc(P, torch.as_tensor(L), torch.float64)
    Q = rt.AudioEnc(P, S)
    A = torch.softmax(Q @ K.transpose(1, 2) / np.sqrt(Hyperparams.d), -1)
    return A.transpose(1, 2).numpy()


def _ends(L):
    return (np.asarray(L) == EOS).argmax(1)


def _check_search(e, A, n, ends, out):
    """GPU outputs (path, chars, durations, score) against ref_align on the same alignments; returns the near-tie rows."""
    path, chars, dur, score = (x.cpu().numpy() for x in out)
    r = search_batch(A, n, ends, e.hp.attention_win_size)
    near = []
    for b in range(len(n)):
        k = int(n[b])
        assert admissible(chars[b, :k], ends[b], e.hp.attention_win_size), b
        assert (chars[b, k:] == -1).all() and (path[b, k:] == -1).all(), b
        assert path[b, 0] == 0 and (path[b, 1:k] == chars[b, :k - 1]).all(), b
        assert dur[b].sum() == k and (dur[b] == np.bincount(chars[b, :k], minlength=A.shape[1])).all(), b
        assert abs(path_score(A[b], chars[b, :k]) - r["score"][b]) <= 1e-12 * abs(r["score"][b]), b
        assert abs(score[b] - r["score"][b]) <= 1e-12 * abs(r["score"][b]), b
        if r["margin"][b] < NEAR_TIE:
            near.append(b)
            continue
        assert (chars[b] == r["chars"][b]).all() and (path[b] == r["path"][b]).all(), b
        assert (dur[b] == r["durations"][b]).all(), b
    return near


HANDLES = {"stock": {}, "N300_T60": dict(max_N=300, max_T=60)}


@pytest.mark.parametrize("handle", list(HANDLES))
@pytest.mark.parametrize("tp", [1, 0], ids=["tensorpath", "fp32path"])
def test_alignments_and_search_against_references(engine, side_engine, params, handle, tp):
    e = engine if handle == "stock" else side_engine(type("H_" + handle, (Hyperparams,), HANDLES[handle]))
    e.set_tensor_path(tp)
    try:
        wm = _wav_mel(e)
        worst = 0.0
        for B in (1, 5, 32):
            L, mels, n = _batch(e, B, 100 + B, wm)
            out = e.text2mel_align(L, torch.as_tensor(mels).cuda(), lengths=n, want_alignments=True)
            A = out[4].cpu().numpy()
            err = float(np.abs(A - _oracle(params, L, mels)).max())
            worst = max(worst, err)
            assert err <= ATOL[tp], (B, err)
            near = _check_search(e, A, n, _ends(L), out[:4])
            assert len(near) <= max(1, B // 8), near
        print("align oracle %s tp=%d worst |A - A64| = %.3e" % (handle, tp, worst))
    finally:
        e.set_tensor_path(1)


def _synthetic(kind, B, N, T, w, rng):
    n = rng.integers(1, T + 1, B)
    n[0] = T
    ends = np.array([int(rng.integers(0, min(N - 1, (w - 1) * k) + 1)) for k in n])
    if kind == "uniform":
        A = np.full((B, N, T), np.float32(1.0 / N))
    elif kind == "floors":
        A = rng.random((B, N, T)).astype(np.float32)
        A[rng.random(A.shape) < 0.7] = 0
        A[rng.random(A.shape) < 0.1] = np.float32(1e-35)
    else:
        A = rng.random((B, N, T)).astype(np.float32) * 0.05
        for b in range(B):
            k = int(n[b])
            diag = np.floor(np.arange(k) * ends[b] / max(1, k - 1) + 1e-9).astype(np.int64)
            A[b, diag, np.arange(k)] += 1.0
        A /= A.sum(1, keepdims=True)
    return A, n, ends


@pytest.mark.parametrize("win", [1, 2, 3, 4])
def test_search_on_synthetic_alignments_is_exact(engine, side_engine, win):
    e = engine if win == 3 else side_engine(type("Hw%d" % win, (Hyperparams,), {"attention_win_size": win}))
    rng = np.random.default_rng(win)
    for kind in ("uniform", "floors", "diagonal"):
        for B, N, T in ((1, 7, 5), (6, 60, 90), (33, 180, 210)):
            A, n, ends = _synthetic(kind, B, N, T, win, rng)
            out = e.align_search(torch.as_tensor(A).cuda(), n, ends)
            assert _check_search(e, A, n, ends, out) == [] or kind != "diagonal", (kind, B)
            r = search_batch(A, n, ends, win)
            path, chars, dur, _ = (x.cpu().numpy() for x in out)
            assert (chars == r["chars"]).all() and (path == r["path"]).all() and (dur == r["durations"]).all(), (kind, B)


def test_batch_invariance_tensor_path(tp_engine):
    e = tp_engine
    e.set_tensor_path(1)
    L, mels, n = _batch(e, 9, 7, _wav_mel(e))
    full = e.text2mel_align(L, torch.as_tensor(mels).cuda(), lengths=n, want_alignments=True)
    for b in range(len(n)):
        k = int(n[b])
        one = e.text2mel_align(L[b:b + 1], torch.as_tensor(mels[b:b + 1, :k]).cuda(), want_alignments=True)
        for x, y in zip(one[:3], full[:3]):
            assert torch.equal(x[0], y[b, :x.shape[1]]), b
        assert torch.equal(one[3][0], full[3][b]), b
        assert torch.equal(one[4][0], full[4][b, :, :k]), b
    perm = np.random.default_rng(3).permutation(len(n))
    pm = e.text2mel_align(L[perm], torch.as_tensor(mels[perm]).cuda(), lengths=n[perm], want_alignments=True)
    for x, y in zip(pm, full):
        assert torch.equal(x, y[torch.as_tensor(perm).cuda()])


def test_batch_invariance_fp32_path(tp_engine):
    e = tp_engine
    e.set_tensor_path(0)
    L, mels, n = _batch(e, 6, 8, _wav_mel(e))
    full = e.text2mel_align(L, torch.as_tensor(mels).cuda(), lengths=n, want_alignments=True)
    A = full[4].cpu().numpy()
    r = search_batch(A, n, _ends(L), e.hp.attention_win_size)
    for b in range(len(n)):
        k = int(n[b])
        one = e.text2mel_align(L[b:b + 1], torch.as_tensor(mels[b:b + 1, :k]).cuda(), want_alignments=True)
        assert float((one[4][0] - full[4][b, :, :k]).abs().max()) <= 2 * ATOL[0], b     # two results, each within ATOL
        if r["margin"][b] >= NEAR_TIE:
            assert torch.equal(one[1][0], full[1][b, :k]), b


def test_refusals_name_the_utterance(tp_engine):
    e = tp_engine
    h = e.hp
    L, mels, n = _batch(e, 4, 9)
    md = torch.as_tensor(mels).cuda()
    before = e.launch_count()
    bad_len = n.copy(); bad_len[2] = 0
    with pytest.raises(DcttsError, match="utterance 2"):
        e.text2mel_align(L, md, lengths=bad_len)
    bad_len[2] = h.max_T + 1
    with pytest.raises(DcttsError, match="utterance 2"):
        e.text2mel_align(L, md, lengths=bad_len)
    short = n.copy(); short[3] = 1
    L3 = L.copy(); L3[3] = 0; L3[3, :10] = 5; L3[3, 10] = EOS
    with pytest.raises(DcttsError, match="utterance 3.*too long"):
        e.text2mel_align(L3, md, lengths=short)
    noeos = L.copy(); noeos[1] = 7
    with pytest.raises(DcttsError, match="utterance 1 has no EOS"):
        e.text2mel_align(noeos, md, lengths=n)
    with pytest.raises(DcttsError, match="max_T"):
        e.text2mel_align(L, torch.zeros(4, h.max_T + 1, h.n_mels, device="cuda"))
    assert e.launch_count() == before
    # the C-ABI's own checks, past the Python ones: nothing launched, the outputs untouched
    import ctypes as C
    B, N, T = 4, h.max_N, h.max_T
    outs = [torch.full((B, T), 77, dtype=torch.int32, device="cuda"), torch.full((B, T), 77, dtype=torch.int32, device="cuda"),
            torch.full((B, N), 77, dtype=torch.int32, device="cuda"), torch.full((B,), 77.0, dtype=torch.float64, device="cuda")]
    Ld = torch.as_tensor(L).cuda()
    for lens, ends, msg in ((bad_len, _ends(L), "utterance 2"), (short, _ends(L3), "utterance 3"),
                            (n, np.where(np.arange(4) == 1, N, _ends(L)), "utterance 1")):
        ln, en = np.ascontiguousarray(lens, np.int32), np.ascontiguousarray(ends, np.int32)
        rc = e._lib.dctts_text2mel_align(e._h, C.c_void_p(Ld.data_ptr()), C.c_void_p(md.data_ptr()), B, T,
                                         C.c_void_p(ln.ctypes.data), C.c_void_p(en.ctypes.data),
                                         *[C.c_void_p(o.data_ptr()) for o in outs], None, e._stream())
        assert rc != 0 and msg in e._lib.dctts_last_error(e._h).decode(), msg
    torch.cuda.synchronize()
    assert e.launch_count() == before
    assert all(bool((o == 77).all()) for o in outs)


def test_replay_and_synthesize_timing_from(tp_engine, tmp_path, monkeypatch):
    from scipy.io import wavfile

    from dc_tts_b200 import synthesize as syn
    from dc_tts_b200 import utils
    from dc_tts_b200.data_load import load_data
    from dc_tts_b200.hyperparams import Hyperparams as hp
    from dc_tts_b200.train import Graph
    from dc_tts_b200.utils import stretch_path
    e = tp_engine
    # every recovered path replays
    L, mels, n = _batch(e, 5, 21, _wav_mel(e))
    path, chars, _, _ = e.text2mel_align(L, torch.as_tensor(mels).cuda(), lengths=n)
    _, P, _ = e.text2mel_generate_path(L, path.cpu().numpy(), n)
    assert torch.equal(P[:, :path.shape[1]], path) and bool((P[:, path.shape[1]:] == -1).all())

    sents = tmp_path / "sents.txt"
    sents.write_text("header\n1. the birch canoe slid on the\n2. glue the sheet to the\n3. it is easy to tell\n")
    wavs = []
    for i, (sec, sr) in enumerate(((2.2, hp.sr), (1.6, 16000), (2.9, hp.sr))):
        p = str(tmp_path / ("rec%d.wav" % i))
        wavfile.write(p, sr, _noise_wav(sec, 40 + i, sr))
        wavs.append(p)
    got = {}

    def fake_vocoder(Z, lengths=None, momentum=0.0):
        got["Z"], got["lengths"] = np.array(Z), np.array(lengths)
        return [np.zeros(10, np.float32) for _ in range(len(Z))]
    monkeypatch.setattr(utils, "spectrograms2wavs", fake_vocoder)
    monkeypatch.setattr(hp, "sampledir", str(tmp_path / "samples"))
    Lt = load_data("synthesize", str(sents))
    _, mt, _, t = utils.load_spectrograms_batch(wavs, e, resample=True)
    for scale in (1.0, 1.3):
        Y, Z = syn.synthesize(sentences=str(sents), timing_from=wavs, duration_scale=scale)
        g = Graph(mode="synthesize", engine=e)
        p, _, _, _ = g.align(Lt, mt, t)
        nn = t
        if scale != 1.0:
            p, nn = stretch_path(p, t, scale)
        Yh, _, _ = g.generate_along(Lt, p, nn)
        _, Zh = e.ssrn(Yh[:, :int(nn.max())], want_logits=False, lengths=nn)
        assert (got["lengths"] == hp.r * np.asarray(nn)).all(), scale
        assert np.array_equal(Y, Yh.cpu().numpy()), scale
        assert np.array_equal(Z[:, :hp.r * int(nn.max())], Zh.cpu().numpy()) and not Z[:, hp.r * int(nn.max()):].any(), scale
    with pytest.raises(ValueError, match="rec1.wav"):
        long = str(tmp_path / "rec1.wav")
        wavfile.write(long, 16000, _noise_wav(hp.max_T * hp.r * hp.hop_length / hp.sr + 1.0, 5, 16000))
        syn.synthesize(sentences=str(sents), timing_from=wavs)


def test_no_side_effects_on_synthesis(engine, side_engine, params):
    e = engine
    e.set_tensor_path(1)
    L = np.concatenate([synthetic_text(1, 30 + 20 * i, seed=60 + i) for i in range(3)])
    Y0, P0 = e.text2mel_generate(L)[:2]
    Yu0 = e.text2mel_generate_until(L, tail=2)
    mels = torch.rand(3, 150, e.hp.n_mels, device="cuda")
    e.text2mel_align(L, mels)
    with pytest.raises(DcttsError):
        e.decode_history("Y")
    Y1, P1 = e.text2mel_generate(L)[:2]
    assert torch.equal(Y0, Y1) and torch.equal(P0, P1)
    e.text2mel_align(L, mels)
    Yu1 = e.text2mel_generate_until(L, tail=2)
    assert all(torch.equal(a, b) for a, b in zip(Yu0, Yu1))

    # a trained handle whose packing is stale aligns on the fp32 kernels
    stale = side_engine()
    stale.train_init(1)
    name = "Text2Mel/AudioEnc/C_1/conv1d/bias"
    stale.train_set_tensor(name, params[name])
    ref = side_engine()
    ref.set_tensor_path(0)
    a = stale.text2mel_align(L, mels, want_alignments=True)
    b = ref.text2mel_align(L, mels, want_alignments=True)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
