"""The autoregressive decode one block at a time: after a generation, every block's output rows (Engine.decode_history) are
checked against the float64 reference of that block (tests/ref_decode_blocks.py) computed on the previous block's rows as
the decode left them, so that each block is held to its own rounding: |got - ref| <= tau S.

Rows checked (DESIGN.md, "The decode one block at a time"): every AudioEnc row below the last executed frame s (they never
depend on the window); of AudioDec block i the audiodec_rows[i] rows ending at s - 1, which the last window's frame or
recompute produced from inputs of the same triangle; on a constant window path with the recompute off, every row of every
block.  C_1's input R is the float64 attention of the decode's own Q rows and K | V under the last window, and the decode's
stored R rows are checked against it where it wrote them.  The argmax of every frame must be the float64 argmax wherever the
top-2 margin exceeds its error bound."""
import numpy as np
import pytest
import torch

import ref_decode_blocks as rb
from dc_tts_b200.arch import audiodec_layers, audioenc_layers
from dc_tts_b200.engine import DcttsError, Engine
from dc_tts_b200.hyperparams import Hyperparams
from dc_tts_b200.params import init_params

pytestmark = pytest.mark.gpu

ENC_L, DEC_L = audioenc_layers(), audiodec_layers()
ENC, DEC = "Text2Mel/AudioEnc", "Text2Mel/AudioDec"
WORST = {}                       # group -> worst err / S seen (printed at the end of the module, recorded in DESIGN.md)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\ndecode blocks, worst err / S: " + ", ".join("%s %.3g" % kv for kv in sorted(WORST.items())))


def _texts(B, N, seed, n_max=None):
    n_max = n_max or min(N - 1, 170)
    L = np.zeros((B, N), np.int32)
    for b in range(B):
        rng = np.random.default_rng([seed, b])
        n = 20 + (37 * b + seed) % (n_max - 19)
        L[b, :n] = rng.integers(2, 32, size=n)
        L[b, n] = 1
    return L


def _mode(e, mode, tp=1):
    e.set_tensor_path(tp)
    e.set_option("decode_mode", mode)


def _check(group, got, ref, S, tau, what):
    got = np.asarray(got, np.float64)
    err = np.abs(got - ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(S > 0, err / S, np.where(err > 0, np.inf, 0.0))
    worst = float(r.max()) if r.size else 0.0
    WORST[group] = max(WORST.get(group, 0.0), worst)
    if worst > tau:
        i = np.unravel_index(int(np.argmax(r)), r.shape)
        raise AssertionError("%s: err / S = %.3g > tau = %.3g at %s (got %r, ref %r, S %.3g)"
                             % (what, worst, tau, i, got[i], ref[i], S[i]))


class History:
    """Everything the decode left on the engine, on the host, in the caller's order."""

    def __init__(self, e):
        self.joined = {}
        self.ae = [e.decode_history("audioenc", i)[0].cpu().numpy() for i in range(len(ENC_L))]
        self.ad = []
        for i in range(len(DEC_L)):
            t, j = e.decode_history("audiodec", i)
            self.ad.append(t.cpu().numpy())
            self.joined[i] = j
        self.R = e.decode_history("R")[0].cpu().numpy()
        self.KV = e.decode_history("KV")[0].cpu().numpy()
        self.Y = e.decode_history("Y")[0].cpu().numpy()
        self.windows = e.decode_history("windows")[0].cpu().numpy()


class Params:
    def __init__(self, P):
        self.P = P
        self.enc = [rb.block_params(P, ENC, l) for l in ENC_L]
        self.dec = [rb.block_params(P, DEC, l) for l in DEC_L]


def check_utterance(H, prm, b, s, win, kernels, everything=False):
    """Checks utterance b of the decode left in H, whose last executed frame is s - 1.  kernels: "cluster" (persistent decode),
    "tensorpath" / "fp32path" (graph-per-frame decode on the tensor-core / float32 block kernels), with "tc" in the set when
    the graph-per-frame decode ran its wide AudioDec blocks on the tensor cores (B >= 8).  everything: every row of every
    block (a constant window path without the recompute).

    The stored R rows are checked where the decode wrote them under the last window: the graph-per-frame step attends the
    rows[0] rows ending at its frame (so every row of the triangle was last written by a frame at or after the last window
    move, under that window); the persistent decode writes R only in its recompute, rows f - rows[0] + 1 .. f - 1 at a
    recompute frame f, and a later recompute under the same window rewrites them with the same bits."""
    T = H.Y.shape[1]
    rows = rb.audiodec_rows(DEC_L, T)
    kind, tc, force = kernels
    w = H.windows[b]
    # AudioEnc: Y[j - 1] -> C_1 -> ... -> Q
    x = rb.shifted_feed(H.Y[b])
    for i, l in enumerate(ENC_L):
        ref, S = rb.block(prm.enc[i], l, x, np.arange(s))
        _check("fp32 AudioEnc", H.ae[i][b, :s], ref, S, rb.TAU_FP32, "%s utt %d AudioEnc %s" % (kind, b, l.scope))
        x = H.ae[i][b]
    # the last recompute of the persistent decode: the frame f at or before s - 1 where the window last moved
    f_last = -1
    if kind == "cluster":
        moves = [j for j in range(1, s) if w[j] != w[j - 1] or force]
        f_last = moves[-1] if moves else -1
    # attention of the triangle's rows under the last window (every row under its own window when `everything`)
    lo = 0 if everything else max(0, s - rows[0])
    wins = w[lo:s] if everything else np.full(s - lo, w[s - 1])
    a = rb.attention_rows(H.ae[-1][b, lo:s], H.KV[b], wins, win)
    rr = np.arange(max(lo, f_last - rows[0] + 1), f_last) if kind == "cluster" else np.arange(lo, s)
    if len(rr):
        _check("fp32 attention", H.R[b, rr], a["R"][rr - lo], a["S"][rr - lo], rb.TAU_FP32, "%s utt %d R" % (kind, b))
    x = np.zeros((T, a["R"].shape[1]))
    xs = np.zeros_like(x)
    x[lo:s], xs[lo:s] = a["R"], a["S"]               # R's own float32 error enters C_1 like its input rounding
    for i, l in enumerate(DEC_L):
        r = np.arange(0 if everything else max(0, s - rows[i]), s)
        ref, S = rb.block(prm.dec[i], l, x, r, xs)
        if kind == "cluster":
            split = (rows[i] > 1) & (r < f_last) & (r >= f_last - rows[i] + 1)
        else:
            split = np.full(len(r), bool(tc) and i < 4 and rows[i] >= 32)
        tiles = kind != "cluster"                        # the graph decode's 128-row tiles, else the pre-pass
        for grp, m, tau in (("fp32 AudioDec", ~split, rb.TAU_FP32),
                            ("tiles AudioDec" if tiles else "split AudioDec", split, rb.TAU_TILES if tiles else rb.TAU_SPLIT)):
            if m.any():
                _check(grp, H.ad[i][b, r[m]], ref[m], S[m], tau,
                       "%s utt %d AudioDec %s%s" % (kind, b, l.scope, " (joined planes)" if H.joined[i] else ""))
        x, xs = H.ad[i][b], None
    y, S = rb.mel_sigmoid(H.ad[-1][b, :s])
    _check("fp32 Y", H.Y[b, :s], y, S, rb.TAU_FP32, "%s utt %d Y" % (kind, b))
    return a


def check_argmax(H, b, n, win, amax, windows):
    """amax[j] (j < n) is the argmax of row j under windows[j] wherever the top-2 margin exceeds its bound."""
    a = rb.attention_rows(H.ae[-1][b, :n], H.KV[b], windows[:n], win)
    sure = a["margin"] > 4 * rb.TAU_FP32 * a["Sp"]
    bad = np.flatnonzero(sure & (np.asarray(amax[:n]) != a["argmax"]))
    assert not bad.size, "utt %d: argmax %s at frames %s, float64 %s" % (b, amax[bad], bad, a["argmax"][bad])
    return int(sure.sum())


KERNELS = {"cluster": (1, 1), "tensorpath": (0, 1), "fp32path": (0, 0)}     # name -> (decode_mode, tensor_path)
# Batches of 8: the graph-per-frame decode runs its wide AudioDec blocks as 128-row tensor-core tiles from B = 8 on (below
# that "tensorpath" would run the float32 kernels); a subset of the utterances is checked, to keep the references cheap.
B8, CHECK8 = 8, [0, 3, 7]


def _run_free(e, prm, L, steps, name, force=0, check=None):
    mode, tp = KERNELS[name]
    _mode(e, mode, tp)
    e.set_option("decode_force_prepass", force)
    try:
        _, P, _, _ = e.text2mel_generate(L, steps=steps)
    finally:
        e.set_option("decode_force_prepass", 0)
    H = History(e)
    B = L.shape[0]
    assert np.array_equal(H.windows[:, :steps], P.cpu().numpy()[:, :steps])
    kern = (name, mode == 0 and tp == 1 and B >= 8, force)
    for b in (range(B) if check is None else check):
        check_utterance(H, prm, b, steps, e.hp.attention_win_size, kern)
        # p_hist[:, j + 1] is the argmax of row j
        check_argmax(H, b, steps - 1, e.hp.attention_win_size, H.windows[b, 1:steps], H.windows[b])
    return H


def _run_path(e, prm, L, path, n, name, force=0, everything=False, check=None):
    mode, tp = KERNELS[name]
    _mode(e, mode, tp)
    e.set_option("decode_force_prepass", force)
    try:
        _, _, M = e.text2mel_generate_path(L, path, n)
    finally:
        e.set_option("decode_force_prepass", 0)
    H = History(e)
    M = M.cpu().numpy()
    B = L.shape[0]
    kern = (name, mode == 0 and tp == 1 and B >= 8, force)
    for b in (range(B) if check is None else check):
        s = int(n[b])
        assert np.array_equal(H.windows[b, :s], path[b, :s])
        check_utterance(H, prm, b, s, e.hp.attention_win_size, kern, everything=everything)
        check_argmax(H, b, s, e.hp.attention_win_size, M[b], path[b])
    return H


@pytest.fixture(scope="module")
def prm(params):
    return Params(params)


@pytest.fixture
def eng(engine):
    yield engine
    engine.set_option("decode_force_prepass", 0)
    _mode(engine, 1, 1)


def _need(e, name):
    if KERNELS[name][0] == 1 and not e.get_option("decode_available"):
        pytest.skip("no persistent decode on this device")


# ---------------------------------------------------------------------------------------------- free runs, truncated
@pytest.mark.parametrize("name,force", [("cluster", 0), ("cluster", 1), ("tensorpath", 0), ("fp32path", 0)])
def test_free_runs_truncated(eng, prm, name, force):
    """Runs ending right at a window move, one frame after, and long after (first utterance's moves)."""
    _need(eng, name)
    L = _texts(B8, eng.hp.max_N, 17)
    _mode(eng, *KERNELS[name])
    _, P, _, _ = eng.text2mel_generate(L)
    p = P.cpu().numpy()[0]
    moves = [j for j in range(1, len(p)) if p[j] != p[j - 1]]
    assert len(moves) >= 2
    for s in sorted({moves[0] + 1, moves[0] + 2, moves[len(moves) // 2] + 1, eng.hp.max_T}):
        _run_free(eng, prm, L, s, name, force, check=CHECK8)


# ---------------------------------------------------------------------------------------------- utterances per cluster
@pytest.mark.parametrize("G", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("name", ["cluster", "tensorpath"])
def test_utterances_per_cluster(eng, prm, G, name):
    """B = (G - 1) mc + 1 and G mc, so that the persistent decode runs G utterances per cluster with a partial and a full
    last cluster; a path with moves and a jump, the recompute forced on every second B.  The first and last utterance of
    every cluster are checked."""
    _need(eng, "cluster")
    mc = max(1, eng.get_option("decode_max_clusters"))
    N, steps = eng.hp.max_N, 30
    for k, B in enumerate(sorted({max(1, (G - 1) * mc + 1), G * mc})):
        g = 1
        while g < 5 and -(-B // g) > mc:
            g += 1
        assert g == G or B < G, (B, g, G)
        L = _texts(B, N, 30 + B)
        rng = np.random.default_rng(B)
        path = np.clip(np.cumsum(rng.choice([0, 0, 0, 1, 1, 2, 9], size=(B, steps)), 1) - 1, 0, N - 1)
        n = np.full(B, steps)
        n[::3] = steps - 1 - np.arange(len(n[::3])) % 7
        order = np.argsort(n, kind="stable")            # the decode order: clusters are consecutive utterances of it
        check = sorted({int(order[c]) for i in range(0, B, g) for c in (i, min(B, i + g) - 1)})
        _run_path(eng, prm, L, path, n, name, force=k % 2 if name == "cluster" else 0, check=check)


# ---------------------------------------------------------------------------------------------- windows
@pytest.mark.parametrize("name", ["cluster", "tensorpath", "fp32path"])
def test_constant_windows_every_row(eng, prm, name):
    """A constant window at 0 and at N - 3, N - 2, N - 1 (fewer live keys): every row of every block, every frame."""
    _need(eng, name)
    N, steps = eng.hp.max_N, 48
    L = _texts(B8, N, 5)
    path = np.repeat(np.array([0, N - 3, N - 2, N - 1, 0, N - 3, N - 2, N - 1])[:, None], steps, 1)
    n = np.array([steps, steps, steps - 5, steps, steps - 1, steps, steps, steps - 2])
    _run_path(eng, prm, L, path, n, name, everything=True, check=[0, 1, 2, 3, 7])


@pytest.mark.parametrize("name,force", [("cluster", 0), ("cluster", 1), ("tensorpath", 0), ("fp32path", 0)])
def test_arbitrary_paths(eng, prm, name, force):
    """Stretched and jumping paths, windows at the end of the text, ragged lengths (tests/test_gpu_window_path.py)."""
    from test_gpu_window_path import _arbitrary_paths
    _need(eng, name)
    steps = 40
    L = _texts(B8, eng.hp.max_N, 70)
    _mode(eng, *KERNELS[name])
    _, Pf, _, _ = eng.text2mel_generate(L, steps=steps)
    for path, n in _arbitrary_paths(Pf.cpu().numpy(), steps):
        _run_path(eng, prm, L, path, n, name, force, check=CHECK8)


# ---------------------------------------------------------------------------------------------- parameter sets
def _const_params(P, value, near=False):
    """A zero kernel (or the kernel times 1e-6) and a constant bias in AudioEnc C_3, AudioDec HC_2 and the 80-channel C_11."""
    Q = dict(P)
    for s in ("Text2Mel/AudioEnc/C_3", "Text2Mel/AudioDec/HC_2", "Text2Mel/AudioDec/C_11"):
        Q[s + "/conv1d/kernel"] = (P[s + "/conv1d/kernel"] * np.float32(1e-6)) if near else np.zeros_like(P[s + "/conv1d/kernel"])
        Q[s + "/conv1d/bias"] = np.full_like(P[s + "/conv1d/bias"], value)
    return Q


@pytest.fixture
def side_engine():
    """Handles of a test's own (parameter sets, hyperparameters), closed at its end."""
    made = []

    def make(P, H=Hyperparams):
        e = Engine(0, hparams=H)
        e.load_params(P)
        made.append(e)
        return e
    yield make
    for e in made:
        e.close()


@pytest.mark.parametrize("scheme", ["tf_default", "const0.75", "const1e3", "near_const"])
def test_parameter_sets(side_engine, params, scheme):
    if scheme == "tf_default":
        P = init_params(0, "tf_default")
    else:
        P = _const_params(params, 0.75 if scheme != "const1e3" else 1e3, near=scheme == "near_const")
    e = side_engine(P)
    prm = Params(P)
    L = _texts(B8, e.hp.max_N, 9)
    names = ["cluster", "tensorpath", "fp32path"] if e.get_option("decode_available") else ["tensorpath", "fp32path"]
    for name in names:
        H = _run_free(e, prm, L, 36, name, force=1 if name == "cluster" else 0, check=CHECK8)
        if scheme == "tf_default":
            # frame 0: AudioEnc C_1 reads zeros and every bias is 0, so every AudioEnc row 0 is beta = 0 exactly
            for i in range(len(ENC_L)):
                assert not H.ae[i][:, 0].any(), (name, i)
        elif scheme != "near_const":
            b3 = P["Text2Mel/AudioEnc/C_3/normalize/beta"]
            b11 = P["Text2Mel/AudioDec/C_11/normalize/beta"]
            assert (H.ae[2][:, :36] == b3).all(), name                  # exactly beta
            assert (H.ad[-1][:, :36] == b11).all(), name                # the logits: beta of the 5-channel-slice block


# ---------------------------------------------------------------------------------------------- hyperparameters
HANDLES = {"win1": dict(attention_win_size=1), "win2": dict(attention_win_size=2), "win4": dict(attention_win_size=4),
           "N300": dict(max_N=300), "T60": dict(max_T=60), "T300": dict(max_T=300)}


@pytest.mark.parametrize("handle", list(HANDLES))
def test_handles(side_engine, params, handle):
    """Window sizes 1, 2, 4; max_N = 300 with windows up to 299; max_T = 60 (shorter than the receptive field) and 300."""
    H = type("H_" + handle, (Hyperparams,), HANDLES[handle])
    e = side_engine(params, H)
    prm = Params(params)
    names = ["cluster", "tensorpath", "fp32path"]
    if not e.get_option("decode_available"):
        with pytest.raises(DcttsError, match="persistent decode"):
            e.set_option("decode_mode", 1)
        names = names[1:]
    N, T, W = H.max_N, H.max_T, H.attention_win_size
    L = _texts(B8, N, 4, n_max=N - 1)
    steps = min(T, 50)
    rng = np.random.default_rng(2)
    path = np.clip(np.cumsum(rng.choice([0, 0, 1, 1, 3, 40], size=(B8, steps)), 1), 0, N - 1)
    path[2] = N - 1 - np.arange(steps) % W
    n = np.full(B8, steps)
    n[1::3] -= 3
    for name in names:
        _run_free(e, prm, L, T if T <= 60 else steps, name, force=1 if name == "cluster" else 0, check=[0, 2, 7])
        _run_path(e, prm, L, path, n, name, check=[0, 1, 2, 7])
    if T > 210:                                   # past the default max_T: one whole-length run
        _run_free(e, prm, L, T, names[0], check=[1])


# ---------------------------------------------------------------------------------------------- full-sequence attention
@pytest.mark.parametrize("win", [1, 2, 3, 4])
@pytest.mark.parametrize("tp", [1, 0], ids=["tc", "simt"])
def test_full_sequence_attention(side_engine, engine, params, win, tp):
    """Engine.attention(monotonic=True) at each window size: attention_tc_kernel (tensor path 1) and the SIMT
    attention_kernel (0) against the float64 attention."""
    e = engine if win == 3 else side_engine(params, type("Hw%d" % win, (Hyperparams,), {"attention_win_size": win}))
    e.set_tensor_path(tp)
    try:
        B, T, N, d = 3, 64, e.hp.max_N, e.hp.d
        g = torch.Generator().manual_seed(win)
        Q, K, V = (torch.randn(B, n, d, generator=g) for n in (T, N, N))
        pma = np.array([0, N // 2, N - 1])
        R, A, M = e.attention(Q, K, V, monotonic=True, prev_max_attentions=pma)
        R, M = R.cpu().numpy(), M.cpu().numpy()
        tau = rb.TAU_ATTN_TC if tp == 1 else rb.TAU_FP32
        for b in range(B):
            a = rb.attention_rows(Q[b].numpy(), torch.cat([K[b], V[b]], 1).numpy(), np.full(T, pma[b]), win)
            _check("%s attention" % ("split" if tp else "fp32"), R[b], a["R"], a["S"], tau, "attention b %d win %d" % (b, win))
            sure = a["margin"] > 4 * tau * a["Sp"]
            assert np.array_equal(M[b][sure], a["argmax"][sure]), b
    finally:
        e.set_tensor_path(1)


# ---------------------------------------------------------------------------------------------- the aid itself
def test_history_refuses_stale_state(eng):
    """decode_history reads a generation's buffers only while nothing else has written them, and launches nothing."""
    e = eng
    L = _texts(2, e.hp.max_N, 3)
    e.text2mel_generate(L, steps=12)
    before = e.launch_count()
    t, joined = e.decode_history("audiodec", 0)
    assert t.shape == (2, e.hp.max_T, e.hp.d) and not joined
    assert e.launch_count() == before
    stale = [lambda: e.text2mel_generate(L, steps=12, want_final_attention=True),
             lambda: e.text2mel_forward(L, torch.zeros(2, e.hp.max_T, e.hp.n_mels), np.zeros(2, np.int32)),
             lambda: e.textenc(L)]
    for writer in stale:
        e.text2mel_generate(L, steps=12)
        e.decode_history("Y")
        writer()
        before = e.launch_count()
        for what in ("audioenc", "audiodec", "R", "KV", "Y", "windows"):
            with pytest.raises(DcttsError, match="do not hold a generation"):
                e.decode_history(what)
        assert e.launch_count() == before
    e.text2mel_generate_path(L, np.zeros((2, 10), np.int64))
    e.decode_history("R")
    with pytest.raises(DcttsError, match="no block %d" % len(DEC_L)):
        e.decode_history("audiodec", len(DEC_L))


def test_history_refuses_after_a_workspace_growth(side_engine, params):
    e = side_engine(params)
    e.text2mel_generate(_texts(2, e.hp.max_N, 3), steps=5)
    e.decode_history("audioenc", 3)
    e.reserve(3)                                   # reallocates the decode's buffers
    with pytest.raises(DcttsError, match="do not hold a generation"):
        e.decode_history("audioenc", 3)


def test_joined_planes_on_the_tensor_path(eng):
    """The graph-per-frame decode at B >= 8 on the tensor path keeps C_1, HC_2 and HC_3 of AudioDec as planes only."""
    e = eng
    _mode(e, 0, 1)
    e.text2mel_generate(_texts(8, e.hp.max_N, 1), steps=4)
    assert [e.decode_history("audiodec", i)[1] for i in range(len(DEC_L))] == [True] * 3 + [False] * (len(DEC_L) - 3)
    _mode(e, 0, 0)
    e.text2mel_generate(_texts(8, e.hp.max_N, 1), steps=4)
    assert not any(e.decode_history("audiodec", i)[1] for i in range(len(DEC_L)))
