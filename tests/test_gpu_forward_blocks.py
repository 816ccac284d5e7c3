"""The full-sequence networks one block at a time: after a call, every block's output rows (Engine.chain_history) are
checked against the float64 reference of that block (tests/ref_forward_blocks.py) computed on that block's input rows as
the chain left them, so that each block is held to its own rounding: |got - ref| <= tau S, with one tau per kernel set
(DESIGN.md, "The full-sequence networks one block at a time").

The fp32 path's routes, from launch_conv_gemm and launch_ln_rows (csrc/kernels_simt.cu), for M = B L rows of a launch and
ldw columns (256 for a d-wide conv1d, 512 for a highway block's two halves; SSRN: 512, 1024, 1040 and 1032):
  M <= 256: the split-K skinny GEMM, its partials summed in the LayerNorm (B = 1 at L <= 210, B = 3 at L = 64);
  else 128-row tiles when ceil(M / 128) ceil(ldw / 128) >= 120, 64-row tiles below: B = 3, L = 210 (630 rows) and
  B = 5, L = 210 (1050) take 64-row tiles at 256 and 512 columns; B = 32, L = 210 (6720) 128-row tiles at 512 columns
  and 64-row tiles at 256; B = 36, L = 210 (7560 rows, 60 row tiles) 128-row tiles at 256 columns too;
  ln_row_cta_kernel at C <= 256 and M <= 1024 rows, ln_rows_kernel<8 | 16 | 32 | 33 | 65> otherwise (by C), with
  2 warps per CTA below 2048 rows (C = 256 at 1050 rows: ln_rows_kernel<8>) and 8 from 2048 on.
"""
import numpy as np
import pytest
import torch

import ref_decode_blocks as rb
import ref_forward_blocks as rf
from dc_tts_b200.arch import NETWORKS, textenc_layers
from dc_tts_b200.engine import DcttsError, Engine
from dc_tts_b200.hyperparams import Hyperparams
from dc_tts_b200.params import init_params

pytestmark = pytest.mark.gpu

NETS = {"textenc": "Text2Mel/TextEnc", "audioenc": "Text2Mel/AudioEnc", "audiodec": "Text2Mel/AudioDec", "ssrn": "SSRN"}
TAU = {1: rf.TAU_TC, 0: rf.TAU_FP32}
WORST = {}                       # group -> worst err / S seen (printed at the end of the module, recorded in DESIGN.md)
EDGE = (0, 1, 63, 64, 126, 127, 128, 129, 255, 256, 383, 384, 511, 512, 639, 640, 767, 768)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nforward blocks, worst err / S: " + ", ".join("%s %.3g" % kv for kv in sorted(WORST.items())))


def _check(group, got, ref, S, tau, what):
    got = np.asarray(got, np.float64)
    err = np.abs(got - ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(S > 0, err / S, np.where(err > 0, np.inf, 0.0))
    r = np.where(np.isnan(r), np.inf, r)                 # a NaN anywhere fails
    worst = float(r.max()) if r.size else 0.0
    WORST[group] = max(WORST.get(group, 0.0), worst)
    if worst > tau:
        i = np.unravel_index(int(np.argmax(r)), r.shape)
        raise AssertionError("%s: err / S = %.3g > tau = %.3g at %s (got %r, ref %r, S %.3g)"
                             % (what, worst, tau, i, got[i], ref[i], S[i]))


@pytest.fixture
def eng(engine):
    engine.set_option("chain_history", 1)
    yield engine
    engine.set_option("chain_history", 0)
    for o, v in (("tc_occ2", 0), ("tc_mcast", 1), ("tc_resid_tma", 1), ("fused_ln", 0)):
        engine.set_option(o, v)
    engine.set_tensor_path(1)


@pytest.fixture
def side_engine():
    """Handles of a test's own (parameter sets, hyperparameters) with the history on, closed at its end."""
    made = []

    def make(P, H=Hyperparams):
        e = Engine(0, hparams=H)
        e.load_params(P)
        e.set_option("chain_history", 1)
        made.append(e)
        return e
    yield make
    for e in made:
        e.close()


_PRM = {}


def _prm(P, net, layers):
    key = (id(P), net, len(layers), layers[-1].cout)
    if key not in _PRM:                                  # P is kept with its blocks, so that its id stays unique
        _PRM[key] = (P, [rf.block_params(P, NETS[net], l) for l in layers])
    return _PRM[key][1]


def _joined(x):
    return sum(p.astype(np.float32) for p in rf.split_f16(x))


def _embedded(P, L):
    """TextEnc's input: the embedding rows of the ids, row 0 of the table read as zeros (modules.py:36-38)."""
    table = np.array(P["Text2Mel/TextEnc/embed_1/lookup_table"], np.float32)
    table[0] = 0
    return table[np.asarray(L)]


def check_chain(e, P, net, tp, lengths=None, utts=None, edge_utts=(), extra_shift=0, layers=None, group=None, x_in=None):
    """Every block of the last chain of `net` on the engine: utterances `utts` on all their live rows, `edge_utts` on the
    tile-edge rows only; with `lengths` (ragged), utterance b's block i on its own live rows, and every row past them exactly 0.
    x_in: the network input the caller passed (TextEnc: the embedding rows), which the first block's recorded input must
    be: bit for bit on the fp32 path; on the tensor path the joined split planes, of x times the utterance's power-of-two
    scale and times its inverse for a network input (rows past the lengths 0), of the rows themselves for TextEnc.
    Returns the blocks' outputs."""
    layers = layers or NETWORKS[NETS[net]]()
    prm = _prm(P, net, layers)
    x, joined_in = e.chain_history(net, 0, "input")
    assert joined_in == (tp == 1), (net, joined_in)
    x = x.cpu().numpy()
    if x_in is not None:
        x_in = np.asarray(x_in.cpu() if isinstance(x_in, torch.Tensor) else x_in, np.float32)
        want = x_in if tp == 0 else (_joined(x_in) if net == "textenc" else rf.input_planes(x_in, lengths))
        bad = np.argwhere(x != want)
        assert not bad.size, "%s tp %d: the first block's input differs from the caller's at %s (%r, want %r)" % (
            net, tp, bad[0], x[tuple(bad[0])], want[tuple(bad[0])])
    B, L = x.shape[0], x.shape[1]
    n = list(lengths) if lengths is not None else [L] * B
    utts = range(B) if utts is None else utts
    tau = TAU[tp]
    group = group or ("tc" if tp else "fp32")
    outs = []
    for i, l in enumerate(layers):
        t, joined = e.chain_history(net, i, "output")
        out = t.cpu().numpy()
        assert joined == (tp == 1 and i + 1 < len(layers)), (net, i, joined)
        for b in list(utts) + [u for u in edge_utts if u not in utts]:
            ins, live = rf.live_rows(layers, n[b])
            rows = np.arange(live[i]) if b in utts else np.array([r for r in EDGE if r < live[i]] + [live[i] - 1])
            ref, S = rf.block_rows(prm[i], l, x[b, :ins[i]], rows, extra_shift if i == 0 else 0)
            if joined:
                S = S + rf.S_PLANES
            _check(group, out[b, rows], ref, S, tau, "%s tp %d utt %d %s (L %d)" % (net, tp, b, l.scope, n[b]))
            if lengths is not None:
                assert not out[b, live[i]:].any(), "%s utt %d %s: rows past %d not zero" % (net, b, l.scope, live[i])
        outs.append(out)
        x = out
    return outs


def _mels(B, T, seed, levels=None):
    Y = np.random.default_rng(seed).uniform(0, 1, (B, T, 80)).astype(np.float32)
    if levels is not None:
        Y *= np.asarray(levels, np.float32)[:, None, None]
    return Y


def _texts(B, N, seed):
    L = np.zeros((B, N), np.int32)
    for b in range(B):
        rng = np.random.default_rng([seed, b])
        n = min(N - 1, 5 + (53 * b + seed) % (N - 5))
        L[b, :n] = rng.integers(2, 32, size=n)
        L[b, n] = 1
    return L


def _sigmoid_check(tp, logits, Z, utts, what):
    for b in utts:
        y, S = rb.mel_sigmoid(logits[b])
        _check("tc" if tp else "fp32", Z[b], y, S, TAU[tp], what + " sigmoid utt %d" % b)


def _utts(B):
    """All utterances of a small batch; of a larger one the first and last on all rows, the rest on the tile edges."""
    return (list(range(B)), ()) if B <= 3 else ([0, B - 1], tuple(range(1, B - 1)))


TP = pytest.mark.parametrize("tp", [1, 0], ids=["tc", "fp32"])


# ---------------------------------------------------------------------------------------------- each network alone
@TP
@pytest.mark.parametrize("B,T", [(1, 1), (1, 127), (3, 128), (3, 129), (3, 210), (5, 210), (32, 210), (36, 210)])
def test_audioenc_audiodec(eng, params, tp, B, T):
    eng.set_tensor_path(tp)
    u, edge = _utts(B)
    mels = _mels(B, T, 10 * B + T)
    eng.audioenc(mels)
    check_chain(eng, params, "audioenc", tp, utts=u, edge_utts=edge, x_in=mels)
    R = torch.randn(B, T, 2 * eng.hp.d, generator=torch.Generator().manual_seed(T))
    logits, Y = eng.audiodec(R)
    outs = check_chain(eng, params, "audiodec", tp, utts=u, edge_utts=edge, x_in=R)
    assert np.array_equal(outs[-1], logits.cpu().numpy())
    _sigmoid_check(tp, outs[-1], Y.cpu().numpy(), u, "AudioDec")


@TP
@pytest.mark.parametrize("B,T", [(1, 1), (1, 32), (3, 64), (1, 210), (32, 210)])
def test_ssrn(eng, params, tp, B, T):
    eng.set_tensor_path(tp)
    u, edge = _utts(B)
    mels = _mels(B, T, 7 * B + T)
    logits, Z = eng.ssrn(mels)
    outs = check_chain(eng, params, "ssrn", tp, utts=u, edge_utts=edge, x_in=mels)
    assert np.array_equal(outs[-1], logits.cpu().numpy())
    _sigmoid_check(tp, outs[-1], Z.cpu().numpy(), u, "SSRN")


@TP
@pytest.mark.parametrize("B", [1, 3, 32])
def test_textenc(eng, params, tp, B):
    eng.set_tensor_path(tp)
    u, edge = _utts(B)
    L = _texts(B, eng.hp.max_N, B)
    K, V = eng.textenc(L)
    outs = check_chain(eng, params, "textenc", tp, utts=u, edge_utts=edge, x_in=_embedded(params, L))
    d = eng.hp.d
    assert np.array_equal(outs[-1][..., :d], K.cpu().numpy()) and np.array_equal(outs[-1][..., d:], V.cpu().numpy())


@TP
@pytest.mark.parametrize("B", [1, 3])
def test_text2mel_forward(eng, params, tp, B):
    """text2mel_forward's front (TextEnc, AudioEnc on the mels read one frame back, the dense attention) and AudioDec
    reading R: on the tensor path through the attention's split planes, which must be the split of R bit for bit.  The
    attention runs under the monotonic windows at prev_max_attentions, at the text's start, middle and last key."""
    eng.set_tensor_path(tp)
    e, T, d, N = eng, eng.hp.max_T, eng.hp.d, eng.hp.max_N
    pma = np.array([0, N // 2, N - 1])[:B]
    mels = _mels(B, T, B)
    Y, M, A = e.text2mel_forward(_texts(B, N, 3 + B), mels, pma)
    check_chain(e, params, "audioenc", tp, extra_shift=-1, x_in=mels)
    outs = check_chain(e, params, "audiodec", tp)
    _sigmoid_check(tp, outs[-1], Y.cpu().numpy(), range(B), "text2mel_forward Y")
    R = e.chain_history("attention")[0].cpu().numpy()
    Rin, joined = e.chain_history("audiodec", 0, "input")
    assert joined == (tp == 1)
    if tp == 1:
        hi, lo = rf.split_f16(R)
        assert np.array_equal(Rin.cpu().numpy(), hi.astype(np.float32) + lo.astype(np.float32))
    else:
        assert np.array_equal(Rin.cpu().numpy(), R)
    KV = e.chain_history("textenc", len(textenc_layers()) - 1)[0].cpu().numpy()
    Q = e.chain_history("audioenc", len(NETWORKS[NETS["audioenc"]]()) - 1)[0].cpu().numpy()
    _check_attention(tp, Q, KV, R, A.cpu().numpy(), M.cpu().numpy(), pma, e.hp.attention_win_size, "text2mel_forward")
    L_emb = _embedded(params, _texts(B, N, 3 + B))
    check_chain(e, params, "textenc", tp, x_in=L_emb)


def _check_attention(tp, Q, KV, R, A, M, pma=None, win=None, what=""):
    """R (B, T, 2d), A (B, N, T) and the argmax M (B, T) of every utterance against the float64 attention of its Q and KV."""
    tau = rf.TAU_ATTN_TC if tp else rf.TAU_ATTN_FP32
    tau_a = rf.TAU_ATTN_TC_A if tp else rf.TAU_ATTN_FP32_A
    grp = "attn " + ("tc" if tp else "fp32")
    for b in range(len(Q)):
        a = rf.dense_attention(Q[b], KV[b], None if pma is None else pma[b], win)
        _check(grp, R[b], a["R"], a["S"], tau, "%s R utt %d" % (what, b))
        _check(grp + " A", A[b].T, a["A"], a["SA"], tau_a, "%s A utt %d" % (what, b))
        sure = a["margin"] > 4 * tau * a["Sp"]
        assert np.array_equal(M[b][sure], a["argmax"][sure]), (what, b)


@TP
def test_text2mel_align_front(eng, params, tp):
    """The aligner's front: TextEnc, AudioEnc on the recorded mels read one frame back, and the dense attention."""
    eng.set_tensor_path(tp)
    e, B, T = eng, 3, 150
    L, mels = _texts(B, e.hp.max_N, 21), _mels(B, T, 21)
    *_, A = e.text2mel_align(L, mels, want_alignments=True)
    check_chain(e, params, "textenc", tp, x_in=_embedded(params, L))
    check_chain(e, params, "audioenc", tp, extra_shift=-1, x_in=mels)
    R = e.chain_history("attention")[0].cpu().numpy()
    KV = e.chain_history("textenc", len(textenc_layers()) - 1)[0].cpu().numpy()
    Q = e.chain_history("audioenc", len(NETWORKS[NETS["audioenc"]]()) - 1)[0].cpu().numpy()
    A = A.cpu().numpy()
    _check_attention(tp, Q, KV, R, A, A.argmax(1), what="text2mel_align")
    with pytest.raises(DcttsError, match="no rows of AudioDec"):
        e.chain_history("audiodec", 0)


# ---------------------------------------------------------------------------------------------- ragged SSRN
def test_ragged_ssrn(eng, params):
    """Per-utterance lengths on the tensor path: lengths of 1 and L, and ones whose x2 and x4 rows end on a tile edge (32 ->
    128 rows, 64 -> 128 and 256, 127 -> 254 and 508); live rows within tau S of each utterance alone, rows past them 0."""
    eng.set_tensor_path(1)
    T = 210
    n = [1, T, 32, 64, 127, 33, 96, 160]
    mels = _mels(len(n), T, 5)
    logits, Z = eng.ssrn(mels, lengths=np.array(n))
    check_chain(eng, params, "ssrn", 1, lengths=n, utts=[0, 1, 2, 3], edge_utts=(4, 5, 6, 7), x_in=mels)


def test_ragged_ssrn_fp32_is_refused(eng):
    """On the fp32 kernels the ragged chain runs once per utterance: the aid refuses rather than stitch them."""
    eng.set_tensor_path(0)
    eng.ssrn(_mels(2, 16, 1), lengths=np.array([3, 16]))
    before = eng.launch_count()
    with pytest.raises(DcttsError, match="once per utterance"):
        eng.chain_history("ssrn", 0)
    assert eng.launch_count() == before


# ---------------------------------------------------------------------------------------------- levels and LayerNorm edges
@TP
def test_input_levels_in_one_batch(eng, params, tp):
    """Silence at 1e-8, 1e-3 and 1 in one batch: each utterance's first block held to its own S (per-utterance in_inv)."""
    eng.set_tensor_path(tp)
    lv = [1e-8, 1e-3, 1.0]
    mels = _mels(3, 40, 2, lv)
    eng.ssrn(mels)
    check_chain(eng, params, "ssrn", tp, x_in=mels)
    mels = _mels(3, 130, 3, lv)
    eng.audioenc(mels)
    check_chain(eng, params, "audioenc", tp, x_in=mels)


def _const_params(P, value, near=False):
    """A zero kernel (or the kernel times 1e-6) and a constant bias in SSRN HC_2 and C_10 and AudioEnc C_2 and HC_4."""
    Q = dict(P)
    for s in ("SSRN/HC_2", "SSRN/C_10", "Text2Mel/AudioEnc/C_2", "Text2Mel/AudioEnc/HC_4"):
        Q[s + "/conv1d/kernel"] = (P[s + "/conv1d/kernel"] * np.float32(1e-6)) if near else np.zeros_like(P[s + "/conv1d/kernel"])
        Q[s + "/conv1d/bias"] = np.full_like(P[s + "/conv1d/bias"], value)
    return Q


@pytest.mark.parametrize("scheme", ["const0.75", "const1e3", "near_const", "tf_default"])
def test_layernorm_edges(side_engine, params, scheme):
    """Exact rows of beta from a zero kernel with a constant bias; the same kernel times 1e-6 (large kappa); the reference
    initialisers, where TextEnc's padding rows and AudioEnc's row 0 are exact."""
    if scheme == "tf_default":
        P = init_params(0, "tf_default")
    else:
        P = _const_params(params, 0.75 if scheme != "const1e3" else 1e3, near=scheme == "near_const")
    e = side_engine(P)
    for tp in (1, 0):
        e.set_tensor_path(tp)
        e.ssrn(_mels(3, 50, 4))
        ss = check_chain(e, P, "ssrn", tp)
        e.audioenc(_mels(2, 129, 6))
        ae = check_chain(e, P, "audioenc", tp)
        if scheme in ("const0.75", "const1e3"):
            # exactly beta (relu'd in C_2); on the tensor path the hidden rows are kept as planes: hi + lo of beta
            for got, beta in ((ae[1], np.maximum(P["Text2Mel/AudioEnc/C_2/normalize/beta"], 0)),
                              (ss[9], P["SSRN/C_10/normalize/beta"])):
                want = sum(p.astype(np.float32) for p in rf.split_f16(beta)) if tp else beta
                assert (got == want).all(), tp
        if scheme == "tf_default":
            L = _texts(3, e.hp.max_N, 1)
            e.textenc(L)
            te = check_chain(e, P, "textenc", tp)
            e.text2mel_forward(L, _mels(3, e.hp.max_T, 2), np.zeros(3, np.int32))
            ae = check_chain(e, P, "audioenc", tp, extra_shift=-1)
            for i in range(len(ae)):
                assert not ae[i][:, 0].any(), (tp, i)       # row 0 reads zeros: beta = 0 exactly
            pad = int((L[0] != 0).sum()) + 83                # past TextEnc's receptive field: 2 (1 + 3 + 9 + 27) + 2 rows
            assert not te[-1][0, pad:].any(), tp


# ---------------------------------------------------------------------------------------------- options and sizes
@pytest.mark.parametrize("opt", ["tc_occ2", "tc_mcast", "tc_resid_tma"])
def test_block_kernel_options(eng, params, opt):
    eng.set_tensor_path(1)
    for v in (0, 1):
        eng.set_option(opt, v)
        eng.ssrn(_mels(32, 64, 8))
        check_chain(eng, params, "ssrn", 1, utts=[0], edge_utts=(13, 31))
        eng.audioenc(_mels(32, 210, 9))
        check_chain(eng, params, "audioenc", 1, utts=[0], edge_utts=(17, 31))


@pytest.mark.parametrize("fused", [0, 1])
def test_fused_ln(eng, params, fused):
    """fp32 path, GEMM and LayerNorm in one launch where the launch is skinny (M <= 256, C <= 256)."""
    eng.set_tensor_path(0)
    eng.set_option("fused_ln", fused)
    eng.audioenc(_mels(1, 200, 11))
    check_chain(eng, params, "audioenc", 0)
    eng.audiodec(torch.randn(2, 100, 2 * eng.hp.d, generator=torch.Generator().manual_seed(2)))
    check_chain(eng, params, "audiodec", 0)


@pytest.mark.parametrize("F,sr", [(513, 16000), (2049, 44100)])
def test_ssrn_widths(side_engine, F, sr):
    """F = 513 and F = 2049 (the 144-column, 16-CTA-cluster instantiation and ln_rows_kernel<65>)."""
    from dc_tts_b200.arch import ssrn_layers
    from sample_rates import at_rate
    with at_rate(sr) as H:
        P = init_params(0, "perturbed")
        e = side_engine(P, H)
        layers = ssrn_layers()
        assert layers[-1].cout == F
        for tp in (1, 0):
            e.set_tensor_path(tp)
            e.ssrn(_mels(3, 40, F))
            check_chain(e, P, "ssrn", tp, layers=layers, utts=[0, 2], edge_utts=(1,))


def test_textenc_long_text(side_engine, params):
    e = side_engine(params, type("H300", (Hyperparams,), {"max_N": 300}))
    for tp in (1, 0):
        e.set_tensor_path(tp)
        L = _texts(2, 300, 299)
        e.textenc(L)
        check_chain(e, params, "textenc", tp, x_in=_embedded(params, L))


# ---------------------------------------------------------------------------------------------- dense attention
@pytest.mark.parametrize("tp", [1, 0], ids=["tc", "fp32"])
def test_dense_attention(eng, tp):
    """Engine.attention(monotonic=False) on both kernels at key counts around the tensor kernel's 64-key blocks and query
    counts around its tiles; R, A and the argmax against the float64 attention."""
    eng.set_tensor_path(tp)
    tau = rf.TAU_ATTN_TC if tp else rf.TAU_ATTN_FP32
    tau_a = rf.TAU_ATTN_TC_A if tp else rf.TAU_ATTN_FP32_A
    grp = "attn " + ("tc" if tp else "fp32")
    d = eng.hp.d
    g = torch.Generator().manual_seed(1)
    for N in (1, 63, 64, 65, 180, 192, 193, 300):
        for T in ((1, 63, 64, 65, 210) if N in (65, 193) else (65,)):
            Q, K, V = (torch.randn(2, n, d, generator=g) for n in (T, N, N))
            R, A, M = eng.attention(Q, K, V)
            for b in range(2):
                a = rf.dense_attention(Q[b].numpy(), torch.cat([K[b], V[b]], 1).numpy())
                _check(grp, R[b].cpu().numpy(), a["R"], a["S"], tau, "R N %d T %d" % (N, T))
                _check(grp + " A", A[b].T.cpu().numpy(), a["A"], a["SA"], tau_a, "A N %d T %d" % (N, T))
                sure = a["margin"] > 4 * tau * a["Sp"]
                assert np.array_equal(M[b].cpu().numpy()[sure], a["argmax"][sure]), (N, T)


@pytest.mark.parametrize("tp", [1, 0], ids=["tc", "fp32"])
def test_dense_attention_saturated_and_duplicated(eng, tp):
    """Scores of +-hundreds (one key takes all the mass); exactly duplicated best keys in the same 64-key block and in
    different ones: the argmax is the first of them, as numpy's."""
    eng.set_tensor_path(tp)
    tau = rf.TAU_ATTN_TC if tp else rf.TAU_ATTN_FP32
    d, N, T = eng.hp.d, 180, 70
    g = torch.Generator().manual_seed(5)
    Q, K, V = torch.randn(3, T, d, generator=g), torch.randn(3, N, d, generator=g), torch.randn(3, N, d, generator=g)
    Q[0] *= 40                                                    # saturated: scores of several hundred
    for b, (i, j) in ((1, (10, 20)), (2, (40, 150))):
        K[b, :] *= 0.01
        K[b, i] = K[b, j] = Q[b].mean(0) * 50                     # two identical winning keys
    R, A, M = eng.attention(Q, K, V)
    for b in range(3):
        a = rf.dense_attention(Q[b].numpy(), torch.cat([K[b], V[b]], 1).numpy())
        _check("attn " + ("tc" if tp else "fp32"), R[b].cpu().numpy(), a["R"], a["S"], tau, "saturated/duplicate b %d" % b)
        if b:
            win = M[b].cpu().numpy()
            top = a["A"].max(1) > 0.45                            # the two copies share the mass
            assert top.sum() > T // 2 and (win[top] == {1: 10, 2: 40}[b]).all(), (b, win[top])
        else:
            sure = a["margin"] > 4 * tau * a["Sp"]
            assert sure.sum() > T // 2 and np.array_equal(M[b].cpu().numpy()[sure], a["argmax"][sure])


# ---------------------------------------------------------------------------------------------- the aid itself
def test_history_refuses_stale_state(eng, params):
    e = eng
    Y = _mels(2, 20, 0)
    L = _texts(2, e.hp.max_N, 3)
    stale = {"a decode": lambda: e.text2mel_generate(L, steps=4),
             "op-level block": lambda: e.hc("SSRN/HC_2", torch.zeros(1, 4, e.hp.c)),
             "op-level attention": lambda: e.attention(*(torch.zeros(1, 4, e.hp.d) for _ in range(3))),
             "ran no full-sequence chain": lambda: e.audioenc(Y)}
    for why, writer in stale.items():
        e.ssrn(Y)
        e.chain_history("ssrn", 3)
        writer()
        before = e.launch_count()
        with pytest.raises(DcttsError, match=why):
            e.chain_history("ssrn", 3)
        with pytest.raises(DcttsError, match=why):
            e.chain_history("ssrn", 0, "input")
        assert e.launch_count() == before
    e.set_option("chain_history", 0)
    e.ssrn(Y)
    with pytest.raises(DcttsError, match="option chain_history was off"):
        e.chain_history("ssrn", 0)
    e.set_option("chain_history", 1)
    e.ssrn(Y, want_logits=False)
    e.chain_history("ssrn", 14)
    with pytest.raises(DcttsError, match="kept no output of block 15"):
        e.chain_history("ssrn", 15)
    with pytest.raises(DcttsError, match="only the first block's input"):
        e.chain_history("ssrn", 1, "input")


def test_history_refuses_after_the_weights_change(side_engine, params):
    """A training workspace takes the handle's weights over (the optimiser may change them): older records refuse."""
    e = side_engine(params)
    e.audiodec(torch.zeros(1, 8, 2 * e.hp.d))
    e.chain_history("audiodec", 2)
    e.train_init(1, 0.0)
    with pytest.raises(DcttsError, match="training took over the weights"):
        e.chain_history("audiodec", 2)


def test_history_refuses_after_a_workspace_growth(side_engine, params):
    e = side_engine(params)
    e.audiodec(torch.zeros(1, 8, 2 * e.hp.d))
    e.chain_history("audiodec", 2)
    e.reserve(4)
    with pytest.raises(DcttsError, match="workspace grew"):
        e.chain_history("audiodec", 2)


@TP
def test_option_changes_nothing(eng, tp):
    """The same launches and the same bits with the history on and off."""
    eng.set_tensor_path(tp)
    L, mels = _texts(2, eng.hp.max_N, 8), _mels(2, eng.hp.max_T, 8)
    res = {}
    for on in (0, 1):
        eng.set_option("chain_history", on)
        c0 = eng.launch_count()
        Y, M, A = eng.text2mel_forward(L, mels, np.zeros(2, np.int32))
        lg, Z = eng.ssrn(Y, lengths=np.array([100, 210]) if tp else None)
        torch.cuda.synchronize()
        res[on] = (eng.launch_count() - c0, [t.cpu().numpy() for t in (Y, M, A, lg, Z)])
    assert res[0][0] == res[1][0]
    for a, b in zip(res[0][1], res[1][1]):
        assert np.array_equal(a, b)
