"""GPU parity on quiet and silent inputs.  The other parity tests draw inputs from uniform(0, 1) or uniform(-1, 1); real
inputs are not like that: normalised mels sit at the 1e-8 floor on silence (get_spectrograms clips there, reference
utils.py:59-60), a trained Text2Mel emits sigmoid outputs near 0 there, and the reference initialisers (scheme
"tf_default") give zero biases, so a first block's conv output comes from the input alone and LayerNorm magnifies
whatever the input planes lost.  On the tensor-core path a network input is carried in per-utterance power-of-two
scaled split-fp16 planes (kernels_tc.cu, f32_to_planes_scaled_kernel); these tests hold both kernel sets to the same
tolerances as the uniform-input tests, against the fp64 numpy oracle."""
import numpy as np
import pytest
import torch

from dc_tts_b200 import arch
from dc_tts_b200.hyperparams import Hyperparams as hp
from dc_tts_b200.params import init_params, synthetic_text
from oracle import ref_features as rf
from oracle import ref_numpy as rn
from oracle import ref_torch as rt

pytestmark = pytest.mark.gpu
BLOCK_TOL = 2e-4
NET_TOL = 1e-3
FLOOR = 1e-8                      # get_spectrograms' clip floor
LEVELS = ["floor", "1e-6", "1e-5", "1e-4", "1e-3", "1", "zero", "one_loud", "rows_mixed", "batch_mixed"]


@pytest.fixture(scope="module")
def tf_params():
    return init_params(0, "tf_default")


@pytest.fixture(scope="module")
def tf_engine(tf_params):
    """A second engine with the reference initialisers committed; the session `engine` stays the default one."""
    from dc_tts_b200.engine import Engine
    e = Engine(0)
    e.load_params(tf_params)
    yield e
    e.close()


@pytest.fixture(params=["tf_default", "perturbed"])
def weights(request):
    return request.param


@pytest.fixture(params=[0, 1], ids=["fp32path", "tensorpath"])
def tensor_path(request):
    return request.param


@pytest.fixture
def eng(request, weights, tensor_path):
    """(engine, params) with the weights of `weights`, running the kernel set of `tensor_path`."""
    if weights == "tf_default":
        e, P = request.getfixturevalue("tf_engine"), request.getfixturevalue("tf_params")
    else:
        e, P = request.getfixturevalue("engine"), request.getfixturevalue("params")
    e.set_tensor_path(tensor_path)
    yield e, P
    e.set_tensor_path(1)


def quiet_input(kind, B, L, C, seed, signed=False):
    """Deterministic (B, L, C) float32 inputs at the levels silence produces.  Levels "1e-6" ... "1" are level *
    uniform(0, 1) (uniform(-1, 1) when `signed`), kept at or above the floor like a clipped mel; "floor" is the floor
    exactly; "one_loud" is the floor with one loud channel in one row; "rows_mixed" cycles every level row by row inside
    each utterance; "batch_mixed" alternates loud and silent utterances in one batch."""
    rng = np.random.default_rng([seed, B, L, C])

    def at(level, shape):
        u = rng.uniform(-1, 1, shape) if signed else rng.uniform(0, 1, shape)
        x = level * u
        return x if signed else np.maximum(x, FLOOR)

    if kind == "floor":
        x = np.full((B, L, C), FLOOR)
    elif kind == "zero":
        x = np.zeros((B, L, C))
    elif kind == "one_loud":
        x = np.full((B, L, C), FLOOR)
        x[:, L // 2, 3] = 1.0
    elif kind == "rows_mixed":
        levels = [FLOOR, 1e-6, 1e-5, 1e-4, 1e-3, 1.0, 0.0]
        x = np.stack([at(levels[t % len(levels)], (B, C)) for t in range(L)], 1)
        x[:, 6::len(levels)] = 0.0
        x[:, 0::len(levels)] = FLOOR
    elif kind == "batch_mixed":
        levels = [1.0, FLOOR, 1e-5, 1.0, 1e-6, 1e-4]
        x = np.stack([at(levels[b % len(levels)], (L, C)) for b in range(B)])
        x[1::len(levels)] = FLOOR
    else:
        x = at(float(kind), (B, L, C))
    return x.astype(np.float32)


def speech_mels(B, T, seed):
    """(B, T, n_mels) like a Text2Mel output: silent lead-in and tail at the floor, a pause at 1e-5 and voiced frames
    (uniform(0.05, 1)) between, positions varying per utterance."""
    rng = np.random.default_rng([seed, B, T])
    Y = np.empty((B, T, hp.n_mels))
    for b in range(B):
        y = rng.uniform(0.05, 1.0, (T, hp.n_mels))
        lead, tail = 2 + (3 * b) % (T // 6), 2 + (5 * b) % (T // 6)
        y[:lead] = FLOOR
        y[T - tail:] = FLOOR
        p0 = T // 2 - (b % 4)
        y[p0:p0 + max(2, T // 10)] = 1e-5 * rng.uniform(0, 1, (max(2, T // 10), hp.n_mels))
        Y[b] = y
    return Y.astype(np.float32)


def _layer(net, scope):
    for l in arch.NETWORKS[net]():
        if l.scope == scope:
            return l
    raise KeyError(scope)


def _maxerr(a, b):
    return float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max())


_REF = {}


def _ref(P, fn, *args):
    """fp64 oracle result, computed once per parameter set and input (both kernel sets compare with it)."""
    key = (id(P), fn.__name__) + tuple(a.tobytes() if isinstance(a, np.ndarray) else a for a in args)
    if key not in _REF:
        _REF[key] = fn(P, *[a.astype(np.float64) if isinstance(a, np.ndarray) and a.dtype == np.float32 else a
                            for a in args])
    return _REF[key]


# ------------------------------------------------------------------------------------------------ first blocks
BLOCKS = [("Text2Mel/AudioEnc", "C_1", False), ("SSRN", "C_1", False), ("Text2Mel/AudioDec", "C_1", True)]


@pytest.mark.parametrize("B,L", [(2, 37), (3, 210)], ids=["B2L37", "B3L210"])
@pytest.mark.parametrize("kind", LEVELS)
@pytest.mark.parametrize("net,scope,signed", BLOCKS, ids=["%s/%s" % (n, s) for n, s, _ in BLOCKS])
def test_block_quiet_input(eng, net, scope, signed, kind, B, L, record_property):
    """The blocks that read a network input, through the op-level entry points, which carry these blocks' input in
    scaled planes on the tensor path as the chains do.  AudioDec/C_1 reads R = [A.V ; Q], signed."""
    e, P = eng
    l = _layer(net, scope)
    if kind == "batch_mixed":
        B = max(B, 6)
    x = quiet_input(kind, B, L, l.cin, seed=len(scope) + 7 * B, signed=signed)
    full = net + "/" + scope
    out = e.conv1d(full, x, l.cout, l.rate, l.pad == "CAUSAL", 1 if l.act == "relu" else 0).cpu().numpy()
    ref = _ref(P, rn.conv1d, x, full, l.rate, l.pad, l.act)
    err = _maxerr(out, ref)
    record_property("max_abs_err", err)
    assert out.shape == ref.shape and np.isfinite(out).all()
    assert err < BLOCK_TOL, err


@pytest.mark.parametrize("tp", [0, 1], ids=["fp32path", "tensorpath"])
def test_ssrn_block_by_block_matches_chain_on_quiet_frames(engine, tp):
    """networks.py's SSRN composed from the op-level blocks agrees with the library's chain as closely as on uniform
    inputs (tests/test_gpu_blocks.py), also on frames at the silence floor: the op-level SSRN/C_1 scales its input
    planes as the chain does, and the hidden blocks carry theirs unscaled as the chain does."""
    from dc_tts_b200 import networks
    from dc_tts_b200.modules import variable_scope
    engine.set_tensor_path(tp)
    try:
        Y = speech_mels(2, 24, seed=8)
        with variable_scope("SSRN"):
            _, Z1 = networks.SSRN(Y, training=False, fused=True)
            _, Z2 = networks.SSRN(Y, training=False, fused=False)
    finally:
        engine.set_tensor_path(1)
    assert (Z1 - Z2).abs().max().item() < 1e-6


# ------------------------------------------------------------------------------------------------ networks
@pytest.mark.parametrize("B,T", [(1, 60), (32, 48)])
def test_ssrn_quiet_frames(eng, B, T, record_property):
    e, P = eng
    Y = speech_mels(B, T, seed=4)
    logits, Z = e.ssrn(Y)
    lr, Zr = _ref(P, rn.SSRN, Y)
    ez, el = _maxerr(Z.cpu().numpy(), Zr), _maxerr(logits.cpu().numpy(), lr)
    record_property("max_abs_err", ez)
    record_property("max_abs_err_logits", el)
    assert ez < NET_TOL and el < 5e-3, (ez, el)                          # logits are O(10)


@pytest.mark.parametrize("B,T", [(2, 210), (5, 37)])
def test_audioenc_quiet_frames(eng, B, T, record_property):
    e, P = eng
    S = speech_mels(B, T, seed=5)
    Q = e.audioenc(S).cpu().numpy()
    err = _maxerr(Q, _ref(P, rn.AudioEnc, S))
    record_property("max_abs_err", err)
    assert err < NET_TOL, err


def test_text2mel_forward_quiet_frames(eng, record_property):
    """One teacher-forced sess.run with mels that hold floor rows and a quiet pause.  The window argmax is compared on
    rows whose top-2 attention probabilities in fp64 differ by more than 1e-4 (a closer tie may flip on float32 noise)."""
    e, P = eng
    L = synthetic_text(2, 60, seed=0)
    mels = speech_mels(2, hp.max_T, seed=6)
    pma = np.array([5, 120], np.int32)
    Y, M, A = e.text2mel_forward(L, mels, pma)
    o = _ref(P, rn.text2mel_forward, L, mels, pma)
    err = _maxerr(Y.cpu().numpy(), o["Y"])
    record_property("max_abs_err", err)
    assert err < NET_TOL, err
    a = np.sort(o["alignments"].transpose(0, 2, 1), -1)                 # (B, T, N) fp64 probabilities
    ok = (a[..., -1] - a[..., -2]) > 1e-4
    assert ok.mean() > 0.5
    assert np.array_equal(M.cpu().numpy()[ok], o["max_attentions"][ok])
    assert _maxerr(A.cpu().numpy(), o["alignments"]) < 1e-4


def _speechlike_with_pause(seed, seconds=2.0):
    """tests/test_features.py's speech-like signal (quiet lead-in and tail) with an internal pause of amplitude 1e-5."""
    rng = np.random.default_rng(seed)
    n = int(hp.sr * seconds)
    t = np.arange(n) / hp.sr
    y = 0.3 * np.sin(2 * np.pi * 220 * t) * (0.5 + 0.5 * np.sin(2 * np.pi * 3 * t)) + 0.05 * rng.standard_normal(n)
    y[:3000] *= 1e-5
    y[n - 5000:] *= 1e-5
    y[n // 2:n // 2 + hp.sr // 4] *= 1e-5
    return y.astype(np.float32)


def test_features_of_a_pause_through_ssrn_and_audioenc(eng, record_property):
    """The mels the trainer and a trained model see: the oracle's get_spectrograms / load_spectrograms of a waveform
    with a pause (rows at exactly the 1e-8 floor) into SSRN and AudioEnc."""
    e, P = eng
    y = _speechlike_with_pause(0)
    mel_full, _ = rf.get_spectrograms(y)
    mel_r, _ = rf.load_spectrograms(y)
    assert (mel_full == np.float32(FLOOR)).all(-1).sum() >= 5           # the pause is at the floor
    Y = mel_r[None].astype(np.float32)
    _, Z = e.ssrn(Y, want_logits=False)
    ez = _maxerr(Z.cpu().numpy(), _ref(P, rn.SSRN, Y)[1])
    S = mel_full[None, :hp.max_T].astype(np.float32)
    eq = _maxerr(e.audioenc(S).cpu().numpy(), _ref(P, rn.AudioEnc, S))
    record_property("max_abs_err", max(ez, eq))
    assert ez < NET_TOL and eq < NET_TOL, (ez, eq)


# ------------------------------------------------------------------------------------------------ a quiet hidden layer
_QUIET_HIDDEN = ("limit of the format, not a defect: hidden activations are carried in unscaled planes, and with SSRN/C_1's "
                 "gamma times 1e-3 the input planes of HC_2 hold 1e-3-sized values, whose low plane is subnormal in fp16 "
                 "(about 14 significand bits left); Z is off by 2.2e-3 on an H100 (fp32 path: within 1e-3).  A trained "
                 "LayerNorm gain that small would need a scale on the hidden planes too")


@pytest.mark.parametrize("tp", [0, pytest.param(1, marks=pytest.mark.xfail(reason=_QUIET_HIDDEN, strict=True))],
                         ids=["fp32path", "tensorpath"])
def test_ssrn_quiet_hidden_layer(tf_params, tp, record_property):
    """Hidden activations are carried unscaled: they are LayerNorm outputs, O(1) per row.  With gamma of SSRN/C_1 scaled
    by 1e-3 (beta 0), the input planes of HC_2 hold 1e-3-sized values instead; this pins what that costs."""
    from dc_tts_b200.engine import Engine
    P = dict(tf_params)
    P["SSRN/C_1/normalize/gamma"] = (P["SSRN/C_1/normalize/gamma"] * 1e-3).astype(np.float32)
    e = Engine(0)
    try:
        e.load_params(P)
        e.set_tensor_path(tp)
        Y = speech_mels(2, 48, seed=7)
        _, Z = e.ssrn(Y, want_logits=False)
        err = _maxerr(Z.cpu().numpy(), rn.SSRN(P, Y.astype(np.float64))[1])
    finally:
        e.close()
    record_property("max_abs_err", err)
    assert err < NET_TOL, err


# ------------------------------------------------------------------------------------------------ decode paths
@pytest.mark.parametrize("decode_mode,B", [(1, 3), (0, 8)], ids=["cluster", "graph_b8"])
def test_generate_tf_default_vs_oracle(tf_engine, tf_params, decode_mode, B, record_property):
    """Free-running generation under the reference initialisers.  The persistent cluster kernel runs its GEMV on fp32 and
    the graph decode at B >= 8 runs AudioDec rows on wgmma from R planes written by the attention kernel: neither reads
    a converted network input, and both must match the oracle as on the perturbed weights.  Zero biases and random
    kernels leave the attention nearly uniform, so the argmax feedback ties within float32 noise from the first frames
    and a free-running oracle run drifts to another window.  Every generated frame j is therefore compared with the
    oracle's sess.run on the device's own prefix Y[:j] and window p_j (synthesize.py:48-54), and the next window with
    that run's argmax wherever its top-2 margin exceeds 1e-4."""
    tf_engine.set_tensor_path(1)
    tf_engine.set_option("decode_mode", decode_mode)
    steps = 24
    try:
        L = np.concatenate([synthetic_text(1, 30 + 17 * i, seed=40 + i) for i in range(B)])
        Y, Pg, _, _ = tf_engine.text2mel_generate(L, steps=steps)
    finally:
        tf_engine.set_option("decode_mode", 1)
    Yg, Pg = Y.cpu().numpy(), Pg.cpu().numpy()
    mels = np.zeros((steps, B, hp.max_T, hp.n_mels), np.float32)
    for j in range(steps):
        mels[j, :, :j] = Yg[:, :j]
    with torch.no_grad():
        K, V = rt.TextEnc(tf_params, L)
        o = rt.text2mel_forward(tf_params, np.tile(L, (steps, 1)), mels.reshape(steps * B, hp.max_T, hp.n_mels),
                                Pg[:, :steps].T.reshape(-1), KV=(K.repeat(steps, 1, 1), V.repeat(steps, 1, 1)))
    j = np.repeat(np.arange(steps), B)
    u = np.arange(steps * B)
    Yo = o["Y"].numpy()[u, j].reshape(steps, B, hp.n_mels)
    err = _maxerr(Yg[:, :steps].transpose(1, 0, 2), Yo)
    record_property("max_abs_err", err)
    assert err < NET_TOL, err
    a = o["alignments"].numpy()[u, :, j]                                # (steps * B, N): row j's probabilities
    top2 = np.sort(a, -1)[:, -2:]
    ok = (top2[:, 1] - top2[:, 0] > 1e-4).reshape(steps, B)[:-1]
    nxt = a.argmax(-1).reshape(steps, B)[:-1]
    assert np.array_equal(Pg[:, 1:steps].T[ok], nxt[ok])
