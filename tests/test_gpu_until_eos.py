"""Generation that ends each utterance at its text (Engine.text2mel_generate_until) on both decode paths.

The stop positions are taken from a full-length run's window trajectory, so that the lengths cover the first frame,
the middle, the last frames and "never".  Every row below an utterance's length must be that of the full-length run,
bit for bit: the loop is causal, and the engine's reordering by stop position only changes which utterances share a
decode cluster, which per-utterance arithmetic does not depend on (DESIGN §4, packing)."""
import numpy as np
import pytest
import torch

from dc_tts_b200.data_load import eos_positions, utterance_lengths
from dc_tts_b200.engine import DcttsError
from dc_tts_b200.hyperparams import Hyperparams as hp
from dc_tts_b200.params import init_params, synthetic_text

pytestmark = pytest.mark.gpu

TARGETS = [1, 2, 85, 86, 209, 210, None]          # None: a stop position the trajectory never reaches


@pytest.fixture
def until_engine(engine):
    engine.set_tensor_path(1)
    yield engine
    engine.set_option("decode_force_prepass", 0)
    engine.set_option("decode_mode", 1)


def _stop_positions(P, steps):
    """Per utterance, the stop position whose first frame is the available frame nearest to a target length: frame 0
    (stop position 0) or a frame at which the window moves."""
    m = P[:, 1:steps]                                                 # argmax of rows 0 .. steps - 2
    sp = np.zeros(len(P), np.int64)
    for b in range(len(P)):
        t = TARGETS[b % len(TARGETS)]
        if t is None:
            sp[b] = int(m[b].max()) + 1
            continue
        first = [0] + [j for j in range(1, m.shape[1]) if m[b, j] > m[b, j - 1]]
        j = min(first, key=lambda f: abs(f + 1 - t))
        sp[b] = 0 if j == 0 else int(m[b, j])
    return sp


def _cluster_frames(e, sp, lengths):
    """Frames the persistent decode executes: per cluster (consecutive utterances in stop-position order), its longest.
    Utterances per cluster as the engine picks them: the fewest (<= 5) that let every cluster be co-resident."""
    B, mc = len(sp), max(1, e.get_option("decode_max_clusters"))
    G = 1
    while G < 5 and -(-B // G) > mc:
        G += 1
    clusters = -(-B // G)
    assert e.decode_stats()[2] == clusters
    order = np.argsort(np.where(sp < 0, np.iinfo(np.int32).max, sp), kind="stable")
    return sum(int(lengths[order[c * G:(c + 1) * G]].max()) for c in range(clusters))


@pytest.mark.parametrize("mode", [1, 0], ids=["persistent", "graph"])
@pytest.mark.parametrize("B", [1, 5, 23, 32, 40])
def test_generate_until(until_engine, B, mode):
    e = until_engine
    if mode == 1 and not e.get_option("decode_available"):
        pytest.skip("no persistent decode on this device")
    e.set_option("decode_mode", mode)
    steps = hp.max_T
    L = np.concatenate([synthetic_text(1, 20 + (37 * i) % 150, seed=300 + i) for i in range(B)])
    seen = set()
    for force in ((0, 1) if mode == 1 else (0,)):
        e.set_option("decode_force_prepass", force)
        Yf, Pf, _, _ = e.text2mel_generate(L)
        Pf_np = Pf.cpu().numpy()
        sp = _stop_positions(Pf_np, steps)
        for tail in (0, 7):
            Y, P, n = e.text2mel_generate_until(L, stop_pos=sp, tail=tail)
            n = n.cpu().numpy()
            want = utterance_lengths(Pf_np[:, 1:steps], sp, tail, steps=steps)
            assert np.array_equal(n, want), (force, tail, n, want)
            seen.update(n.tolist())
            for b in range(B):
                k = int(n[b])
                assert torch.equal(Y[b, :k], Yf[b, :k]), (force, tail, b, k)
                assert torch.equal(P[b, :k], Pf[b, :k]), (force, tail, b, k)
                assert not Y[b, k:].any() and bool((P[b, k:] == -1).all()), (force, tail, b, k)
            frames = e.get_option("decode_last_frames")
            assert frames == (_cluster_frames(e, sp, n) if mode == 1 else steps), (force, tail, frames)
    if B >= 7:
        assert {1, 210} <= seen and len(seen) >= 6, sorted(seen)


def test_generate_until_eos_default_and_seeded_weights(until_engine):
    """stop_pos=None: the EOS positions of the texts.  Seeded (unperturbed) weights on a second engine."""
    from dc_tts_b200.engine import Engine
    e2 = Engine(0)
    try:
        e2.load_params(init_params(0))
        L = np.concatenate([synthetic_text(1, 8 + 3 * i, seed=500 + i) for i in range(12)])
        Yf, Pf, _, _ = e2.text2mel_generate(L)
        Y, P, n = e2.text2mel_generate_until(L)
        n = n.cpu().numpy()
        want = utterance_lengths(Pf.cpu().numpy()[:, 1:], eos_positions(L), 0, steps=hp.max_T)
        assert np.array_equal(n, want)
        assert (n < hp.max_T).any()                                  # short texts: some reach their EOS
        for b in range(len(L)):
            assert torch.equal(Y[b, :n[b]], Yf[b, :n[b]]) and not Y[b, n[b]:].any()
        if e2.get_option("decode_available"):
            # the per-cluster counters are summed before a larger batch reallocates their buffers
            e2.text2mel_generate_until(L[:2], stop_pos=[0, 0])       # two clusters of one utterance, one frame each
            e2.reserve(64)
            assert e2.get_option("decode_last_frames") == 2
            assert e2.decode_stats()[2] == 2
    finally:
        e2.close()


def test_generate_until_refuses(until_engine):
    e = until_engine
    L = synthetic_text(2, 30, seed=1)
    with pytest.raises(DcttsError):
        e.text2mel_generate_until(L, tail=-1)
    with pytest.raises(DcttsError):
        e.text2mel_generate_until(L, stop_pos=[3])
    import ctypes as C
    from dc_tts_b200.engine import _ptr
    Ld = e._i32(L)
    sp = e._i32(np.array([3, 3]))
    Y, P, n = e._empty(2, hp.max_T, hp.n_mels), e._empty(2, hp.max_T, dtype=torch.int32), e._empty(2, dtype=torch.int32)
    rc = e._lib.dctts_text2mel_generate_until(e._h, _ptr(Ld), 2, 0, _ptr(sp), -1, _ptr(Y), _ptr(P), _ptr(n), C.c_void_p(0))
    assert rc != 0 and b"tail" in e._lib.dctts_last_error(e._h)


def test_stepwise_loop_applies_the_same_rule(until_engine):
    """The reference's step-wise loop (sess.run per frame, full recompute) with the host rule applied to the fetched
    max_attentions after every frame, stopping once every utterance has ended: a second, independent implementation of
    the rule.  It ends every utterance at the frame generate_until_eos gives, with the same mel rows."""
    from dc_tts_b200.train import Graph, Session
    L = np.concatenate([synthetic_text(1, n, seed=900 + n) for n in (6, 9, 14)])
    g = Graph(mode="synthesize")
    Yd, _, nd = g.generate_until_eos(L)
    nd = nd.cpu().numpy()
    assert (nd < hp.max_T).any()
    sp = eos_positions(L)
    Y = np.zeros((len(L), hp.max_T, hp.n_mels), np.float32)
    M = np.zeros((len(L), hp.max_T), np.int64)
    pma = np.zeros((len(L),), np.int32)
    with Session() as sess:
        for j in range(hp.max_T):
            _Y, _M = sess.run([g.Y, g.max_attentions], {g.L: L, g.mels: Y, g.prev_max_attentions: pma})
            Y[:, j] = _Y[:, j]
            M[:, j] = _M[:, j]
            pma = _M[:, j].astype(np.int32)
            n = utterance_lengths(M[:, :j + 1], sp, 0, steps=hp.max_T)
            if (n <= j + 1).all():
                break
    assert np.array_equal(n, nd), (n, nd)
    for b, k in enumerate(n):
        Y[b, k:] = 0
    assert np.abs(Y - Yd.cpu().numpy()).max() < 1e-4
