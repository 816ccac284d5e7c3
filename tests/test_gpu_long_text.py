"""Texts longer than 192 characters: the attention kernels at any key count, and handles with hp.max_N = 300 through
TextEnc, the teacher-forced and free-running synthesis graph, synthesize() and the Text2Mel training step.  The
teacher-forced pass is checked against the reference's own graph at max_N = 300 (refshim_long_text.npz, generator
tests/golden/make_golden_refchecks_long.py, whose oracle checks are tests/test_long_text_reference.py).

The op-level cases run on the session engine (max_N = 180; dctts_attention takes any N) on both kernel sets.  The
network and training cases build engines of their own at max_N = 300: the module fixture `hp300` patches
Hyperparams.max_N, which the oracles and `Graph`-side helpers read, and restores it at teardown."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from dc_tts_b200 import trainer
from dc_tts_b200.hyperparams import Hyperparams
from dc_tts_b200.params import init_params, synthetic_bucket
from oracle import ref_torch as rt

import ref_train_bucket as rtb
from conftest import ROOT, golden

sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_golden_refchecks_long import synth_inputs, window_summary      # noqa: E402

pytestmark = pytest.mark.gpu
NET_TOL = 1e-3
LONG_N = 300


def _rand(shape, seed, lo=-1.0, hi=1.0):
    return np.random.default_rng(seed).uniform(lo, hi, shape).astype(np.float32)


def _windows(N):
    """Window starts at 0, at both sides of every 64-key block edge, and at N-3, N-2, N-1."""
    w = {0, N - 3, N - 2, N - 1}
    for e in range(64, N, 64):
        w.update((e - 1, e))
    return sorted(p for p in w if 0 <= p < N)


def _same_argmax(M, Mr, Ar, what, dense, rel_tie=8 * np.finfo(np.float32).eps):
    """max_attentions equal to the oracle's.  Under the monotonic window (three keys) they must be equal everywhere.  A
    dense row of up to 4096 random scores may hold two top probabilities that agree to within float32 rounding; there
    the order is decided by the last bits of S (split-fp16 x3 or the fp32 kernel against torch's float32 matmul), and
    the device may pick the other key only if the oracle's two probabilities agree within `rel_tie` of their size."""
    for b, t in zip(*np.nonzero(M != Mr)):
        p_dev, p_ref = Ar[b, M[b, t], t], Ar[b, Mr[b, t], t]
        assert dense and abs(p_dev - p_ref) <= rel_tie * p_ref, (what, b, t, M[b, t], Mr[b, t], p_dev, p_ref)


def _attention_case(engine, Q, K, V, mono, pma, what):
    N = K.shape[1]
    R, A, M = engine.attention(Q, K, V, mono, pma)
    Rr, Ar, Mr = rt.Attention(torch.from_numpy(Q), torch.from_numpy(K), torch.from_numpy(V), mono, pma)
    A = A.cpu().numpy()
    assert np.abs(R.cpu().numpy() - Rr.numpy()).max() < 1e-4, what
    assert np.abs(A - Ar.numpy()).max() < 1e-5, what
    _same_argmax(M.cpu().numpy(), Mr.numpy(), Ar.numpy(), what, dense=not mono)
    if mono:
        for b, p in enumerate(pma):
            live = np.zeros(N, bool); live[p:p + 3] = True
            assert (A[b][~live] == 0).all(), what       # exact zeros outside the window


# ------------------------------------------------------------------------------------------- op level, any N
@pytest.mark.parametrize("tensor_path", [0, 1], ids=["fp32path", "tensorpath"])
@pytest.mark.parametrize("N", [1, 63, 64, 65, 191, 192, 193, 256, 300, 1024])
def test_attention_any_key_count(engine, monkeypatch, tensor_path, N):
    monkeypatch.setattr(Hyperparams, "max_N", N)     # the oracle's window mask is built at hp.max_N keys
    engine.set_tensor_path(tensor_path)
    try:
        for T in (1, 129, 210):
            for B in (1, 3):
                seed = N * 1000 + T * 10 + B
                Q, K, V = _rand((B, T, 256), seed), _rand((B, N, 256), seed + 1), _rand((B, N, 256), seed + 2)
                _attention_case(engine, Q, K, V, False, np.zeros(B, np.int32), (N, T, B, "dense"))
                starts = _windows(N)
                for i in range(0, len(starts), B):          # every window start at both batch sizes
                    group = starts[i:i + B]
                    group += [group[-1]] * (B - len(group))
                    _attention_case(engine, Q, K, V, True, np.asarray(group, np.int32), (N, T, B, group))
    finally:
        engine.set_tensor_path(1)


@pytest.mark.parametrize("tensor_path", [0, 1], ids=["fp32path", "tensorpath"])
def test_attention_past_48_kb_of_scores(engine, monkeypatch, tensor_path):
    """N = 4096: the fp32 kernel's per-block score buffer (16 bytes per key) passes the 48 KB default of dynamic shared
    memory and is granted by attribute; the wgmma kernel's shared memory does not depend on N."""
    N, T, B = 4096, 129, 3
    monkeypatch.setattr(Hyperparams, "max_N", N)
    engine.set_tensor_path(tensor_path)
    try:
        Q, K, V = _rand((B, T, 256), 41), _rand((B, N, 256), 42), _rand((B, N, 256), 43)
        _attention_case(engine, Q, K, V, False, np.zeros(B, np.int32), (N, "dense"))
        _attention_case(engine, Q, K, V, True, np.array([0, 2047, N - 1], np.int32), (N, "monotonic"))
    finally:
        engine.set_tensor_path(1)


def test_fp32_attention_beyond_shared_memory_fails_cleanly(engine):
    """16,384 keys need 256 KB of scores per block of the fp32 kernel, more than an H100 grants: the call fails with a
    message, and the engine keeps working afterwards (no error left behind for the next launch to report)."""
    from dc_tts_b200.engine import DcttsError
    engine.set_tensor_path(0)
    try:
        Q, K, V = _rand((1, 4, 256), 51), _rand((1, 16384, 256), 52), _rand((1, 16384, 256), 53)
        with pytest.raises(DcttsError, match="shared memory"):
            engine.attention(Q, K, V, False, None)
        Q, K, V = _rand((1, 4, 256), 54), _rand((1, 65, 256), 55), _rand((1, 65, 256), 56)
        R, _, _ = engine.attention(Q, K, V, False, None)
        Rr, _, _ = rt.Attention(torch.from_numpy(Q), torch.from_numpy(K), torch.from_numpy(V))
        assert np.abs(R.cpu().numpy() - Rr.numpy()).max() < 1e-4
    finally:
        engine.set_tensor_path(1)


# ------------------------------------------------------------------------------------------- networks at max_N = 300
@pytest.fixture(scope="module")
def hp300():
    old = Hyperparams.max_N
    Hyperparams.max_N = LONG_N
    yield Hyperparams
    Hyperparams.max_N = old


@pytest.fixture(scope="module")
def params300(hp300):
    return init_params(0, "perturbed")


@pytest.fixture(scope="module")
def engine300(hp300, params300):
    from dc_tts_b200.engine import Engine
    e = Engine(0, hparams=hp300)
    e.load_params(params300)
    yield e
    e.close()


@pytest.fixture(params=["fp32path", "tensorpath", "cluster"])
def path300(engine300, request):
    from conftest import KERNEL_SETS
    tp, dm = KERNEL_SETS[request.param]
    engine300.set_tensor_path(tp)
    engine300.set_option("decode_mode", dm)
    yield request.param
    engine300.set_tensor_path(1)
    engine300.set_option("decode_mode", 1)


def _text(B, lengths, seed):
    rng = np.random.default_rng(seed)
    L = np.zeros((B, LONG_N), np.int32)
    for b, n in enumerate(lengths):
        L[b, :n] = rng.integers(2, 32, n)
        L[b, n] = 1                                   # E, then P padding
    return L


def test_textenc_long_and_short_texts(engine300, params300, path300):
    """260 characters and 5 characters on one handle of max_N = 300: the short one is mostly padding, which TextEnc's
    SAME convolutions see up to key 299 (quirk Q2)."""
    L = _text(2, (260, 5), seed=3)
    K, V = engine300.textenc(L)
    Kr, Vr = rt.TextEnc(params300, L)
    assert K.shape == (2, LONG_N, 256)
    assert np.abs(K.cpu().numpy() - Kr.numpy()).max() < NET_TOL
    assert np.abs(V.cpu().numpy() - Vr.numpy()).max() < NET_TOL


def test_teacher_forced_pass_with_windows_past_192(engine300, path300):
    """One sess.run of the synthesis graph at N = 300 with the window at keys below, at and past 192 and at the edge,
    against the reference's own graph at max_N = 300 (refshim_long_text.npz)."""
    g = golden("refshim_long_text.npz")
    L, mels, pma = synth_inputs()
    Y, M, A = engine300.text2mel_forward(L, mels, pma)
    assert np.abs(Y.cpu().numpy() - g["synth_Y"]).max() < NET_TOL
    assert np.array_equal(M.cpu().numpy(), g["synth_max_attentions"])
    aw, outside = window_summary(A.cpu().numpy(), pma)
    assert np.abs(aw - g["synth_align_win"]).max() < 1e-4
    assert (outside == 0).all()                       # exact zeros outside the window, as in the reference


def test_generate_long_text_frame_by_frame(engine300, params300, path300):
    """Free-running decode of a 250-character text.  Frames j are checked against the oracle's sess.run on the device's
    own prefix Y[:j] and window P[j] (the discipline of test_gpu_input_range.py).  With the seeded weights the window
    does not travel past key 192 within 210 frames, so keys past 192 under the window are covered by the op-level and
    teacher-forced cases above."""
    L = _text(2, (250, 210), seed=6)
    Y, P, _, _ = engine300.text2mel_generate(L)
    Y, P = Y.cpu().numpy(), P.cpu().numpy()
    assert np.isfinite(Y).all()
    T = Hyperparams.max_T
    for j in (0, 1, 100, T - 1):
        prefix = Y.copy()
        prefix[:, j:] = 0
        ref = rt.text2mel_forward(params300, L, torch.from_numpy(prefix), P[:, j])
        assert np.abs(Y[:, j] - ref["Y"].numpy()[:, j]).max() < NET_TOL, j
        if j + 1 < T:
            assert np.array_equal(P[:, j + 1], ref["max_attentions"].numpy()[:, j]), j


def test_synthesize_long_sentence_to_wav(engine, engine300, tmp_path, monkeypatch):
    """synthesize(...) end to end on a 250-character sentence with max_N = 300: text file -> Graph -> mel loop -> SSRN ->
    Griffin-Lim -> wav."""
    from scipy.io.wavfile import read as read_wav
    from dc_tts_b200 import synthesize as syn
    from dc_tts_b200.engine import get_engine, set_engine
    words = "the birch canoe slid on the smooth planks and glue the sheet to the dark blue background "
    sent = (words * 4)[:249].strip() + "."
    assert len(sent) > 192
    path = tmp_path / "long.txt"
    path.write_text("header\n1. %s\n" % sent)
    monkeypatch.chdir(tmp_path)
    prev = get_engine()
    set_engine(engine300)
    try:
        Y, Z = syn.synthesize(sentences=str(path), fast=True, write=True)
    finally:
        set_engine(prev)
    assert Y.shape == (1, Hyperparams.max_T, Hyperparams.n_mels) and np.isfinite(Y).all() and np.isfinite(Z).all()
    sr, wav = read_wav(tmp_path / "samples" / "1.wav")
    assert sr == Hyperparams.sr and wav.dtype == np.float32 and len(wav) > 0 and np.isfinite(wav).all()


# ------------------------------------------------------------------------------------------- training at max_N = 300
def _engine(hp, P, tc):
    from dc_tts_b200.engine import Engine
    e = Engine(0, hparams=hp)
    e.load_params(P)
    e.set_option("train_tc", tc)
    return e


@pytest.mark.parametrize("B,N,T,seed", [(2, LONG_N, 53, 11), (3, 250, 149, 4), (2, 37, 53, 5)])
def test_train_step_long_text_vs_oracle(hp300, B, N, T, seed):
    """Losses (the guided-attention loss on the (300, max_T) table included) and every gradient against the bucket-shape
    oracle, on the wgmma and the fp32 kernel sets."""
    from test_train import _compare_grads, _tie_free
    P = _tie_free(init_params(0, "perturbed"))
    L, mels = synthetic_bucket(B, N, T, seed=seed)
    _, _, info = rtb.train_step(P, L, mels, global_step=7, seed=seed, rate=0.05)
    for tc in (7, 0):
        eng = _engine(hp300, P, tc)
        try:
            eng.train_init(B, 0.05)
            out = eng.train_step(L, mels, global_step=7, seed=seed, apply=False)
            for k in ("loss", "loss_mels", "loss_bd1", "loss_att"):
                assert abs(out[k] - info[k]) < 1e-5 * max(1.0, abs(info[k])), (tc, k, out[k], info[k])
            _compare_grads(eng, info["grads"])
        finally:
            eng.close()


def test_train_step_past_48_kb_of_attention_scores(hp300, monkeypatch):
    """N = 3200 on a max_N = 3200 handle: the attention backward's per-block dA buffer (16 bytes per key) and the fp32
    forward's score buffer pass the 48 KB default of dynamic shared memory.  Losses and every gradient against the
    bucket-shape oracle on both kernel sets."""
    from test_train import _compare_grads, _tie_free
    monkeypatch.setattr(Hyperparams, "max_N", 3200)
    P = _tie_free(init_params(0, "perturbed"))
    L, mels = synthetic_bucket(1, 3200, 24, seed=8)
    _, _, info = rtb.train_step(P, L, mels, global_step=7, seed=8, rate=0.05)
    for tc in (7, 0):
        eng = _engine(Hyperparams, P, tc)
        try:
            eng.train_init(1, 0.05)
            out = eng.train_step(L, mels, global_step=7, seed=8, apply=False)
            for k in ("loss", "loss_mels", "loss_bd1", "loss_att"):
                assert abs(out[k] - info[k]) < 1e-5 * max(1.0, abs(info[k])), (tc, k, out[k], info[k])
            _compare_grads(eng, info["grads"])
        finally:
            eng.close()


class _Recorder:
    def __init__(self, hp):
        self.hp, self.shapes = hp, []

    def train_init(self, B, dropout_rate=None):
        pass

    def restore_training(self, logdir, scope):
        return None

    def train_step(self, L, mels, global_step=0, seed=0, apply=True):
        self.shapes.append(L.shape)
        return {"loss": 0.0}


def _long_batches():
    for N, T in ((193, 60), (250, 120), (LONG_N, 210)):
        L, mels = synthetic_bucket(2, N, T, seed=N)
        yield L, mels, None, ["x", "y"]


def test_trainer_takes_long_texts_at_max_n_300_and_skips_them_at_180(hp300, tmp_path):
    big = _Recorder(hp300)
    logs = []
    trainer.train(1, big, _long_batches(), num_iterations=10, logdir=str(tmp_path / "a"), log=logs.append)
    assert big.shapes == [(2, 193), (2, 250), (2, LONG_N)] and not any("skipped" in m for m in logs)
    small = _Recorder(types.SimpleNamespace(max_N=180, max_T=hp300.max_T))
    logs = []
    trainer.train(1, small, _long_batches(), num_iterations=10, logdir=str(tmp_path / "b"), log=logs.append)
    assert small.shapes == [] and sum("skipped" in m for m in logs) == 3


def test_cuda_trainer_run_and_capacity_at_max_n_300(engine300, hp300, tmp_path):
    """trainer.train on a real handle takes every 193..300-character bucket; N = 301 still fails and launches nothing."""
    from dc_tts_b200.engine import DcttsError
    eng = _engine(hp300, init_params(0, "perturbed"), 7)
    try:
        logs = []
        gs = trainer.train(1, eng, _long_batches(), num_iterations=10, logdir=str(tmp_path), log=logs.append, save_every=10 ** 6)
        assert gs == 3 and not any("skipped" in m for m in logs)
        L, mels = synthetic_bucket(2, 40, 50, seed=1)
        eng.train_step(L, mels, apply=False)
        n0 = eng.launch_count()
        Lbig, _ = synthetic_bucket(2, LONG_N + 1, 50, seed=1)
        with pytest.raises(DcttsError):
            eng.train_step(Lbig, mels, apply=False)
        assert eng.launch_count() == n0
    finally:
        eng.close()
