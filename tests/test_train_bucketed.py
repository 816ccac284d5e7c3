"""Training steps at a length-bucketed batch's own shape (reference data_load.py:122-129, dynamic_pad=True; losses
train.py:83-108 at that shape).  CPU: the autograd oracle against the reference's own training graphs on bucket-shaped
batches (refshim_train_bucket.npz, tests/golden/make_golden_refchecks_bucket.py), the trainer loop and Graph(mode="train")
with bucketed batches, sharded buckets.  GPU: both CUDA trainers at bucket shapes against the oracle, shape changes on one
handle, the capacity checks, and an end-to-end bucketed run."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, golden
from dc_tts_b200 import trainer
from dc_tts_b200.hyperparams import Hyperparams as hp
from dc_tts_b200.params import init_params, synthetic_bucket
from oracle import ref_train as rtr

import ref_train_bucket as rtb

sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_golden_refchecks_bucket import SSRN_CASES, T2M_CASES, ssrn_batch      # noqa: E402

HAVE_REF = os.path.isfile("/root/reference/train.py")
F = 1 + hp.n_fft // 2


# ------------------------------------------------------------------------------------------- oracle vs reference
def _oracle_t2m(P, N, T, seed, rate):
    L, mels = synthetic_bucket(2, N, T, seed=7)
    W = {n: torch.tensor(np.asarray(P[n], np.float32)) for n in rtr.text2mel_names()}
    with torch.no_grad():
        return rtb.forward(W, L, mels, seed, rate)


def _oracle_ssrn(P, T):
    mels, mags = ssrn_batch(T)
    W = {n: torch.tensor(np.asarray(P[n], np.float32)) for n in rtr.ssrn_names()}
    with torch.no_grad():
        return rtr.forward_ssrn(W, mels, mags, 9)


def test_oracle_losses_vs_reference_training_graph_at_bucket_shapes():
    g = golden("refshim_train_bucket.npz")
    P = init_params(0, "perturbed")
    for tag, N, T, seed, rate in T2M_CASES:
        assert int(g[tag + "_ncalls"]) == (38 if rate > 0 else 0)
        o = _oracle_t2m(P, N, T, seed, rate)
        for k, ref in zip(("loss", "loss_mels", "loss_bd1", "loss_att"), g[tag]):
            assert abs(float(o[k]) - ref) < 2e-6 * max(1.0, abs(ref)), (tag, k, float(o[k]), ref)
    for tag, T in SSRN_CASES:
        assert int(g[tag + "_ncalls"]) == 16
        o = _oracle_ssrn(P, T)
        for k, ref in zip(("loss", "loss_mags", "loss_bd2"), g[tag]):
            assert abs(float(o[k]) - ref) < 2e-6 * max(1.0, abs(ref)), (tag, k, float(o[k]), ref)


def test_bucket_oracle_is_the_fixed_shape_oracle_at_full_shape():
    """At (max_N, max_T) the -1 padding of train.py:91 is empty: the bucket-shape oracle is ref_train's, bit for bit."""
    P = init_params(0, "perturbed")
    L, mels = synthetic_bucket(1, hp.max_N, hp.max_T, seed=3)
    W = {n: torch.tensor(np.asarray(P[n], np.float32)) for n in rtr.text2mel_names()}
    with torch.no_grad():
        a = rtb.forward(W, L, mels, 11, 0.05)
        b = rtr.forward(W, L, mels, 11, 0.05)
    for k in ("loss", "loss_mels", "loss_bd1", "loss_att"):
        assert float(a[k]) == float(b[k]), k


def test_padding_a_bucket_changes_the_objective():
    """Why the step runs at the bucket's shape: the same batch padded to (max_N, max_T) has different losses."""
    P = init_params(0, "perturbed")
    L, mels = synthetic_bucket(2, 37, 53, seed=7)
    Lf, mf, _ = trainer.pad_to_fixed(L, mels, np.zeros((2, 4 * 53, 4), np.float32))
    W = {n: torch.tensor(np.asarray(P[n], np.float32)) for n in rtr.text2mel_names()}
    with torch.no_grad():
        a = rtb.forward(W, L, mels, 0, 0.0)
        b = rtr.forward(W, Lf, mf, 0, 0.0)
    assert abs(float(a["loss_mels"]) - float(b["loss_mels"])) > 1e-2
    assert abs(float(a["loss_att"]) - float(b["loss_att"])) > 1e-4


@pytest.mark.skipif(not HAVE_REF, reason="/root/reference is not present on this machine")
def test_oracle_losses_vs_reference_training_graph_at_bucket_shapes_live():
    import tf_shim
    P = init_params(0, "perturbed")
    tf_shim.install(tf_shim.Store(P))
    import hyperparams as ref_hp
    for tag, N, T, seed, rate in T2M_CASES[:2]:
        L, mels = synthetic_bucket(2, N, T, seed=7)
        ref_hp.Hyperparams.dropout_rate = rate
        try:
            ref, _ = tf_shim.run_train_graph(L, mels, lambda x, r, i: x * rtr.dropout_keep(x.shape, i, seed, r))
        finally:
            ref_hp.Hyperparams.dropout_rate = hp.dropout_rate
        o = _oracle_t2m(P, N, T, seed, rate)
        for k in ("loss", "loss_mels", "loss_bd1", "loss_att"):
            assert abs(float(o[k]) - ref[k]) < 2e-6 * max(1.0, abs(ref[k])), (tag, k, float(o[k]), ref[k])
    mels, mags = ssrn_batch(9)
    ref, _ = tf_shim.run_train_graph_ssrn(mels, mags, lambda x, r, i: x * rtr.dropout_keep(x.shape, i, 9, r))
    o = _oracle_ssrn(P, 9)
    for k in ("loss", "loss_mags", "loss_bd2"):
        assert abs(float(o[k]) - ref[k]) < 2e-6 * max(1.0, abs(ref[k])), (k, float(o[k]), ref[k])


# ------------------------------------------------------------------------------------------- trainer loop (CPU)
class _Recorder:
    """Engine stand-in: records the shapes each step receives."""

    def __init__(self):
        self.calls, self.init, self.inits, self.saved = [], None, 0, []

    def train_init(self, B):
        self.init = ("t2m", B); self.inits += 1

    def train_init_ssrn(self, B, T):
        self.init = ("ssrn", B, T); self.inits += 1

    def train_step(self, L, mels, global_step=0, seed=0, apply=True):
        self.calls.append((L.shape, mels.shape))
        return {"loss": 1.0, "loss_mels": 0.3, "loss_bd1": 0.69, "loss_att": 0.01}

    def train_step_ssrn(self, mels, mags, global_step=0, seed=0, apply=True):
        self.calls.append((mels.shape, mags.shape))
        return {"loss": 1.0, "loss_mags": 0.3, "loss_bd2": 0.7}

    def save_checkpoint(self, prefix, gs, scope):
        self.saved.append(gs)

    def restore_training(self, logdir, scope):
        return None


def _buckets(B=2):
    """(L, mels, mags, names, bucket) tuples at their own shapes; the third is longer than max_T."""
    out = []
    for N, T in ((37, 53), (120, 171), (60, hp.max_T + 5), (hp.max_N, hp.max_T)):
        L, mels = synthetic_bucket(B, N, T, seed=1)
        out.append((L, mels, np.zeros((B, 4 * T, 3), np.float32), ["u"] * B, 0))
    return out


@pytest.mark.parametrize("num", [1, 2])
def test_trainer_takes_bucketed_batches_at_their_own_shape(tmp_path, num):
    eng, log = _Recorder(), []
    gs = trainer.train(num, eng, iter(_buckets()), num_iterations=100, logdir=str(tmp_path / "ld"), global_step=0, log=log.append)
    assert gs == 3 and eng.inits == 1
    assert eng.init == (("t2m", 2) if num == 1 else ("ssrn", 2, hp.max_T))          # SSRN capacity hp.max_T, allocated once
    if num == 1:
        assert eng.calls == [((2, 37), (2, 53, hp.n_mels)), ((2, 120), (2, 171, hp.n_mels)), ((2, hp.max_N), (2, hp.max_T, hp.n_mels))]
    else:
        assert eng.calls == [((2, 53, hp.n_mels), (2, 212, 3)), ((2, 171, hp.n_mels), (2, 684, 3)), ((2, hp.max_T, hp.n_mels), (2, 840, 3))]
    skips = [s for s in log if s.startswith("skipped")]
    assert len(skips) == 1 and "T=%d" % (hp.max_T + 5) in skips[0] and "1 skipped so far" in skips[0]


def test_over_capacity_text_is_skipped_by_text2mel_only(tmp_path):
    L, mels = synthetic_bucket(2, hp.max_N + 3, 40, seed=2)
    batch = (L, mels, np.zeros((2, 160, 3), np.float32), ["u", "u"])
    assert trainer.over_capacity(1, L, mels) and not trainer.over_capacity(2, L, mels)
    eng = _Recorder()
    assert trainer.train(1, eng, [batch], logdir=str(tmp_path / "a"), global_step=0, log=lambda *_: None) == 0 and not eng.calls
    eng = _Recorder()
    assert trainer.train(2, eng, [batch], logdir=str(tmp_path / "b"), global_step=0, log=lambda *_: None) == 1 and len(eng.calls) == 1


def test_graph_train_takes_bucketed_batches():
    from dc_tts_b200.train import Graph, Session
    for num in (1, 2):
        eng = _Recorder()
        g = Graph(num=num, engine=eng, batches=iter(_buckets()), global_step=10)
        with Session() as sess:
            for _ in range(3):
                sess.run([g.global_step, g.train_op])
        assert g.skipped_batches == 1 and g.global_step_value == 13 and eng.inits == 1
        assert eng.init == (("t2m", 2) if num == 1 else ("ssrn", 2, hp.max_T))
        shapes = [c[0] if num == 1 else c[0][:2] for c in eng.calls]
        assert shapes == [(2, 37), (2, 120), (2, hp.max_N)] if num == 1 else shapes == [(2, 53), (2, 171), (2, hp.max_T)]
    with pytest.raises(ValueError, match="bucketed_batches"):
        Graph(num=1, engine=_Recorder())


def test_sharded_bucketed_batches_are_disjoint():
    rng = np.random.default_rng(2)
    n = 80
    lens = [int(x) for x in rng.integers(12, 150, n)]
    texts = [rng.integers(2, 30, l).astype(np.int32) for l in lens]
    store = {"U%03d.wav" % i: (np.full((l + 5, hp.n_mels), i, np.float32), np.full((4 * (l + 5), 3), i, np.float32)) for i, l in enumerate(lens)}
    fpaths = ["wavs/U%03d.wav" % i for i in range(n)]
    loader = lambda p: (os.path.basename(p),) + store[os.path.basename(p)]
    seen = []
    for rank in (0, 1, 2):
        names = [nm for b in trainer.bucketed_batches(fpaths, lens, texts, B=2, seed=4, loader=loader, epochs=1, rank=rank, world=3) for nm in b[3]]
        assert names
        seen.append(set(names))
    assert not (seen[0] & seen[1]) and not (seen[0] & seen[2]) and not (seen[1] & seen[2])
    whole = [nm for b in trainer.bucketed_batches(fpaths, lens, texts, B=2, seed=4, loader=loader, epochs=1) for nm in b[3]]
    assert len(set(whole)) == len(whole)                                   # world = 1 is the unsharded stream


# ------------------------------------------------------------------------------------------- GPU
def _tie_free_t2m(P):
    from test_train import _tie_free
    return _tie_free(P)


def _tie_free_ssrn(P):
    """LayerNorm beta + 8 on SSRN's ReLU blocks: every pre-activation clears zero, so a correct float32 forward cannot flip
    a ReLU mask (the same device as the Text2Mel tie-free set, tests/test_train.py)."""
    from dc_tts_b200 import arch
    P = dict(P)
    for l in arch.ssrn_layers():
        if l.kind == "C" and l.act == "relu":
            n = "SSRN/%s/normalize/beta" % l.scope
            P[n] = (np.asarray(P[n], np.float32) + 8.0).astype(np.float32)
    return P


def _grad_close(a, b, names, rtol):
    """Per tensor: max |a - b| relative to b's max-norm."""
    for n in names:
        x, y = a.train_tensor(n, "grad"), b.train_tensor(n, "grad")
        assert np.abs(x - y).max() <= rtol * max(np.abs(y).max(), 1e-12), n


def _engine(P, tc=7):
    from dc_tts_b200.engine import Engine
    e = Engine(0)
    e.load_params(P)
    e.set_option("train_tc", tc)
    return e


@pytest.mark.gpu
@pytest.mark.parametrize("B,N,T,seed", [(2, 37, 53, 11), (3, 101, 149, 4), (32, 123, 171, 5)])
def test_cuda_train_step_at_bucket_shape_vs_oracle(B, N, T, seed):
    from test_train import _compare_grads
    P = _tie_free_t2m(init_params(0, "perturbed"))
    L, mels = synthetic_bucket(B, N, T, seed=seed)
    newP, st, info = rtb.train_step(P, L, mels, global_step=7, seed=seed, rate=0.05)
    for tc in (7, 0):
        eng = _engine(P, tc)
        eng.train_init(B, 0.05)
        out = eng.train_step(L, mels, global_step=7, seed=seed, apply=False)
        for k in ("loss", "loss_mels", "loss_bd1", "loss_att"):
            assert abs(out[k] - info[k]) < 1e-5 * max(1.0, abs(info[k])), (tc, k, out[k], info[k])
        assert len(info["grads"]) == 209
        _compare_grads(eng, info["grads"])
        eng.train_apply(7)
        for n in ("Text2Mel/TextEnc/embed_1/lookup_table", "Text2Mel/TextEnc/HC_7/conv1d/kernel", "Text2Mel/AudioEnc/C_1/conv1d/kernel",
                  "Text2Mel/AudioDec/HC_3/H2/gamma", "Text2Mel/AudioDec/C_11/conv1d/bias", "Text2Mel/AudioEnc/HC_9/H1/beta"):
            m, v = st[n]
            np.testing.assert_allclose(eng.train_tensor(n, "m"), m, rtol=2e-3, atol=max(1e-9, 1e-4 * np.abs(m).max()))
            np.testing.assert_allclose(eng.train_tensor(n, "v"), v, rtol=4e-3, atol=max(1e-14, 4e-4 * np.abs(v).max()))
            step = np.abs(newP[n] - P[n]).max()
            assert np.abs(eng.train_tensor(n, "param") - newP[n]).max() <= 0.05 * step + 2.4e-7, n
        eng.close()


@pytest.mark.gpu
def test_cuda_ssrn_shapes_on_one_handle_vs_oracle_and_fresh_handles():
    """One handle of capacity 210 steps at T = 9, 53, 150 with Adam applied in between: every step against the oracle's
    step chain (the Adam state survives the shape changes) and its gradients against a fresh handle of capacity T
    loaded with the same weights."""
    from test_train import _compare_grads
    P = _tie_free_ssrn(init_params(0, "perturbed"))
    names = rtr.ssrn_names()
    eng = _engine(P)
    eng.train_init_ssrn(2, hp.max_T, 0.05)
    cur, st = P, None
    for i, T in enumerate((9, 53, 150)):
        gs = 3999 + i
        mels, mags = ssrn_batch(T)
        newP, st, info = rtr.train_step_ssrn(cur, mels, mags, state=st, global_step=gs, seed=i, rate=0.05)
        out = eng.train_step_ssrn(mels, mags, global_step=gs, seed=i, apply=False)
        for k in ("loss", "loss_mags", "loss_bd2"):
            assert abs(out[k] - info[k]) < 1e-5 * max(1.0, abs(info[k])), (T, k, out[k], info[k])
        _compare_grads(eng, info["grads"])
        fresh = _engine(dict(P, **{n: eng.train_tensor(n, "param") for n in names}))
        fresh.train_init_ssrn(2, T, 0.05)
        fresh.train_step_ssrn(mels, mags, global_step=gs, seed=i, apply=False)
        _grad_close(eng, fresh, names, 1e-4)
        fresh.close()
        eng.train_apply(gs)
        for n in ("SSRN/D_4/conv2d_transpose/kernel", "SSRN/HC_12/conv1d/kernel", "SSRN/C_16/conv1d/bias", "SSRN/C_15/normalize/gamma"):
            m, v = st[n]
            np.testing.assert_allclose(eng.train_tensor(n, "m"), m, rtol=2e-3, atol=max(1e-9, 1e-4 * np.abs(m).max()))
            np.testing.assert_allclose(eng.train_tensor(n, "v"), v, rtol=4e-3, atol=max(1e-14, 4e-4 * np.abs(v).max()))
        cur = newP
    eng.close()


@pytest.mark.gpu
def test_cuda_text2mel_shape_changes_match_fresh_handles_and_the_fixed_entry_point():
    import ctypes as C
    from dc_tts_b200.engine import _ptr
    P = _tie_free_t2m(init_params(0, "perturbed"))
    names = rtr.text2mel_names()
    eng = _engine(P)
    eng.train_init(3, 0.05)
    for N, T in ((37, 53), (hp.max_N, hp.max_T), (29, 37)):
        L, mels = synthetic_bucket(3, N, T, seed=N)
        a = eng.train_step(L, mels, global_step=5, seed=N, apply=False)
        fresh = _engine(P)
        fresh.train_init(3, 0.05)
        b = fresh.train_step(L, mels, global_step=5, seed=N, apply=False)
        for k in a:
            assert abs(a[k] - b[k]) <= 1e-4 * max(1.0, abs(b[k])), (N, T, k)
        _grad_close(eng, fresh, names, 1e-4)
        if N == hp.max_N:                                   # the fixed-shape entry point is the shaped one at (max_N, max_T)
            Ld, md = eng._i32(L), eng._f32(mels)
            out = (C.c_float * 4)()
            eng._check(eng._lib.dctts_train_step(eng._h, _ptr(Ld), _ptr(md), 3, 5, N, C.c_float(hp.lr), 0, out, eng._stream()), "fixed")
            assert abs(out[0] - a["loss"]) <= 1e-4 * max(1.0, abs(a["loss"]))
            _grad_close(eng, fresh, names, 1e-4)
        fresh.close()
    eng.close()


@pytest.mark.gpu
def test_cuda_capacity_and_shape_errors_launch_nothing():
    from dc_tts_b200.engine import DcttsError
    P = init_params(0, "perturbed")
    eng = _engine(P)
    eng.train_init(2, 0.0)
    L, mels = synthetic_bucket(2, 40, 50, seed=1)
    eng.train_step(L, mels, apply=False)
    n0 = eng.launch_count()
    Lbig, _ = synthetic_bucket(2, hp.max_N + 1, 50, seed=1)
    _, mbig = synthetic_bucket(2, 40, hp.max_T + 1, seed=1)
    for args in ((Lbig, mels), (L, mbig), (L[0], mels), (L, mels[:, :, :40]), (L, mels[:1])):
        with pytest.raises(DcttsError):
            eng.train_step(*args, apply=False)
    assert eng.launch_count() == n0
    s = _engine(P)
    s.train_init_ssrn(2, 60, 0.0)
    mels, mags = ssrn_batch(20)
    s.train_step_ssrn(mels, mags, apply=False)
    n0 = s.launch_count()
    m61, g61 = ssrn_batch(61)
    for args in ((m61, g61), (mels, mags[:, :79]), (mels, mags[:, :, :1000]), (mels[:, :, :40], mags)):
        with pytest.raises(DcttsError):
            s.train_step_ssrn(*args, apply=False)
    assert s.launch_count() == n0
    eng.close(); s.close()


def _write_varied_dataset(root, n=40, seed=0):
    rng = np.random.default_rng(seed)
    d = root / "LJSpeech-1.0"
    (d / "wavs").mkdir(parents=True)
    (root / "mels").mkdir(); (root / "mags").mkdir()
    lines = []
    for i in range(n):
        nchar = int(rng.integers(10, 150))
        lines.append("LJ%03d|raw|%s" % (i, "".join(rng.choice(list("abcdefghijklmnopqrstuvwxyz '"), nchar))))
        T = int(min(hp.max_T, 12 + 1.3 * nchar + rng.integers(0, 10)))
        base = 0.5 + 0.4 * np.sin(np.linspace(0, 3 + i % 5, T))[:, None] * np.cos(np.linspace(0, 2, hp.n_mels))[None, :]
        mel = np.clip(base + 0.02 * rng.standard_normal((T, hp.n_mels)), 0, 1).astype(np.float32)
        mag = np.clip(np.repeat(base[:, :1], hp.r, 0) * np.linspace(1, 0.2, F)[None, :] + 0.02 * rng.standard_normal((T * hp.r, F)), 0, 1).astype(np.float32)
        np.save(root / "mels" / ("LJ%03d.npy" % i), mel); np.save(root / "mags" / ("LJ%03d.npy" % i), mag)
    (d / "transcript.csv").write_text("\n".join(lines) + "\n", encoding="utf-8")
    return str(d)


@pytest.mark.gpu
@pytest.mark.parametrize("num", [1, 2])
def test_cuda_trainer_on_bucketed_batches_end_to_end(tmp_path, num):
    from dc_tts_b200.checkpoint import latest_checkpoint
    from dc_tts_b200.engine import Engine
    d = _write_varied_dataset(tmp_path)
    fpaths, lens, texts = trainer.load_train_data(d)
    loader = lambda p: trainer._load_spectrograms_npy(p, str(tmp_path / "mels"), str(tmp_path / "mags"))
    B, P = 4, init_params(1)
    shapes = set()

    def recording(batches):
        for b in batches:
            shapes.add(b[1].shape[1])
            yield b
    batches = recording(trainer.bucketed_batches(fpaths, lens, texts, B=B, seed=0, loader=loader))
    eng = Engine(0); eng.load_params(P)
    logdir = str(tmp_path / ("logdir/LJ01-%d" % num))
    gs = trainer.train(num, eng, batches, num_iterations=299, logdir=logdir, save_every=100, log=lambda *_: None)
    assert gs == 300 and len(shapes) > 5                                  # many different bucket shapes
    assert latest_checkpoint(logdir).endswith("model_gs_000k")           # gs // 1000 names the bundle (train.py:152)
    L0, m0, g0 = next(trainer.bucketed_batches(fpaths, lens, texts, B=B, seed=0, loader=loader))[:3]
    fresh = Engine(0); fresh.load_params(P)
    if num == 1:
        fresh.train_init(B, 0.0)
        first = fresh.train_step(L0, m0, global_step=0, apply=False)["loss"]
        last = eng.train_step(L0, m0, global_step=300, apply=False)["loss"]
    else:
        fresh.train_init_ssrn(B, hp.max_T, 0.0)
        first = fresh.train_step_ssrn(m0, g0, global_step=0, apply=False)["loss"]
        last = eng.train_step_ssrn(m0, g0, global_step=300, apply=False)["loss"]
    assert np.isfinite(last) and last < 0.9 * first, (first, last)
    fresh.close()
    more = []
    resumed = Engine(0); resumed.load_params(P)
    gs2 = trainer.train(num, resumed, trainer.bucketed_batches(fpaths, lens, texts, B=B, seed=1, loader=loader), num_iterations=305,
                        logdir=logdir, save_every=100, log=more.append)
    assert gs2 == 306 and any("resumed" in s and "300" in s for s in more)
    eng.close(); resumed.close()
