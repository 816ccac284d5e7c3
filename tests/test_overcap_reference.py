"""Training past (max_N, max_T), as the reference's train.py does.  It caps no batch: train.py:91-95 pads the alignments
with -1 to (max_N, max_T) and crops them to it, so the guided-attention loss covers the table's corner and the mel losses
the whole batch.  CPU checks: the bucket-shape oracle (tests/ref_train_bucket.py) against the reference's own training
graphs at such shapes (refshim_train_overcap.npz, tests/golden/make_golden_refchecks_overcap.py), and the trainer loop and
Graph(mode="train") with beyond_capacity="grow" and capacity=.  tests/test_gpu_train_overcap.py runs the CUDA side."""
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
from make_golden_refchecks_overcap import SSRN_T, T2M_CASES, dropout_hook, ssrn_batch, train_inputs  # noqa: E402

HAVE_REF = os.path.isfile("/root/reference/train.py")
LOSSES = ("loss", "loss_mels", "loss_bd1", "loss_att")


@pytest.fixture(scope="module")
def P():
    return init_params(0, "perturbed")


def _oracle_t2m(P, B, N, T, seed, rate):
    L, mels = train_inputs(B, N, T)
    W = {n: torch.tensor(np.asarray(P[n], np.float32)) for n in rtr.text2mel_names()}
    with torch.no_grad():
        return rtb.forward(W, L, mels, seed, rate)


def test_fixture_is_past_the_table():
    g = golden("refshim_train_overcap.npz")
    assert (hp.max_N, hp.max_T) == (180, 210)
    for tag, B, N, T, seed, rate in T2M_CASES:
        assert N > hp.max_N or T > hp.max_T
        assert int(g[tag + "_ncalls"]) == (38 if rate > 0 else 0)
    assert int(g["ssrn_T%d_ncalls" % SSRN_T]) == 16 and SSRN_T > hp.max_T


def test_bucket_oracle_losses_vs_reference_training_graph_past_the_table(P):
    g = golden("refshim_train_overcap.npz")
    for tag, B, N, T, seed, rate in T2M_CASES:
        o = _oracle_t2m(P, B, N, T, seed, rate)
        for i, k in enumerate(LOSSES):
            ref = g[tag][i]
            assert abs(float(o[k]) - ref) < 2e-6 * max(1.0, abs(ref)), (tag, k, float(o[k]), ref)
    mels, mags = ssrn_batch(SSRN_T)
    W = {n: torch.tensor(np.asarray(P[n], np.float32)) for n in rtr.ssrn_names()}
    with torch.no_grad():
        o = rtr.forward_ssrn(W, mels, mags, 9)
    for i, k in enumerate(("loss", "loss_mags", "loss_bd2")):
        ref = g["ssrn_T%d" % SSRN_T][i]
        assert abs(float(o[k]) - ref) < 2e-6 * max(1.0, abs(ref)), (k, float(o[k]), ref)


def test_guided_attention_loss_is_the_tables_corner(P):
    """The crop: loss_att is the mean over the (max_N, max_T) corner, not over the whole alignment."""
    B, N, T, seed, rate = 3, 200, 240, 0, 0.0
    o = _oracle_t2m(P, B, N, T, seed, rate)
    A = o["alignments"]
    assert tuple(A.shape) == (B, N, T)
    gts = torch.from_numpy(rtr.guided_attention())
    corner = (A[:, :hp.max_N, :hp.max_T] * gts).abs().sum() / (B * hp.max_N * hp.max_T)
    assert float(o["loss_att"]) == float(corner)


@pytest.mark.skipif(not HAVE_REF, reason="/root/reference is not present on this machine")
def test_reference_live_past_the_table(P):
    import tf_shim
    tf_shim.install(tf_shim.Store(P))
    import hyperparams as ref_hp
    g = golden("refshim_train_overcap.npz")
    tag, B, N, T, seed, rate = T2M_CASES[0]
    L, mels = train_inputs(B, N, T)
    ref_hp.Hyperparams.dropout_rate = rate
    try:
        ref, _ = tf_shim.run_train_graph(L, mels, dropout_hook(seed))
    finally:
        ref_hp.Hyperparams.dropout_rate = hp.dropout_rate
    for i, k in enumerate(LOSSES):
        assert abs(ref[k] - g[tag][i]) < 1e-12 * max(1.0, abs(ref[k])), k


# ------------------------------------------------------------------------------------------- trainer loop (CPU)
class _Recorder:
    """Engine stand-in: records the shapes each step receives and every reserve, and refuses a step past the capacity
    as the CUDA engine does."""

    def __init__(self):
        self.calls, self.reserves, self.inits, self.saved = [], [], 0, []
        self.cap = None

    def train_init(self, B):
        self.inits += 1; self.cap = [hp.max_N, hp.max_T]

    def train_init_ssrn(self, B, T):
        self.inits += 1; self.cap = [0, T]

    def train_reserve(self, N, T):
        self.reserves.append((N, T))
        self.cap = [max(self.cap[0], N), max(self.cap[1], T)]

    def train_step(self, L, mels, global_step=0, seed=0, apply=True):
        assert L.shape[1] <= self.cap[0] and mels.shape[1] <= self.cap[1]
        self.calls.append((L.shape, mels.shape))
        return {"loss": 1.0, "loss_mels": 0.3, "loss_bd1": 0.69, "loss_att": 0.01}

    def train_step_ssrn(self, mels, mags, global_step=0, seed=0, apply=True):
        assert mels.shape[1] <= self.cap[1]
        self.calls.append((mels.shape, mags.shape))
        return {"loss": 1.0, "loss_mags": 0.3, "loss_bd2": 0.7}

    def save_checkpoint(self, prefix, gs, scope):
        self.saved.append(gs)

    def restore_training(self, logdir, scope):
        return None


SHAPES = ((37, 53), (187, 171), (60, hp.max_T + 5), (190, 215), (hp.max_N, hp.max_T), (200, 240), (150, 230))


def _buckets(B=2):
    out = []
    for N, T in SHAPES:
        L, mels = synthetic_bucket(B, N, T, seed=1)
        out.append((L, mels, np.zeros((B, 4 * T, 3), np.float32), ["u"] * B, 0))
    return out


@pytest.mark.parametrize("num", [1, 2])
def test_trainer_grows_and_trains_every_batch(tmp_path, num):
    eng, log = _Recorder(), []
    gs = trainer.train(num, eng, iter(_buckets()), num_iterations=100, logdir=str(tmp_path / "ld"), global_step=0, log=log.append,
                       beyond_capacity="grow")
    assert gs == len(SHAPES) and eng.inits == 1 and len(eng.calls) == len(SHAPES)
    assert not [s for s in log if s.startswith("skipped")]
    if num == 1:
        assert eng.reserves == [(192, 210), (192, 256), (256, 256)]     # 187 -> 192; 215 -> 256; 200 -> 256
    else:
        assert eng.reserves == [(0, 256)]                                   # N is ignored; 215 -> 256, then 240 fits
    grew = [s for s in log if s.startswith("grew")]
    assert len(grew) == len(eng.reserves)


def test_trainer_default_still_skips(tmp_path):
    eng, log = _Recorder(), []
    gs = trainer.train(1, eng, iter(_buckets()), num_iterations=100, logdir=str(tmp_path / "ld"), global_step=0, log=log.append)
    assert gs == 2 and not eng.reserves
    assert len([s for s in log if s.startswith("skipped")]) == len(SHAPES) - 2


@pytest.mark.parametrize("num", [1, 2])
def test_capacity_reserves_once(tmp_path, num):
    eng, log = _Recorder(), []
    gs = trainer.train(num, eng, iter(_buckets()), num_iterations=100, logdir=str(tmp_path / "ld"), global_step=0, log=log.append,
                       capacity=(256, 256))
    assert gs == len(SHAPES) and eng.reserves == [(256, 256) if num == 1 else (0, 256)]
    assert not [s for s in log if s.startswith(("skipped", "grew"))]
    eng, log = _Recorder(), []                                             # a capacity below the batches: skip past it
    gs = trainer.train(1, eng, iter(_buckets()), num_iterations=100, logdir=str(tmp_path / "ld2"), global_step=0, log=log.append,
                       capacity=(190, 220))
    assert eng.reserves == [(190, 220)] and gs == 5                       # (200, 240) and (150, 230) are beyond it
    skips = [s for s in log if s.startswith("skipped")]
    assert len(skips) == 2 and "(N=190, T=220)" in skips[0]
    eng = _Recorder()                                                      # capacity + grow: one reserve up front, then growth
    trainer.train(1, eng, iter(_buckets()), num_iterations=100, logdir=str(tmp_path / "ld3"), global_step=0, log=lambda *_: None,
                  capacity=(190, 220), beyond_capacity="grow")
    assert eng.reserves == [(190, 220), (256, 256)] and len(eng.calls) == len(SHAPES)


def test_capacity_within_the_table_reserves_nothing(tmp_path):
    eng = _Recorder()
    trainer.train(1, eng, iter(_buckets()[:2]), logdir=str(tmp_path / "ld"), global_step=0, log=lambda *_: None, capacity=(100, 100),
                  beyond_capacity="grow")
    assert eng.reserves == [(192, 210)]


def test_bad_options_are_refused(tmp_path):
    with pytest.raises(ValueError, match="beyond_capacity"):
        trainer.train(1, _Recorder(), iter(_buckets()), logdir=str(tmp_path / "a"), beyond_capacity="pad")
    with pytest.raises(ValueError, match="capacity"):
        trainer.train(1, _Recorder(), iter(_buckets()), logdir=str(tmp_path / "b"), capacity=(0, 100))


def test_graph_train_grows():
    from dc_tts_b200.train import Graph, Session
    for num in (1, 2):
        eng = _Recorder()
        g = Graph(num=num, engine=eng, batches=iter(_buckets()), global_step=10, beyond_capacity="grow")
        with Session() as sess:
            for _ in range(len(SHAPES)):
                sess.run([g.global_step, g.train_op])
        assert g.skipped_batches == 0 and g.global_step_value == 10 + len(SHAPES) and eng.inits == 1
        assert eng.reserves == ([(192, 210), (192, 256), (256, 256)] if num == 1 else [(0, 256)])
        eng = _Recorder()
        g = Graph(num=num, engine=eng, batches=iter(_buckets()), capacity=(256, 256))
        with Session() as sess:
            for _ in range(len(SHAPES)):
                sess.run(g.train_op)
        assert g.skipped_batches == 0 and eng.reserves == [(256, 256) if num == 1 else (0, 256)]
    eng = _Recorder()
    g = Graph(num=1, engine=eng, batches=iter(_buckets()))                 # the default still skips
    with Session() as sess:
        sess.run(g.train_op); sess.run(g.train_op)
    assert g.skipped_batches == 3 and len(eng.calls) == 2                 # (187, 171), (60, 215), (190, 215) before (180, 210)
    with pytest.raises(StopIteration):
        sess.run(g.train_op)
    assert g.skipped_batches == len(SHAPES) - 2 and not eng.reserves
