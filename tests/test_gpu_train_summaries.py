"""Forward-only evaluations of the training graph on the GPU (Engine.train_eval / train_eval_ssrn, dctts_train_eval*): the
bucket-shape oracle's losses, Y, alignments and Z on both training kernel sets (train_tc 7: wgmma, 0: fp32 CUDA cores);
the step's losses; the training state left bit for bit as it was; the capacity check; Graph(mode="train") fetches of
alignments and merged; and trainer.train(..., summaries=True) end to end."""
import os

import numpy as np
import pytest
import torch

from dc_tts_b200 import summary, trainer
from dc_tts_b200.hyperparams import Hyperparams as hp
from dc_tts_b200.params import init_params, synthetic_bucket
from oracle import ref_train as rtr

import ref_train_bucket as rtb
from sample_rates import at_rate

pytestmark = pytest.mark.gpu
LOSSES = ("loss", "loss_mels", "loss_bd1", "loss_att")
SSRN_LOSSES = ("loss", "loss_mags", "loss_bd2")
Y_TOL, ALIGN_TOL, Z_TOL = 1e-5, 1e-5, 1e-5        # DESIGN.md 8f, with the worst values measured


def _engine(P, tc, hparams=hp):
    from dc_tts_b200.engine import Engine
    e = Engine(0, hparams=hparams)
    e.load_params(P)
    e.set_option("train_tc", tc)
    return e


def _tie_free_t2m(P):
    from test_train import _tie_free
    return _tie_free(P)


def _tie_free_ssrn(P):
    from test_train_bucketed import _tie_free_ssrn
    return _tie_free_ssrn(P)


T2M_SHAPES = [(2, 37, 53), (3, 101, 149), (32, 123, 171), (2, hp.max_N, hp.max_T), (2, 197, 230)]


@pytest.mark.parametrize("rate", [0.05, 0.0])
@pytest.mark.parametrize("B,N,T", T2M_SHAPES)
def test_train_eval_vs_oracle(B, N, T, rate):
    """Losses within the step tests' 1e-5; Y and alignments elementwise within Y_TOL / ALIGN_TOL; the last shape is past
    the capacity on a grown handle."""
    P = _tie_free_t2m(init_params(0, "perturbed"))
    L, mels = synthetic_bucket(B, N, T, seed=N)
    W = {n: torch.tensor(np.asarray(P[n], np.float32)) for n in rtr.text2mel_names()}
    with torch.no_grad():
        o = rtb.forward(W, L, mels, seed=5, rate=rate)
    for tc in (7, 0):
        eng = _engine(P, tc)
        eng.train_init(B, rate)
        if N > hp.max_N or T > hp.max_T:
            eng.train_reserve(N, T)
        losses, t = eng.train_eval(L, mels, seed=5)
        for k in LOSSES:
            assert abs(losses[k] - float(o[k])) < 1e-5 * max(1.0, abs(float(o[k]))), (tc, k, losses[k], float(o[k]))
        assert tuple(t["Y"].shape) == (B, T, hp.n_mels) and tuple(t["alignments"].shape) == (B, N, T)
        dy = float(np.abs(t["Y"].cpu().numpy() - o["Y"].numpy()).max())
        da = float(np.abs(t["alignments"].cpu().numpy() - o["alignments"].numpy()).max())
        print("train_eval B=%d N=%d T=%d rate=%g train_tc=%d: max|dY| %.2e max|dA| %.2e" % (B, N, T, rate, tc, dy, da))
        assert dy < Y_TOL and da < ALIGN_TOL, (tc, dy, da)
        eng.close()


@pytest.mark.parametrize("F,sr", [(513, 16000), (1025, hp.sr), (2049, 44100)])
@pytest.mark.parametrize("T", [9, 53, 210])
def test_train_eval_ssrn_vs_oracle(F, sr, T):
    B, rate = 2, 0.05
    with at_rate(sr) as H:
        P = _tie_free_ssrn(init_params(0, "perturbed"))
        mels = np.random.default_rng(T).uniform(0, 1, (B, T, hp.n_mels)).astype(np.float32)
        mags = np.random.default_rng(T + 1).uniform(0, 1, (B, 4 * T, F)).astype(np.float32)
        W = {n: torch.tensor(np.asarray(P[n], np.float32)) for n in rtr.ssrn_names()}
        with torch.no_grad():
            o = rtr.forward_ssrn(W, mels, mags, 9, rate)
        for tc in (7, 0):
            eng = _engine(P, tc, H)
            eng.train_init_ssrn(B, hp.max_T, rate)
            if T > hp.max_T:
                eng.train_reserve(0, T)
            losses, t = eng.train_eval_ssrn(mels, mags, seed=9)
            for k in SSRN_LOSSES:
                assert abs(losses[k] - float(o[k])) < 1e-5 * max(1.0, abs(float(o[k]))), (F, tc, k, losses[k], float(o[k]))
            assert tuple(t["Z"].shape) == (B, 4 * T, F)
            dz = float(np.abs(t["Z"].cpu().numpy() - o["Z"].numpy()).max())
            print("train_eval_ssrn F=%d T=%d train_tc=%d: max|dZ| %.2e" % (F, T, tc, dz))
            assert dz < Z_TOL, (F, T, tc, dz)
            eng.close()


def _state(eng, names):
    """Every variable, Adam m and v, and the gradient arena, copied to the host."""
    s = {(n, w): eng.train_tensor(n, w) for n in names for w in ("param", "m", "v")}
    s["grads"] = eng.train_grads().cpu().numpy()
    return s


def _assert_same_state(x, y):
    for k in x:
        assert np.array_equal(x[k], y[k]), k


def _eval_keeps_state(a, b, names, step, evaluate, apply, tol=1e-5):
    """a and b hold the same trained state.  On a: step(apply=False) -> eval -> train_apply, with the whole state (variables,
    m, v, gradient arena) compared bit for bit across the eval -- the data-parallel window -- and the eval's losses equal
    to the step's on the same batch and seed.  Then the next step on a and on b (which never evaluated) agree to `tol`,
    the run-to-run spread of the step's float atomics."""
    ev = evaluate(a, 0)
    st = step(a, 0, False)
    for k in st:
        assert abs(ev[k] - st[k]) <= 1e-6 * max(1.0, abs(st[k])), (k, ev[k], st[k])
    before = _state(a, names)
    evaluate(a, 1)
    _assert_same_state(before, _state(a, names))
    apply(a)
    step(b, 0, True)
    la, lb = step(a, 2, True), step(b, 2, True)
    for k in la:
        assert abs(la[k] - lb[k]) <= tol * max(1.0, abs(lb[k])), (k, la[k], lb[k])
    sa, sb = _state(a, names), _state(b, names)
    for k in sa:
        assert np.abs(sa[k] - sb[k]).max() <= 1e-4 * max(np.abs(sb[k]).max(), 1e-12), k


@pytest.mark.parametrize("tc", [7, 0])
def test_eval_losses_equal_the_step_and_leave_the_state(tc):
    P = _tie_free_t2m(init_params(0, "perturbed"))
    a, b = _engine(P, tc), _engine(P, tc)
    for e in (a, b):
        e.train_init(2, 0.05)
    batches = [synthetic_bucket(2, N, T, seed=i) for i, (N, T) in enumerate(((61, 97), (150, 200), (88, 120)))]

    def step(e, i, apply):
        return e.train_step(*batches[i], global_step=4 + i, seed=4 + i, apply=apply)

    def evaluate(e, i):
        return e.train_eval(*batches[i], seed=4 + i if i == 0 else trainer.EVAL_SEED)[0]
    _eval_keeps_state(a, b, rtr.text2mel_names(), step, evaluate, lambda e: e.train_apply(4))
    a.close(); b.close()


@pytest.mark.parametrize("tc", [7, 0])
def test_ssrn_eval_leaves_the_state(tc):
    P = _tie_free_ssrn(init_params(0, "perturbed"))
    a, b = _engine(P, tc), _engine(P, tc)
    for e in (a, b):
        e.train_init_ssrn(2, hp.max_T, 0.05)
    rng = np.random.default_rng(1)
    batches = [(rng.uniform(0, 1, (2, T, hp.n_mels)).astype(np.float32),
                rng.uniform(0, 1, (2, 4 * T, 1 + hp.n_fft // 2)).astype(np.float32)) for T in (40, 53, 30)]

    def step(e, i, apply):
        return e.train_step_ssrn(*batches[i], global_step=1 + i, seed=1 + i, apply=apply)

    def evaluate(e, i):
        return e.train_eval_ssrn(*batches[i], seed=1 + i if i == 0 else trainer.EVAL_SEED)[0]
    _eval_keeps_state(a, b, rtr.ssrn_names(), step, evaluate, lambda e: e.train_apply(1))
    a.close(); b.close()


def test_eval_beyond_the_capacity_fails_before_launching():
    from dc_tts_b200.engine import DcttsError
    P = init_params(0, "perturbed")
    e = _engine(P, 7)
    e.train_init(2, 0.0)
    L, mels = synthetic_bucket(2, hp.max_N + 1, 53, seed=1)
    n0 = e.launch_count()
    with pytest.raises(DcttsError) as step_err:
        e.train_step(L, mels, apply=False)
    with pytest.raises(DcttsError) as eval_err:
        e.train_eval(L, mels)
    assert e.launch_count() == n0
    assert str(eval_err.value).split(": ", 1)[1] == str(step_err.value).split(": ", 1)[1]
    e.close()
    s = _engine(P, 7)
    s.train_init_ssrn(2, 20, 0.0)
    mels = np.zeros((2, 21, hp.n_mels), np.float32); mags = np.zeros((2, 84, 1 + hp.n_fft // 2), np.float32)
    n0 = s.launch_count()
    with pytest.raises(DcttsError, match="outside the handle's capacity"):
        s.train_eval_ssrn(mels, mags)
    assert s.launch_count() == n0
    s.close()


def test_graph_train_mode_fetches_alignments_and_merged():
    from dc_tts_b200.engine import Engine
    from dc_tts_b200.train import Graph, Session
    P = init_params(0, "perturbed")
    e = Engine(0); e.load_params(P)
    shapes = [(37, 53), (61, 80), (44, 70), (90, 120)]
    consumed = []

    def batches():
        for i, (N, T) in enumerate(shapes):
            consumed.append(i)
            L, mels = synthetic_bucket(2, N, T, seed=i)
            yield L, mels, None
    g = Graph(1, mode="train", engine=e, batches=batches())
    with Session() as sess:
        A = sess.run(g.alignments)
        assert A.shape == (2, 37, 53) and consumed == [0] and int(sess.run(g.global_step)) == 0
        gs, _ = sess.run([g.global_step, g.train_op])
        assert gs == 1 and consumed == [0, 1]
        merged = sess.run(g.merged)
        assert consumed == [0, 1, 2] and int(sess.run(g.global_step)) == 1
        assert [t for t, _ in summary.parse_summary(merged)] == [
            "train/loss_mels", "train/loss_bd1", "train/loss_att", "train/mel_gt/image/0", "train/mel_hat/image/0", "lr"]
        with pytest.raises(ValueError, match="train_op"):
            sess.run([g.train_op, g.alignments])
    e.close()


def _write_dataset(tmp_path):
    from test_gpu_trainer_run import _write_dataset as w
    return w(tmp_path)


@pytest.mark.parametrize("num", [1, 2])
def test_trainer_summaries_end_to_end(tmp_path, num):
    from dc_tts_b200.engine import Engine
    d = _write_dataset(tmp_path)
    fpaths, lens, texts = trainer.load_train_data(d)
    loader = lambda p: trainer._load_spectrograms_npy(p, str(tmp_path / "mels"), str(tmp_path / "mags"))
    P = init_params(1)
    eng = Engine(0); eng.load_params(P)
    logdir = str(tmp_path / ("logdir/LJ01-%d" % num))
    gs = trainer.train(num, eng, trainer.bucketed_batches(fpaths, lens, texts, B=2, seed=0, loader=loader), num_iterations=1000,
                       logdir=logdir, log=lambda s: None, summaries=True, summary_secs=0)
    assert gs == 1001
    files = sorted(f for f in os.listdir(logdir) if f.startswith("events.out.tfevents."))
    assert len(files) == 1
    ev = summary.read_events(os.path.join(logdir, files[0]))
    assert ev[0]["file_version"] == "brain.Event:2"
    assert [e["step"] for e in ev[1:]] == list(range(1, 1002))
    want = (["train/loss_mels", "train/loss_bd1", "train/loss_att", "train/mel_gt/image/0", "train/mel_hat/image/0"] if num == 1
            else ["train/loss_mags", "train/loss_bd2", "train/mag_gt/image/0", "train/mag_hat/image/0"]) + ["lr", "global_step/sec"]
    for e in ev[1:]:
        assert [t for t, _ in e["summary"]] == want
    assert os.path.exists(os.path.join(logdir, "alignment_001k.png")) == (num == 1)
    # a resumed run opens a second event file and counts on from the restored step
    gs2 = trainer.train(num, eng, trainer.bucketed_batches(fpaths, lens, texts, B=2, seed=1, loader=loader), num_iterations=1002,
                        logdir=logdir, log=lambda s: None, summaries=True, summary_secs=0)
    assert gs2 == 1003
    new = sorted(f for f in os.listdir(logdir) if f.startswith("events.out.tfevents.") and f != files[0])
    assert len(new) == 1, new
    ev2 = summary.read_events(os.path.join(logdir, new[0]))
    assert [e["step"] for e in ev2[1:]] == [1001, 1002, 1003]
    eng.close()
