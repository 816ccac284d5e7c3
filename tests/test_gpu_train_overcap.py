"""Training past (max_N, max_T) on the GPU, on both training kernel sets (train_tc 7: wgmma, 0: fp32 CUDA cores), with the
workspace grown in place by Engine.train_reserve.  The steps against the bucket-shape oracle (tests/ref_train_bucket.py,
pinned to the reference's own graphs by refshim_train_overcap.npz), the optimiser state across a growth, in-table steps on
a grown handle, SSRN past max_T, and the trainer end to end on a wav corpus of long texts and clips."""
import os
import sys

import numpy as np
import pytest

from conftest import ROOT, golden
from dc_tts_b200 import trainer
from dc_tts_b200.hyperparams import Hyperparams as hp
from dc_tts_b200.params import init_params, synthetic_bucket
from oracle import ref_train as rtr

import ref_train_bucket as rtb

sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_golden_refchecks_overcap import T2M_CASES, train_inputs      # noqa: E402

pytestmark = pytest.mark.gpu
LOSSES = ("loss", "loss_mels", "loss_bd1", "loss_att")


def _engine(P, tc=7):
    from dc_tts_b200.engine import Engine
    e = Engine(0)
    e.load_params(P)
    e.set_option("train_tc", tc)
    return e


def _tie_free_t2m(P):
    from test_train import _tie_free
    return _tie_free(P)


CASES = [(tag, B, N, T, seed, rate) for tag, B, N, T, seed, rate in T2M_CASES] + \
        [(None, 2, 193, 53, 3, 0.05), (None, 32, 190, 215, 6, 0.05)]


@pytest.mark.parametrize("tag,B,N,T,seed,rate", CASES)
def test_cuda_step_past_the_table_vs_oracle(tag, B, N, T, seed, rate):
    """Losses within 1e-5 and every gradient within 2e-3 of its max-norm of the oracle, at the fixture's shapes (whose
    losses are the reference's), at N_b = 193 (past a 64-key block) and at B = 32."""
    from test_train import _compare_grads
    P = _tie_free_t2m(init_params(0, "perturbed"))
    L, mels = train_inputs(B, N, T) if tag else synthetic_bucket(B, N, T, seed=seed)
    _, _, info = rtb.train_step(P, L, mels, global_step=7, seed=seed, rate=rate)
    if tag:                                                       # the plain set's fixture: same inputs, the reference's losses
        g = golden("refshim_train_overcap.npz")
        P0 = init_params(0, "perturbed")
        e = _engine(P0, 0)
        e.train_init(B, rate)
        e.train_reserve(N, T)
        out = e.train_step(L, mels, global_step=7, seed=seed, apply=False)
        for i, k in enumerate(LOSSES):
            assert abs(out[k] - g[tag][i]) < 1e-5 * max(1.0, abs(g[tag][i])), (tag, k, out[k], g[tag][i])
        e.close()
    for tc in (7, 0):
        eng = _engine(P, tc)
        eng.train_init(B, rate)
        eng.train_reserve(N, T)
        assert eng.train_capacity() == (max(N, hp.max_N), max(T, hp.max_T))
        out = eng.train_step(L, mels, global_step=7, seed=seed, apply=False)
        for k in LOSSES:
            assert abs(out[k] - info[k]) < 1e-5 * max(1.0, abs(info[k])), (tc, k, out[k], info[k])
        _compare_grads(eng, info["grads"])
        eng.close()


def _state(eng, names):
    return {n: tuple(eng.train_tensor(n, w) for w in ("param", "m", "v")) for n in names}


@pytest.mark.parametrize("tc", [7, 0])
def test_growth_keeps_the_optimiser_state(tc):
    """Three applied steps at the default capacity, then a reserve: every variable, m and v is bit-identical and the
    gradient arena keeps its address.  The next steps -- in the table and past it -- match a handle given the same state
    (within the float-atomic reordering the step has from run to run)."""
    P = _tie_free_t2m(init_params(0, "perturbed"))
    names = rtr.text2mel_names()
    eng = _engine(P, tc)
    eng.train_init(2, 0.05)
    for i, (N, T) in enumerate(((37, 53), (120, 171), (hp.max_N, hp.max_T))):
        L, mels = synthetic_bucket(2, N, T, seed=i)
        eng.train_step(L, mels, global_step=4000 + i, seed=i)
    assert eng.train_capacity() == (hp.max_N, hp.max_T)
    before, addr = _state(eng, names), eng.train_grads().data_ptr()
    eng.train_reserve(256, 256)
    eng.train_reserve(200, 100)                                   # never shrinks: a no-op
    assert eng.train_capacity() == (256, 256) and eng.train_grads().data_ptr() == addr
    after = _state(eng, names)
    for n in names:
        for x, y in zip(before[n], after[n]):
            assert np.array_equal(x, y), n

    def loaded(reserve):
        e = _engine(P, tc)
        e.train_init(2, 0.05)
        if reserve:
            e.train_reserve(256, 256)
        for n in names:
            for w, a in zip(("param", "m", "v"), before[n]):
                e.train_set_tensor(n, a, w)
        return e
    for (N, T), reserve in (((37, 53), False), ((200, 240), True), ((hp.max_N, hp.max_T), True)):
        other = loaded(reserve)
        L, mels = synthetic_bucket(2, N, T, seed=N)
        a = eng.train_step(L, mels, global_step=4003, seed=9, apply=False)
        b = other.train_step(L, mels, global_step=4003, seed=9, apply=False)
        for k in LOSSES:
            assert abs(a[k] - b[k]) <= 1e-5 * max(1.0, abs(b[k])), (N, T, k, a[k], b[k])
        for n in names:
            x, y = eng.train_tensor(n, "grad"), other.train_tensor(n, "grad")
            assert np.abs(x - y).max() <= 1e-4 * max(np.abs(y).max(), 1e-12), (N, T, n)
        other.close()
    eng.close()


def test_growth_refused_beyond_memory_keeps_the_handle():
    """A reserve the device cannot hold fails with a message and leaves the old capacity; training goes on."""
    from dc_tts_b200.engine import DcttsError
    P = init_params(0, "perturbed")
    eng = _engine(P)
    eng.train_init(2, 0.0)
    eng.train_reserve(200, 240)
    with pytest.raises(DcttsError):
        eng.train_reserve(2 ** 30, 2 ** 30)
    assert eng.train_capacity() == (200, 240)
    L, mels = synthetic_bucket(2, 200, 240, seed=1)
    out = eng.train_step(L, mels, apply=False)
    assert np.isfinite(out["loss"])
    eng.close()


@pytest.mark.parametrize("tc", [7, 0])
def test_cuda_ssrn_grown_past_max_t_vs_oracle(tc):
    from test_train import _compare_grads
    from test_train_bucketed import _tie_free_ssrn
    P = _tie_free_ssrn(init_params(0, "perturbed"))
    eng = _engine(P, tc)
    eng.train_init_ssrn(2, hp.max_T, 0.05)
    assert eng.train_capacity() == (0, hp.max_T)
    eng.train_reserve(0, 300)
    assert eng.train_capacity() == (0, 300)
    for T in (233, 300):
        mels = np.random.default_rng(T).uniform(0, 1, (2, T, hp.n_mels)).astype(np.float32)
        mags = np.random.default_rng(T + 1).uniform(0, 1, (2, 4 * T, 1 + hp.n_fft // 2)).astype(np.float32)
        _, _, info = rtr.train_step_ssrn(P, mels, mags, global_step=7, seed=T, rate=0.05)
        out = eng.train_step_ssrn(mels, mags, global_step=7, seed=T, apply=False)
        for k in ("loss", "loss_mags", "loss_bd2"):
            assert abs(out[k] - info[k]) < 1e-5 * max(1.0, abs(info[k])), (tc, T, k, out[k], info[k])
        _compare_grads(eng, info["grads"])
    eng.close()


def _long_corpus(root, n=12, seed=0):
    """LJ-format corpus: texts of 181..200 characters, clips of 11..14 s -- every batch is past (max_N, max_T)."""
    from scipy.io import wavfile
    from test_gpu_wav_features import _as, _speechlike
    rng = np.random.default_rng(seed)
    d = root / "LJSpeech-1.0"
    (d / "wavs").mkdir(parents=True)
    lines = []
    for i in range(n):
        nchar = int(rng.integers(181, 201))
        lines.append("LJ%03d|raw|%s" % (i, "".join(rng.choice(list("abcdefghijklmnopqrstuvwxyz"), nchar))))
        y = _speechlike(200 + i, int(float(rng.uniform(11.0, 14.0)) * hp.sr), 300, 300)
        wavfile.write(str(d / "wavs" / ("LJ%03d.wav" % i)), hp.sr, _as(y, "int16"))
    (d / "transcript.csv").write_text("\n".join(lines) + "\n", encoding="utf-8")
    return str(d)


def test_trainer_grows_on_long_wav_corpus_end_to_end(tmp_path):
    from dc_tts_b200.checkpoint import latest_checkpoint
    from dc_tts_b200.engine import Engine
    d = _long_corpus(tmp_path)
    fpaths, lens, texts = trainer.load_train_data(d)
    assert min(lens) > hp.max_N
    feat = Engine(0)
    shapes = []

    def counted(batches):
        for b in batches:
            shapes.append((b[0].shape[1], b[1].shape[1]))
            yield b
    P = init_params(1)
    logdir = str(tmp_path / "logdir" / "LJ01-1")
    eng = Engine(0); eng.load_params(P)
    log = []
    gs = trainer.train(1, eng, counted(trainer.bucketed_batches(fpaths, lens, texts, B=2, seed=0, epochs=1, prepro=False, engine=feat)),
                       num_iterations=10 ** 6, logdir=logdir, save_every=1, log=log.append, beyond_capacity="grow")
    assert shapes and all(N > hp.max_N and T > hp.max_T for N, T in shapes), shapes
    assert gs == len(shapes) and not [s for s in log if s.startswith("skipped")]
    grew = [s for s in log if s.startswith("grew")]
    assert grew and eng.train_capacity()[0] >= max(N for N, _ in shapes) and eng.train_capacity()[1] >= max(T for _, T in shapes)
    assert latest_checkpoint(logdir) is not None
    eng.close()
    shapes.clear()
    resumed = Engine(0); resumed.load_params(P)
    more = []
    gs2 = trainer.train(1, resumed, counted(trainer.bucketed_batches(fpaths, lens, texts, B=2, seed=1, epochs=1, prepro=False, engine=feat)),
                        num_iterations=10 ** 6, logdir=logdir, save_every=10 ** 6, log=more.append, beyond_capacity="grow")
    assert any("resumed" in s and str(gs) in s for s in more)
    assert [s for s in more if s.startswith("grew")]                      # a resumed run starts at the default capacity
    assert gs2 == gs + len(shapes) and not [s for s in more if s.startswith("skipped")]
    resumed.close(); feat.close()
