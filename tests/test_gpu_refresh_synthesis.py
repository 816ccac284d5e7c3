"""Synthesis from the weights being trained (Engine.refresh_synthesis, include/dctts.h: dctts_refresh_synthesis).

A handle trained a few steps and refreshed computes, bit for bit, what a fresh handle loaded with its variables computes,
on the same kernels (wgmma blocks, persistent decode); the refresh touches nothing of training; every call that writes a
variable makes the packing stale again, and synthesis then runs on the fp32 kernels with the graph-per-frame decode."""
import numpy as np
import pytest
import torch

from dc_tts_b200 import arch
from dc_tts_b200.hyperparams import Hyperparams as hp
from dc_tts_b200.params import init_params, synthetic_text

from sample_rates import at_rate
from test_train import _batch, _tie_free

pytestmark = pytest.mark.gpu
STALE = "this handle has been trained"


def _names(scope):
    return [n for n in arch.param_shapes() if n.startswith(scope + "/")]


def _engine(P, H=hp):
    from dc_tts_b200.engine import Engine
    e = Engine(0, hparams=H)
    e.load_params(P)
    return e


def _ssrn_batch(B, T, F, seed=3):
    mels = np.random.default_rng(seed).uniform(0, 1, (B, T, hp.n_mels)).astype(np.float32)
    mags = np.random.default_rng(seed + 1).uniform(0, 1, (B, 4 * T, F)).astype(np.float32)
    return mels, mags


def _trained(num, P, train_tc, H=hp, steps=3, reserve=None):
    """(handle trained `steps` steps, the parameters with its trained variables in place)."""
    e = _engine(P, H)
    e.set_option("train_tc", train_tc)
    if num == 1:
        e.train_init(2)
        L, mels = _batch(2)
        for i in range(steps):
            e.train_step(L, mels, global_step=4000 + i, seed=i)
    else:
        F = 1 + H.n_fft // 2
        e.train_init_ssrn(2, 16)
        T = 16
        if reserve:
            e.train_reserve(0, reserve)
            T = reserve
        mels, mags = _ssrn_batch(2, T, F)
        for i in range(steps):
            e.train_step_ssrn(mels, mags, global_step=4000 + i, seed=i)
    Q = dict(P)
    for n in _names("Text2Mel" if num == 1 else "SSRN"):
        Q[n] = e.train_tensor(n, "param")
    return e, Q


def _synth(e, L, ragged=True):
    """Everything synthesis computes: the cluster decode, the decode until EOS, SSRN at full length and ragged."""
    Y, P, _, _ = e.text2mel_generate(L)
    Yu, Pu, n = e.text2mel_generate_until(L)
    out = {"Y": Y, "P": P, "Yu": Yu, "Pu": Pu, "n": n}
    out["Zl"], out["Z"] = e.ssrn(Y[:, :40])
    if ragged:
        m = torch.clamp(n, max=40)
        out["Zrl"], out["Zr"] = e.ssrn(Yu[:, :40], lengths=m)
    torch.cuda.synchronize()
    return out


def _assert_equal(a, b):
    for k in a:
        assert torch.equal(a[k], b[k]), k


def _kernels(e):
    return e.get_option("decode_available"), e.get_option("ssrn_tc_available")


@pytest.mark.parametrize("train_tc", [0, 7])
@pytest.mark.parametrize("num", [1, 2])
def test_refresh_equals_commit(num, train_tc):
    P = _tie_free(init_params(0, "perturbed"))
    A, Q = _trained(num, P, train_tc)
    B = _engine(Q)
    L = synthetic_text(3, 30, seed=2)
    with pytest.raises(RuntimeError, match=STALE):
        A.set_tensor_path(1)
    A.refresh_synthesis()
    assert _kernels(A) == _kernels(B) and A.get_option("decode_available") == 1
    A.set_tensor_path(1)                                        # accepted again
    _assert_equal(_synth(A, L), _synth(B, L))
    A.close(); B.close()


@pytest.mark.parametrize("sr,reserve", [(16000, None), (22050, None), (22050, 48), (44100, None), (44100, 48)])
def test_refresh_equals_commit_ssrn_widths(sr, reserve):
    """SSRN trained at F = 513, 1025 and 2049 (the 16-CTA 144-column planes), on a grown workspace as well."""
    with at_rate(sr) as H:
        P = init_params(0, "perturbed")
        A, Q = _trained(2, P, 7, H, reserve=reserve)
        B = _engine(Q, H)
        A.refresh_synthesis()
        assert _kernels(A) == _kernels(B)
        Y = torch.rand(3, 40, hp.n_mels, device="cuda", generator=torch.Generator("cuda").manual_seed(5))
        n = torch.tensor([40, 7, 23], dtype=torch.int32, device="cuda")
        for e in (A, B):
            e.set_tensor_path(1)
        za = A.ssrn(Y) + A.ssrn(Y, lengths=n)
        zb = B.ssrn(Y) + B.ssrn(Y, lengths=n)
        for x, y in zip(za, zb):
            assert torch.equal(x, y)
        A.close(); B.close()


def _state(e, names):
    return {(n, w): e.train_tensor(n, w) for n in names for w in ("param", "m", "v")}


def test_refresh_leaves_training_state():
    P = _tie_free(init_params(0, "perturbed"))
    A, _ = _trained(1, P, 7, steps=2)
    names = _names("Text2Mel")
    L, mels = _batch(2)
    A.train_step(L, mels, global_step=4002, seed=2, apply=False)
    before, grads = _state(A, names), A.train_grads().clone()
    A.refresh_synthesis()
    _synth(A, synthetic_text(2, 30, seed=4))
    after = _state(A, names)
    for k in before:
        assert np.array_equal(before[k], after[k]), k
    assert torch.equal(A.train_grads(), grads)                  # a refresh between apply=False and train_apply changes nothing
    A.train_apply(4002)
    with pytest.raises(RuntimeError, match=STALE):
        A.set_tensor_path(1)
    A.close()


def test_next_step_agrees_with_a_handle_that_never_sampled():
    P = _tie_free(init_params(0, "perturbed"))
    A, _ = _trained(1, P, 7, steps=2)
    C, _ = _trained(1, P, 7, steps=2)
    A.refresh_synthesis()
    _synth(A, synthetic_text(2, 30, seed=4))
    L, mels = _batch(2)
    la = A.train_step(L, mels, global_step=4002, seed=2)
    lc = C.train_step(L, mels, global_step=4002, seed=2)
    for k in la:
        assert abs(la[k] - lc[k]) <= 1e-5 * max(1.0, abs(lc[k])), (k, la[k], lc[k])
    for n in _names("Text2Mel")[::7]:
        assert np.abs(A.train_tensor(n, "param") - C.train_tensor(n, "param")).max() <= 1e-4, n
    A.close(); C.close()


@pytest.mark.parametrize("writer", ["train_step", "train_step_ssrn", "train_apply", "train_set_tensor", "restore_training"])
def test_each_variable_writer_makes_it_stale(writer, tmp_path):
    P = _tie_free(init_params(0, "perturbed"))
    num = 2 if writer == "train_step_ssrn" else 1
    A, Q = _trained(num, P, 7, steps=1)
    if writer == "restore_training":
        A.save_checkpoint(str(tmp_path / "model_gs_000k"), 1, "Text2Mel")
    A.refresh_synthesis()
    assert A.get_option("decode_available") == 1
    L, mels = _batch(2)
    if writer == "train_step":
        A.train_step(L, mels, global_step=4001, seed=1)
    elif writer == "train_step_ssrn":
        A.train_step_ssrn(*_ssrn_batch(2, 16, 1 + hp.n_fft // 2), global_step=4001, seed=1)
    elif writer == "train_apply":
        A.train_step(L, mels, global_step=4001, seed=1, apply=False)
        A.train_apply(4001)
    elif writer == "train_set_tensor":
        n = "Text2Mel/AudioDec/C_11/conv1d/bias"
        A.train_set_tensor(n, Q[n] + 0.01)
    else:
        assert A.restore_training(str(tmp_path)) == 1
    with pytest.raises(RuntimeError, match=STALE):
        A.set_tensor_path(1)
    assert A.get_option("decode_available") == 0
    # synthesis = a handle with the same weights on the fp32 kernels and the graph-per-frame decode
    R = dict(P)
    for n in _names("Text2Mel" if num == 1 else "SSRN"):
        R[n] = A.train_tensor(n, "param")
    D = _engine(R)
    D.set_tensor_path(0)
    D.set_option("decode_mode", 0)
    Ls = synthetic_text(2, 20, seed=6)
    ya, pa, _, _ = A.text2mel_generate(Ls, steps=24)
    yd, pd, _, _ = D.text2mel_generate(Ls, steps=24)
    assert torch.equal(ya, yd) and torch.equal(pa, pd)
    assert torch.equal(A.ssrn(ya[:, :12])[1], D.ssrn(yd[:, :12])[1])
    A.close(); D.close()


def test_unapplied_step_and_evaluation_keep_the_refresh():
    P = _tie_free(init_params(0, "perturbed"))
    A, Q = _trained(1, P, 7, steps=1)
    A.refresh_synthesis()
    L, mels = _batch(2)
    A.train_step(L, mels, global_step=4001, seed=1, apply=False)
    A.train_eval(L, mels)
    A.set_tensor_path(1)
    assert A.get_option("decode_available") == 1
    B = _engine(Q)
    Ls = synthetic_text(2, 30, seed=2)
    _assert_equal(_synth(A, Ls), _synth(B, Ls))
    A.close(); B.close()


def test_refresh_on_an_untrained_handle_changes_nothing():
    P = init_params(0, "perturbed")
    A = _engine(P)
    L = synthetic_text(2, 30, seed=2)
    before = _synth(A, L)
    A.refresh_synthesis()
    _assert_equal(before, _synth(A, L))
    A.close()


def test_trainer_writes_samples_at_checkpoints(tmp_path):
    from dc_tts_b200 import summary, trainer
    from dc_tts_b200.utils import spectrograms2wavs
    P = init_params(0, "perturbed")
    e = _engine(P)
    L, mels = _batch(2)
    mags = np.zeros((2, 4 * hp.max_T, 1 + hp.n_fft // 2), np.float32)
    batches = [(L, mels, mags)] * 8
    sents = ["The birch canoe slid on the smooth planks.", "Glue the sheet to the dark blue background.", "A pot of tea helps."]
    gs = trainer.train(1, e, batches, num_iterations=3, logdir=str(tmp_path), save_every=2, log=lambda *_: None,
                       summaries=True, summary_secs=1e9, samples=sents)
    assert gs == 4
    for k in ("000k",):
        d = tmp_path / ("samples_" + k)
        assert sorted(p.name for p in d.iterdir()) == ["1.wav", "2.wav", "3.wav", "alignment_1.png", "alignment_2.png", "alignment_3.png"]
    # the last checkpoint's samples: the same wavs as spectrograms2wavs of the Z computed directly from the handle
    texts = trainer.sample_texts(sents)
    wavs, lengths = trainer.write_samples(e, texts, str(tmp_path / "again"), 4)
    Y, _, n = e.text2mel_generate_until(texts)
    assert np.array_equal(n.cpu().numpy(), lengths)
    _, Z = e.ssrn(Y[:, :int(lengths.max())], want_logits=False, lengths=n)
    direct = spectrograms2wavs(Z, lengths=hp.r * lengths, engine=e)
    assert [len(w) for w in wavs] == [len(w) for w in direct]
    from scipy.io import wavfile
    for i, w in enumerate(direct):
        sr, data = wavfile.read(str(tmp_path / "samples_000k" / ("%d.wav" % (i + 1))))
        assert sr == hp.sr and len(data) == len(w)
    ev = [x for p in tmp_path.glob("events.out.tfevents.*") for x in summary.read_events(str(p)) if "summary" in x]
    steps = [x["step"] for x in ev if any(t.startswith("samples/") for t, _ in x["summary"])]
    assert steps == [2, 4]
    e.close()


def test_trainer_without_samples_writes_what_it_wrote_before(tmp_path):
    from dc_tts_b200 import trainer
    e = _engine(init_params(0, "perturbed"))
    L, mels = _batch(2)
    mags = np.zeros((2, 4 * hp.max_T, 1 + hp.n_fft // 2), np.float32)
    trainer.train(1, e, [(L, mels, mags)] * 4, num_iterations=1, logdir=str(tmp_path), save_every=2, log=lambda *_: None)
    names = [p.name for p in tmp_path.iterdir()]
    assert "checkpoint" in names and not [n for n in names if n.startswith(("samples_", "events.", "alignment_"))], names
    # and the handle was never refreshed: still on the fp32 kernels
    with pytest.raises(RuntimeError, match=STALE):
        e.set_tensor_path(1)
    e.close()
