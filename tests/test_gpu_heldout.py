"""Held-out evaluation on the GPU (dc_tts_b200/heldout.py): HeldOut.run at random weights on short synthetic recordings
for Text2Mel and SSRN, its MCD column against the float64 reference on the same inputs and its window checks against
the host restatement; a deterministic training run with `heldout` writes the bundles of a run without it plus the
held-out files and scalars; and the CLI evaluates the list the trainer wrote."""
import json
import os

import numpy as np
import pytest

import ref_mcd
from dc_tts_b200 import heldout as ho
from dc_tts_b200 import trainer
from dc_tts_b200.hyperparams import Hyperparams as hp
from dc_tts_b200.params import init_params

pytestmark = pytest.mark.gpu


def _write_dataset(root, n=12, seed=0):
    rng = np.random.default_rng(seed)
    d = root / "LJSpeech-1.0"
    (d / "wavs").mkdir(parents=True)
    (root / "mels").mkdir()
    (root / "mags").mkdir()
    F = 1 + hp.n_fft // 2
    lines = []
    for i in range(n):
        text = "".join(rng.choice(list("abcdefghijklmnopqrstuvwxyz '"), int(rng.integers(20, 60))))
        lines.append("LJ%03d|raw|%s" % (i, text))
        T = int(rng.integers(30, 90))
        np.save(root / "mels" / ("LJ%03d.npy" % i), rng.uniform(0, 1, (T, hp.n_mels)).astype(np.float32))
        np.save(root / "mags" / ("LJ%03d.npy" % i), rng.uniform(0, 1, (T * hp.r, F)).astype(np.float32))
    (d / "transcript.csv").write_text("\n".join(lines) + "\n", encoding="utf-8")
    return str(d)


def _engine(P=None):
    from dc_tts_b200.engine import Engine
    e = Engine(0)
    e.load_params(init_params(0, "perturbed") if P is None else P)
    return e


def _capture(obj, name, store):
    fn = getattr(obj, name)

    def wrapped(*a, **k):
        out = fn(*a, **k)
        store.append(out)
        return out
    setattr(obj, name, wrapped)


@pytest.mark.parametrize("num", [1, 2])
def test_heldout_run_against_reference(tmp_path, monkeypatch, num):
    d = _write_dataset(tmp_path, n=7)
    monkeypatch.chdir(tmp_path)
    fpaths, lens, texts = trainer.load_train_data(d)
    e = _engine()
    try:
        if num == 1:
            e.train_init(3)
        else:
            e.train_init_ssrn(3, hp.max_T)
        h = ho.HeldOut(e, fpaths, lens, texts, prepro=True, B=4)
        gen, feats = [], []
        _capture(e, "text2mel_generate_until", gen)
        _capture(e, "load_spectrograms_batch", feats)
        rows, s = h.run(e, num, 1000, train_batch=3)
    finally:
        e.close()
    assert s["evaluated"] == 7 and s["loss_batches"] == 3 and np.isfinite(list(s["losses"].values())).all()
    batches = [h.order[k:k + 4] for k in range(0, 7, 4)]
    outs = gen if num == 1 else feats
    assert len(outs) == len(batches)
    for idx, out in zip(batches, outs):
        t = np.array([h.items[i]["frames"] for i in idx])
        mels = np.zeros((len(idx), t.max(), hp.n_mels), np.float32)
        for b, i in enumerate(idx):
            mels[b, :t[b]] = h.items[i]["mel"]
        if num == 1:
            Y, P, n = (x.cpu().numpy() for x in out)
        else:
            Y, n = out[0].cpu().numpy(), np.asarray(out[2])
        ref = ref_mcd.mcd_batch(Y, n, mels, t)
        for b, i in enumerate(idx):
            r = rows[i]
            assert r["mcd"] == pytest.approx(ref["mcd"][b], rel=1e-9)
            if ref["margin"][b] > 1e-9 * ref["mcd"][b] * ref["pairs"][b]:
                assert r["pairs"] == ref["pairs"][b]
            if num == 1:
                e_b = list(h.items[i]["text"]).index(hp.vocab.index("E"))
                want = ref_mcd.window_checks(P[b], int(n[b]), e_b, int(t[b]), hp.max_T)
                assert {k: r[k] for k in want} == want and r["generated"] == n[b]
                assert np.isfinite(r["mean_log_attention"]) and r["mean_log_attention"] <= 0


def test_training_with_heldout_keeps_the_bundles(tmp_path, monkeypatch):
    from dc_tts_b200 import engine as engine_mod
    from dc_tts_b200.summary import read_events
    d = _write_dataset(tmp_path, n=14)
    monkeypatch.chdir(tmp_path)
    fpaths, lens, texts = trainer.load_train_data(d)
    train, held = ho.split_heldout(fpaths, lens, texts, 5, seed=1)
    P = init_params(1)

    def run(logdir, with_heldout):
        e = _engine(P)
        try:
            ho_set = ho.HeldOut(e, *held, prepro=True, B=4) if with_heldout else None
            batches = trainer.fixed_size_batches(train[0], train[2], B=4, seed=0)
            trainer.train(1, e, batches, num_iterations=19, logdir=logdir, save_every=10, log=lambda s: None,
                          summaries=True, summary_secs=1e9, deterministic=True, heldout=ho_set)
        finally:
            e.close()

    plain, with_ho = str(tmp_path / "plain-1"), str(tmp_path / "held-1")
    run(plain, False)
    run(with_ho, True)
    for f in sorted(os.listdir(plain)):
        if f.startswith("model_gs_") or f == "checkpoint":
            assert open(os.path.join(plain, f), "rb").read() == open(os.path.join(with_ho, f), "rb").read(), f
    new = sorted(set(os.listdir(with_ho)) - set(os.listdir(plain)))
    assert [f for f in new if not f.startswith("events.")] == ["heldout.tsv", "heldout.txt", "heldout_000k.tsv"]
    assert not any(f.startswith("heldout") for f in os.listdir(plain))
    assert open(os.path.join(with_ho, "heldout.txt")).read().split() == [os.path.basename(p) for p in held[0]]
    log = open(os.path.join(with_ho, "heldout.tsv")).read().splitlines()
    assert [l.split("\t")[0] for l in log[1:]] == ["10", "20"]
    table = open(os.path.join(with_ho, "heldout_000k.tsv")).read().splitlines()
    assert table[0].split("\t") == ho.COLUMNS[1] and len(table) == 6
    ev = [e for f in os.listdir(with_ho) if f.startswith("events.") for e in read_events(os.path.join(with_ho, f))]
    tags = {(e["step"], t) for e in ev for t, _ in e.get("summary", [])}
    assert (10, "heldout/mcd_mean") in tags and (20, "heldout/loss/loss_mels") in tags

    # the CLI on the list the trainer wrote, from the step-20 bundle
    from dc_tts_b200.engine import Engine
    fresh = Engine(0)                                        # what get_engine gives the CLI: nothing loaded yet
    monkeypatch.setattr(engine_mod, "get_engine", lambda: fresh)
    monkeypatch.setattr(ho.hp, "logdir", str(tmp_path / "held"))
    try:
        out = str(tmp_path / "cli")
        s = ho.main([d, out, "--list", os.path.join(with_ho, "heldout.txt"), "--batch", "4"])
    finally:
        fresh.close()
    assert s["global_step"] == 20 and s["evaluated"] == 5
    assert json.load(open(os.path.join(out, "summary.json")))["evaluated"] == 5
    cli = [l.split("\t") for l in open(os.path.join(out, "heldout.tsv")).read().splitlines()[1:]]
    tr = [l.split("\t") for l in table[1:]]
    assert [r[0] for r in cli] == [r[0] for r in tr]
    np.testing.assert_allclose([float(r[3]) for r in cli], [float(r[3]) for r in tr], rtol=1e-5)
