"""The held-out evaluation's host logic (dc_tts_b200/heldout.py) with a stub engine: the split, the window checks, the
skip reasons, batching, the TSV and JSON writers, the trainer's log, and the CLI's arguments."""
import json
import os

import numpy as np
import pytest
import torch

import ref_mcd
from dc_tts_b200 import heldout as ho
from dc_tts_b200.hyperparams import Hyperparams

EOS = Hyperparams.vocab.index("E")


class _StubEngine:
    """The engine calls HeldOut.run makes.  The free run of utterance b generates text_length + 1 frames with the window
    path 0, 0, 1, 2, ... (so nothing is skipped, and the first window is held two frames); its MCD is the sum of the
    recorded mels; the mean log-attention is -1 per frame; the losses are the batch's mean mel."""

    class hp(Hyperparams):
        max_N, max_T, attention_win_size, r = 12, 8, 3, 4

    device = "cpu"

    def __init__(self):
        self.calls = []
        self.refreshed = 0

    def refresh_synthesis(self):
        self.refreshed += 1

    def text2mel_generate_until(self, L):
        L = np.asarray(L)
        B = len(L)
        ends = (L == EOS).argmax(1)
        n = np.minimum(ends + 2, self.hp.max_T)
        P = np.full((B, self.hp.max_T), -1, np.int32)
        for b in range(B):
            P[b, :n[b]] = np.minimum(np.maximum(np.arange(n[b]) - 1, 0), ends[b])
        self.calls.append(("generate", L.shape))
        return torch.zeros(B, self.hp.max_T, 80), torch.from_numpy(P), torch.from_numpy(n.astype(np.int32))

    def mcd_dtw(self, X, nx, Y, ny, K=24):
        Yh = Y.cpu().numpy()
        self.calls.append(("mcd", list(nx), list(ny), K))
        for b in range(len(ny)):
            assert not Yh[b, ny[b]:].any()
        return torch.tensor([float(Yh[b].sum()) for b in range(len(ny))], dtype=torch.float64), \
            torch.tensor(np.asarray(ny) + 1, dtype=torch.int32)

    def text2mel_align(self, L, mels, lengths=None):
        return None, None, None, -torch.as_tensor(np.asarray(lengths), dtype=torch.float64)

    def train_capacity(self):
        return self.hp.max_N, 6

    def train_eval(self, L, mels, seed=0, want=("Y",)):
        m = torch.as_tensor(mels)
        self.calls.append(("eval", tuple(np.asarray(L).shape), tuple(m.shape)))
        v = float(m.mean())
        return {"loss": v, "loss_mels": v, "loss_bd1": 0.0, "loss_att": 0.0}, {"Y": m.clone()}


def _corpus(tmp_path, monkeypatch):
    d = tmp_path / "corpus"
    d.mkdir()
    (tmp_path / "mels").mkdir()
    (tmp_path / "mags").mkdir()
    monkeypatch.chdir(tmp_path)
    items = [("a", "abcdef", 4, 1.0), ("b", "ab", 3, 5.0), ("c", "abcdefghijklmn", 6, 1.0), ("d", "abcd", 10, 1.0),
             ("e", "abcdefgh", 2, 1.0), ("f", "abc", 5, 3.0), ("g", "abcde", 6, 2.0)]
    lines = []
    for name, text, frames, level in items:
        lines.append("%s.wav|x|%s|0|1.0" % (name, text))
        np.save(tmp_path / "mels" / (name + ".npy"), np.full((frames, 80), level / 10, np.float32))
        np.save(tmp_path / "mags" / (name + ".npy"), np.zeros((4 * frames, 1025), np.float32))
    (d / "transcript.csv").write_text("\n".join(lines) + "\n")
    return str(d), items


def test_split_heldout_deterministic_disjoint():
    fpaths = ["u%03d.wav" % i for i in range(50)]
    lens = list(range(3, 53))
    texts = [np.arange(n, dtype=np.int32) for n in lens]
    train, held = ho.split_heldout(fpaths, lens, texts, 7, seed=3)
    train2, held2 = ho.split_heldout(list(fpaths), list(lens), list(texts), 7, seed=3)     # another rank, same call
    assert train[0] == train2[0] and held[0] == held2[0]
    assert len(held[0]) == 7 and len(train[0]) == 43
    assert not set(train[0]) & set(held[0]) and set(train[0]) | set(held[0]) == set(fpaths)
    assert held[0] == sorted(held[0]) and train[0] == sorted(train[0])                   # corpus order
    for f, n, t in zip(*held):
        i = fpaths.index(f)
        assert n == lens[i] and t is texts[i]
    assert ho.split_heldout(fpaths, lens, texts, 7, seed=4)[1][0] != held[0]
    for bad in (0, 50, -1):
        with pytest.raises(ValueError):
            ho.split_heldout(fpaths, lens, texts, bad)


@pytest.mark.parametrize("P,n,e,t,want", [
    ([0, 1, 2, 3, 4], 5, 4, 5, dict(eos_reached=True, skipped=0, longest_stall=1, length_ratio=1.0)),
    ([0, 0, 0, 2, 2, 5, -1, -1], 6, 5, 3, dict(eos_reached=True, skipped=3, longest_stall=3, length_ratio=2.0)),
    ([0, 1, 1, 1, 1, 1, 1, 1], 8, 4, 4, dict(eos_reached=False, skipped=2, longest_stall=7, length_ratio=2.0)),
    ([0], 1, 0, 2, dict(eos_reached=True, skipped=0, longest_stall=1, length_ratio=0.5)),
])
def test_window_checks(P, n, e, t, want):
    assert ho.window_checks(np.array(P), n, e, t, 8) == want
    assert ref_mcd.window_checks(np.array(P), n, e, t, 8) == want


def test_heldout_run_rows_skips_and_files(tmp_path, monkeypatch):
    data, items = _corpus(tmp_path, monkeypatch)
    from dc_tts_b200.trainer import load_train_data
    fpaths, lens, texts = load_train_data(data)
    e = _StubEngine()
    h = ho.HeldOut(e, fpaths, lens, texts, prepro=True, B=2)
    rows, s = h.run(e, 1, 3000, train_batch=3)
    by = {r["fname"]: r for r in rows}
    assert [r["fname"] for r in rows] == [n + ".wav" for n, _, _, _ in items]
    assert "max_N" in by["c.wav"]["reason"] and "max_T" in by["d.wav"]["reason"]
    assert "cannot be reached" in by["e.wav"]["reason"]
    assert e.refreshed == 1
    # batches of 2 in text-length order b, f, g, a (d, e set aside)
    assert [c[2] for c in e.calls if c[0] == "mcd"] == [[3, 5], [6, 4]]
    a = by["a.wav"]
    assert a["mcd"] == pytest.approx(4 * 80 * 0.1, rel=1e-6) and a["pairs"] == 5
    assert a["generated"] == 8 and a["eos_reached"] is False and a["skipped"] == 0 and a["longest_stall"] == 2
    assert a["length_ratio"] == 2.0 and a["mean_log_attention"] == -1.0
    assert by["b.wav"]["generated"] == 4 and by["b.wav"]["eos_reached"] is True
    # losses: batches of exactly 3 in text-length order, the last completed from the start: [b f g], [a b f]
    evals = [c for c in e.calls if c[0] == "eval"]
    assert [c[2][:2] for c in evals] == [(3, 6), (3, 5)]
    assert s["loss_batches"] == 2 and s["loss_batches_skipped"] == 0
    assert s["evaluated"] == 4 and s["set_aside"] == 3 and s["utterances"] == 7 and s["global_step"] == 3000
    mcds = [by[n]["mcd"] for n in ("a.wav", "b.wav", "f.wav", "g.wav")]
    assert s["mcd_mean"] == pytest.approx(np.mean(mcds)) and s["mcd_median"] == pytest.approx(np.median(mcds))
    assert s["eos_reached"] == 0.75

    out = str(tmp_path / "out")
    h.write(out, rows, s, 1)
    lines = open(os.path.join(out, "heldout.tsv")).read().splitlines()
    assert lines[0].split("\t") == ho.COLUMNS[1]
    cols = {l.split("\t")[0]: l.split("\t") for l in lines[1:]}
    assert cols["c.wav"][1] == "-" and cols["c.wav"][-1].startswith("skipped: ") and cols["c.wav"][3] == "-"
    assert cols["a.wav"][1:3] == ["4", "7"] and cols["a.wav"][6] == "0" and cols["a.wav"][-1] == ""
    assert json.load(open(os.path.join(out, "summary.json")))["evaluated"] == 4

    log = str(tmp_path / "heldout.tsv")
    ho.append_log(log, 1000, s)
    ho.append_log(log, 2000, s)
    lines = open(log).read().splitlines()
    head = lines[0].split("\t")
    assert head[0] == "global_step" and "mcd_mean" in head and "loss/loss_mels" in head and "num" not in head
    assert [l.split("\t")[0] for l in lines[1:]] == ["1000", "2000"] and len(lines[1].split("\t")) == len(head)


def test_heldout_losses_skip_beyond_capacity(tmp_path, monkeypatch):
    data, _ = _corpus(tmp_path, monkeypatch)
    from dc_tts_b200.trainer import load_train_data
    fpaths, lens, texts = load_train_data(data)
    e = _StubEngine()
    h = ho.HeldOut(e, fpaths, lens, texts, prepro=True, B=4)
    _, s = h.run(e, 1, 0, train_batch=1)        # capacity T = 6: every utterance fits; batches of one
    assert s["loss_batches"] == 4 and s["loss_batches_skipped"] == 0
    e.train_capacity = lambda: (12, 4)
    _, s = h.run(e, 1, 0, train_batch=1)        # f (5 frames) and g (6 frames) go beyond T = 4
    assert s["loss_batches"] == 2 and s["loss_batches_skipped"] == 2


def test_cli_arguments_and_list(tmp_path, monkeypatch):
    a = ho.parser().parse_args(["data", "out"])
    assert (a.list, a.batch, a.wavs, a.resample, a.num) == (None, 32, False, False, 1)
    a = ho.parser().parse_args(["data", "out", "--list", "l.txt", "--batch", "8", "--wavs", "--resample", "--num", "2"])
    assert (a.list, a.batch, a.wavs, a.resample, a.num) == ("l.txt", 8, True, True, 2)
    with pytest.raises(SystemExit):
        ho.parser().parse_args(["data", "out", "--num", "3"])
    lst = tmp_path / "l.txt"
    lst.write_text("b.wav\n\na.wav\n")
    assert ho.read_list(str(lst)) == ["b.wav", "a.wav"]
    f, n, t = ho.select(["x/a.wav", "x/b.wav", "x/c.wav"], [1, 2, 3], ["A", "B", "C"], ho.read_list(str(lst)))
    assert f == ["x/a.wav", "x/b.wav"] and n == [1, 2] and t == ["A", "B"]
    with pytest.raises(ValueError, match="not in the corpus"):
        ho.select(["x/a.wav"], [1], ["A"], ["zz.wav"])
    monkeypatch.setattr(ho.hp, "logdir", str(tmp_path / "nolog"))
    with pytest.raises(FileNotFoundError, match="no Text2Mel checkpoint"):
        ho.main([str(tmp_path), str(tmp_path / "out")])
    with pytest.raises(FileNotFoundError, match="no SSRN checkpoint"):
        ho.main([str(tmp_path), str(tmp_path / "out"), "--num", "2"])
