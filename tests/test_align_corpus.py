"""The corpus aligner's host logic (dc_tts_b200/align.py) with a stub engine: skip rules, batching in text-length order,
the file formats and the ranking."""
import os

import numpy as np
import torch

from dc_tts_b200.align import align_corpus
from dc_tts_b200.hyperparams import Hyperparams


class _StubEngine:
    """text2mel_align's interface: the score of each utterance is minus its mels' sum, every frame on its EOS."""

    class hp(Hyperparams):
        max_N, max_T, attention_win_size = 12, 8, 3

    def __init__(self):
        self.calls = []

    def text2mel_align(self, L, mels, lengths=None):
        m = np.asarray(mels)
        self.calls.append((np.asarray(L).copy(), m.shape, np.asarray(lengths).copy()))
        B = len(L)
        ends = (np.asarray(L) == Hyperparams.vocab.index("E")).argmax(1)
        dur = torch.zeros(B, self.hp.max_N, dtype=torch.int32)
        for b in range(B):
            assert not m[b, lengths[b]:].any()              # zero padding past each recording
            dur[b, ends[b]] = int(lengths[b])
        score = torch.tensor([-float(m[b].sum()) for b in range(B)], dtype=torch.float64)
        return None, None, dur, score


def _corpus(tmp_path, monkeypatch):
    """Texts of 3..14 characters (plus EOS) and recordings of 1..10 frames; mels/*.npy in the working directory."""
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
        np.save(tmp_path / "mels" / (name + ".npy"), np.full((frames, 80), level, np.float32))
        np.save(tmp_path / "mags" / (name + ".npy"), np.zeros((4 * frames, 1025), np.float32))
    (d / "transcript.csv").write_text("\n".join(lines) + "\n")
    return str(d), items


def test_align_corpus_files_and_skips(tmp_path, monkeypatch):
    data, items = _corpus(tmp_path, monkeypatch)
    e = _StubEngine()
    out = str(tmp_path / "out")
    rows = align_corpus(data, e, out, B=2, prepro=True)
    by = {r["fname"]: r for r in rows}
    assert [r["fname"] for r in rows] == [n + ".wav" for n, _, _, _ in items]           # transcript order
    assert "max_N" in by["c.wav"]["reason"] and by["c.wav"]["frames"] is None             # 15 characters > 12
    assert "max_T" in by["d.wav"]["reason"]                                                # 10 frames > 8
    assert "cannot be reached" in by["e.wav"]["reason"]                                    # EOS 8 > 2 * 2 frames
    aligned = [n + ".wav" for n in "abfg"]
    for n in aligned:
        r = by[n]
        assert r.get("reason") is None and sum(r["durations"]) == r["frames"]
        assert len(r["durations"]) == r["text_length"]
    # batches of 2 in stable text-length order (b 3, f 4, d 5, g 6, a 7, e 9), each padded to its longest kept recording
    # -> [b, f], [d, g] without d, [a, e] without e
    assert [c[2].tolist() for c in e.calls] == [[3, 5], [6], [4]]
    assert [(c[0] != 0).sum(1).tolist() for c in e.calls] == [[3, 4], [6], [7]]
    assert all(shape[1] == int(n.max()) for _, shape, n in e.calls)

    lines = open(os.path.join(out, "alignments.tsv")).read().splitlines()
    assert lines[0].split("\t") == ["fname", "frames", "text_length", "mean_log_attention", "durations"]
    cols = {l.split("\t")[0]: l.split("\t") for l in lines[1:]}
    assert len(cols) == len(items)
    assert cols["c.wav"][1] == "-" and cols["c.wav"][4].startswith("skipped: ")
    assert cols["d.wav"][1] == "10" and cols["d.wav"][3] == "-"
    a = cols["a.wav"]
    assert a[1:3] == ["4", "7"] and float(a[3]) == -1.0 * 80
    assert [int(x) for x in a[4].split()] == [0] * 6 + [4]
    ranking = open(os.path.join(out, "ranking.txt")).read().split()
    assert ranking == ["b.wav", "f.wav", "g.wav", "a.wav"]                              # mean: -400, -240, -160, -80
