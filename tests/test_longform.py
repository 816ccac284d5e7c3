"""Long-form synthesis on the host (dc_tts_b200/longform.py): the splitting rule on a table of cases, the invariants of its
pieces on longer texts, and the numpy restatement of the device join that the GPU tests hold the kernel to."""
import re

import numpy as np
import pytest

from ref_longform import join_rows_reference
from dc_tts_b200 import longform as lf
from dc_tts_b200.data_load import text_normalize
from dc_tts_b200.hyperparams import Hyperparams as hp

MAX = hp.max_N - 1


def _pieces(text, max_chars=MAX):
    return [(p[:-1], k) for p, k in lf.split_text(text, max_chars)]


@pytest.mark.parametrize("text,max_chars,want", [
    ("The birch canoe slid. Glue the sheet! Is it easy? Yes",
     MAX, [("the birch canoe slid.", "sentence"), ("glue the sheet", "sentence"), ("is it easy?", "sentence"),
           ("yes", "none")]),
    ("Hello.", MAX, [("hello.", "none")]),
    ("Hello!!  World?", MAX, [("hello", "sentence"), ("world?", "none")]),
    ("Wait... what?", MAX, [("wait...", "sentence"), ("what?", "none")]),
    ("Version 2.5 is out", MAX, [("version . is out", "none")]),              # "." before a digit is no sentence end
    ("Mr. Smith went home.", MAX, [("mr.", "sentence"), ("smith went home.", "none")]),   # no abbreviations
    ('"Stop!" he said. Then  he   left.', MAX, [("stop he said.", "sentence"), ("then he left.", "none")]),
    ("Tab\tends here.\nNext line", MAX, [("tab ends here.", "sentence"), ("next line", "none")]),
    ("!!! ... Go.", MAX, [("...", "sentence"), ("go.", "none")]),              # "!!!" normalises to nothing
    ("!!! ; --", MAX, []),
    ("!!! ?", MAX, [("?", "none")]),                                          # "?" is in the vocabulary
    ("", MAX, []),
    ("one two, three four, five six", 12, [("one two", "clause"), ("three four", "clause"), ("five six", "none")]),
    ("alpha beta; gamma: delta", 12, [("alpha beta", "clause"), ("gamma delta", "none")]),
    ("alpha beta; gamma: delta", 8, [("alpha", "clause"), ("beta", "clause"), ("gamma", "clause"), ("delta", "none")]),
    ("alpha — beta - gamma-delta", 12, [("alpha beta", "clause"), ("gamma delta", "none")]),
    ("alpha — beta - gamma-delta", 6, [("alpha", "clause"), ("beta", "clause"), ("gamma", "clause"), ("delta", "none")]),
    ("aaa bbb ccc ddd eee", 8, [("aaa bbb", "clause"), ("ccc ddd", "clause"), ("eee", "none")]),
    ("abcdefghijkl", 5, [("abcde", "clause"), ("fghij", "clause"), ("kl", "none")]),
    ("a, bcdefghijkl", 5, [("a", "clause"), ("bcdef", "clause"), ("ghijk", "clause"), ("l", "none")]),
    ("Café naïve.", MAX, [("cafe naive.", "none")]),
])
def test_split_text_cases(text, max_chars, want):
    assert _pieces(text, max_chars) == want


def test_split_prefers_the_last_clause_mark_within_the_limit():
    text = "one, two, three, four five six seven"
    assert _pieces(text, 20) == [("one two three", "clause"), ("four five six seven", "none")]


def test_split_uses_the_last_space_when_no_mark_fits():
    # the only comma leaves a first part of 25 characters: too long for 20, so the split is at a space
    text = "aaaa bbbb cccc dddd eeee, ffff"
    assert _pieces(text, 20) == [("aaaa bbbb cccc dddd", "clause"), ("eeee ffff", "none")]


def test_limit_edges():
    exact = "a" * MAX
    assert lf.split_text(exact) == [(exact + "E", "none")]
    over = "a" * (MAX + 1)
    assert lf.split_text(over) == [("a" * MAX + "E", "clause"), ("aE", "none")]
    words = " ".join(["abcd"] * 60)                       # 299 characters
    ps = lf.split_text(words)
    assert [len(p) for p, _ in ps] == [180, 120]          # 36 words + "E", the other 24
    assert lf.split_text("x" * (hp.max_N - 2) + ".") == [("x" * (hp.max_N - 2) + ".E", "none")]


def test_split_refuses_a_zero_limit():
    with pytest.raises(ValueError, match="max_chars"):
        lf.split_text("abc", 0)


PARAGRAPH = ("It was the best of times, it was the worst of times, it was the age of wisdom, it was the age of foolishness, "
             "it was the epoch of belief, it was the epoch of incredulity, it was the season of Light, it was the season "
             "of Darkness, it was the spring of hope, it was the winter of despair; we had everything before us, we had "
             "nothing before us!  We were all going direct to Heaven -- we were all going direct the other way. "
             "In short, the period was so far like the present period, that some of its noisiest authorities insisted "
             "on its being received, for good or for evil, in the superlative degree of comparison only. ")


@pytest.mark.parametrize("text", [
    PARAGRAPH,
    PARAGRAPH * 3,
    "word " * 400,
    "x" * 1000,
    "Short. " * 50,
    "".join(chr(0x61 + (i * 7) % 26) + (" " if i % 11 == 0 else "") + ("," if i % 97 == 0 else "") for i in range(2000)),
])
@pytest.mark.parametrize("max_chars", [MAX, 40, 7])
def test_pieces_fit_and_concatenate_to_the_text(text, max_chars):
    ps = lf.split_text(text, max_chars)
    assert ps and ps[-1][1] == "none" and all(k in ("sentence", "clause") for _, k in ps[:-1])
    for p, _ in ps:
        assert p.endswith("E") and 2 <= len(p) <= max_chars + 1 and p == p.strip()
        assert re.fullmatch("[{}]+".format(re.escape(hp.vocab[2:])), p[:-1]), p
    whole = text_normalize(text).strip()
    got = [p[:-1] for p, _ in ps]
    assert "".join(got).replace(" ", "") == whole.replace(" ", "")
    # apart from the hard cuts, the pieces joined with a space are the normalised text
    if max_chars >= 40 and "x" * 50 not in text:
        assert " ".join(got) == whole
    L = lf.encode_pieces(ps)
    assert L.shape == (len(ps), hp.max_N) and (L == 1).sum(1).tolist() == [1] * len(ps)


def test_plan_and_pause_rows():
    pieces, owner, pause = lf.plan(["One. Two, three", "Four"], pause=(8, 4), max_chars=MAX)
    assert [k for _, k in pieces] == ["sentence", "none", "none"]
    assert owner.tolist() == [0, 0, 1] and pause.tolist() == [8, 0, 0]
    _, _, pause = lf.plan(["a, b, c. d"], pause=(5, 3), max_chars=2)
    assert pause.tolist() == [3, 3, 5, 0]
    with pytest.raises(ValueError, match="text 1 has nothing to read"):
        lf.plan(["ok", "!!!"])
    for bad in [(-1, 4), (8,), "ab", None]:
        with pytest.raises(ValueError, match="pause"):
            lf.pause_rows(["none"], bad)


def _join_loops(Y, n, text, pause, K, silence, T_out):
    """The join written row by row, to check the restatement against."""
    P, T, C = Y.shape
    out = np.zeros((K, T_out, C), np.float32)
    pos = [0] * K
    for p in range(P):
        k = text[p]
        for t in range(min(max(n[p], 0), T)):
            out[k, pos[k]] = Y[p, t]
            pos[k] += 1
        for _ in range(pause[p]):
            out[k, pos[k]] = silence
            pos[k] += 1
    return out, np.array(pos, np.int32)


@pytest.mark.parametrize("case", ["ragged", "zero pause", "one piece", "K=1", "long"])
def test_join_reference(case):
    rng = np.random.default_rng(len(case))
    T, C = 30, 5
    if case == "one piece":
        text, pause = [0], [0]
    elif case == "K=1":
        text, pause = [0, 0, 0, 0], [3, 0, 2, 0]
    elif case == "long":
        text = [0] * 40 + [1] * 3
        pause = [8 if i % 3 else 4 for i in range(39)] + [0, 8, 4, 0]
    else:
        text, pause = [0, 0, 1, 2, 2, 2], [8, 0, 0, 4, 8, 0]
        if case == "zero pause":
            pause = [0] * 6
    P, K = len(text), max(text) + 1
    Y = rng.uniform(0, 1, (P, T, C)).astype(np.float32)
    n = rng.integers(1, T + 1, P)
    n[0] = T
    if P > 1:
        n[-1] = 1
    T_out = int(max(np.bincount(text, weights=T + np.array(pause), minlength=K)))
    out, m = join_rows_reference(Y, n, text, pause, K, 1e-8, T_out)
    ref, mr = _join_loops(Y, n, text, pause, K, np.float32(1e-8), T_out)
    assert np.array_equal(out, ref) and np.array_equal(m, mr)
    assert out.shape == (K, T_out, C)
    for k in range(K):
        assert not out[k, m[k]:].any()
        assert m[k] == sum(n[p] + pause[p] for p in range(P) if text[p] == k)
    if case == "zero pause":
        assert not (out == np.float32(1e-8)).any()
