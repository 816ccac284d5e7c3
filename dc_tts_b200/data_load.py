"""Text -> id adaptor of the synthesis path (reference data_load.py:19-31, :79-86).

Only the pure-Python pieces `synthesize.py` needs are provided; the TF queue-runner
training pipeline (`get_batch`, data_load.py:88-131) is out of scope (SURVEY.md 2.1).
"""
import codecs
import re
import unicodedata

import numpy as np

from .hyperparams import Hyperparams as hp


def load_vocab():
    """data_load.py:19-22."""
    char2idx = {ch: i for i, ch in enumerate(hp.vocab)}
    idx2char = dict(enumerate(hp.vocab))
    return char2idx, idx2char


def text_normalize(text):
    """data_load.py:24-31: strip accents, lower-case, out-of-vocab -> space, squeeze spaces."""
    text = "".join(ch for ch in unicodedata.normalize("NFD", text) if unicodedata.category(ch) != "Mn")
    text = re.sub("[^{}]".format(hp.vocab), " ", text.lower())
    return re.sub("[ ]+", " ", text)


def eos_positions(texts):
    """(B, N) ids -> (B,) int32: the index of the first EOS id ("E", which load_data appends to every text), -1 for a row
    without one.  The default stop position of Engine.text2mel_generate_until."""
    t = np.asarray(texts)
    hit = t == hp.vocab.index("E")
    return np.where(hit.any(axis=1), hit.argmax(axis=1), -1).astype(np.int32)


def utterance_lengths(max_attentions, stop_pos, tail=0, steps=None):
    """The end-of-utterance rule on a window history.  max_attentions (B, >= steps): the attention argmax of every frame
    (row j is the window of frame j + 1).  Utterance b ends at min(steps, j* + 1 + tail), j* being the first frame
    j < steps whose argmax is >= stop_pos[b], or at `steps` when there is none or stop_pos[b] < 0."""
    m = np.asarray(max_attentions)
    steps = m.shape[1] if steps is None else int(steps)
    if tail < 0:
        raise ValueError("tail must be >= 0")
    out = np.full(m.shape[0], steps, np.int32)
    for b, sp in enumerate(np.asarray(stop_pos).reshape(-1)):
        if sp < 0:
            continue
        hit = np.nonzero(m[b, :steps] >= sp)[0]
        if hit.size:
            out[b] = min(steps, int(hit[0]) + 1 + int(tail))
    return out


def load_data(mode="synthesize", path=None):
    """data_load.py:79-86: sentences file (first line is a header and is dropped, the
    leading "N. " of each line is removed) -> int32 ids (num_sentences, max_N), each
    sentence terminated by E and zero padded."""
    if mode != "synthesize":
        raise NotImplementedError("only the synthesize branch is on the hot path (SURVEY.md 2.1)")
    char2idx, _ = load_vocab()
    lines = codecs.open(path or hp.test_data, "r", "utf-8").readlines()[1:]
    sents = [text_normalize(line.split(" ", 1)[-1]).strip() + "E" for line in lines]
    texts = np.zeros((len(sents), hp.max_N), np.int32)
    for i, sent in enumerate(sents):
        texts[i, :len(sent)] = [char2idx[ch] for ch in sent]
    return texts
