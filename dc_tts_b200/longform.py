"""Long-form synthesis: texts of any length, read as one waveform each.

The model was trained on clips of at most max_T reduced frames (about 10.5 s) and max_N characters, so a long text is
split into pieces, the pieces of every text are decoded as one batch (Engine.text2mel_generate_until), and each text's
pieces are joined on the device into one mel sequence (Engine.join_rows, csrc/kernels_longform.cu) with rows of silence
between them.  SSRN then runs once over the joined sequences (past max_T: the synthesis workspace grows to the call's
length) and Griffin-Lim once per text over its whole magnitude sequence, so the phase is continuous across the joins.

The splitting rule (split_text) works on the raw text, before text_normalize turns ", ; : !" into spaces:
  1. split after every sentence end: ".", "?" or "!" followed by whitespace or the end of the text;
  2. a piece whose normalised text is longer than max_chars is split after the last clause mark ("," ";" ":" an em
     dash, or a "-" between spaces) that keeps the first part within max_chars;
  3. without such a mark, at the last whitespace that keeps the first part within max_chars;
  4. without one either, by a hard cut at the longest prefix within max_chars;
  and rules 2-4 repeat on the rest.  Each piece is then normalised as data_load.load_data does and "E" appended; pieces
  that normalise to nothing are dropped.  A piece's pause kind is "sentence" after a sentence end, "clause" after any
  other split and "none" for the last piece of a text.  The rule knows no abbreviations: "Mr. Smith" splits after "Mr.".

The pauses (8 reduced frames, 0.4 s, after a sentence; 4, 0.2 s, after a clause) and the silence level (1e-8, the
normalised level of digital silence as get_spectrograms clips it) are not tuned: whether they sound natural with a
trained model has not been listened to.

CLI: python -m dc_tts_b200.longform IN.txt OUT_DIR [--momentum M]: one text per non-empty line of IN.txt, one wav per
line (1.wav, 2.wav, ... by line among the non-empty ones) and report.json in OUT_DIR.
"""
import argparse
import json
import os
import re

import numpy as np

from .data_load import load_vocab, text_normalize
from .hyperparams import Hyperparams as hp

PAUSE_KINDS = ("sentence", "clause", "none")
_SENTENCE_END = re.compile(r"[.?!](?=\s|$)")
_CLAUSE_MARK = re.compile(r"[,;:—]|(?<=\s)-(?=\s)")


def _norm(raw):
    return text_normalize(raw).strip()


def _longest_prefix(raw, max_chars, cuts):
    """The largest cut in `cuts` (ascending raw offsets) whose prefix normalises to 1 .. max_chars characters, or None.
    A prefix's normalised length never falls as the prefix grows, so the cut is found by bisection."""
    lo, hi = 0, len(cuts)                   # cuts[:lo] fit within max_chars, cuts[hi:] do not
    while lo < hi:
        mid = (lo + hi) // 2
        if len(_norm(raw[:cuts[mid]])) <= max_chars:
            lo = mid + 1
        else:
            hi = mid
    return cuts[lo - 1] if lo and _norm(raw[:cuts[lo - 1]]) else None


def _split_long(raw, max_chars):
    """Rules 2-4 on one sentence: [(raw part, split kind)], the last part's kind being None."""
    out = []
    while len(_norm(raw)) > max_chars:
        i = _longest_prefix(raw, max_chars, [m.end() for m in _CLAUSE_MARK.finditer(raw)])
        if i is None:
            i = _longest_prefix(raw, max_chars, [m.start() for m in re.finditer(r"\s", raw)])
        if i is None:
            i = _longest_prefix(raw, max_chars, list(range(1, len(raw))))
        out.append((raw[:i], "clause"))
        raw = raw[i:]
    out.append((raw, None))
    return out


def split_text(text, max_chars=hp.max_N - 1):
    """The pieces of one raw text by the module's splitting rule: [(normalised piece + "E", pause kind)], pause kind in
    PAUSE_KINDS.  Every piece has 1 .. max_chars characters before its "E"; a text that normalises to nothing has none."""
    if max_chars < 1:
        raise ValueError("split_text: max_chars must be >= 1, got %r" % max_chars)
    parts, start = [], 0
    for m in _SENTENCE_END.finditer(text):
        parts.append((text[start:m.end()], "sentence"))
        start = m.end()
    parts.append((text[start:], "sentence"))
    pieces = []
    for raw, kind in parts:
        for sub, k in _split_long(raw, max_chars):
            s = _norm(sub)
            if s:
                pieces.append([s + "E", k or kind])
    if pieces:
        pieces[-1][1] = "none"
    return [tuple(p) for p in pieces]


def encode_pieces(pieces, max_N=hp.max_N):
    """(P, max_N) int32 ids of split_text's pieces, zero padded, as load_data writes them."""
    char2idx, _ = load_vocab()
    L = np.zeros((len(pieces), max_N), np.int32)
    for i, (s, _) in enumerate(pieces):
        L[i, :len(s)] = [char2idx[ch] for ch in s]
    return L


def pause_rows(kinds, pause=(8, 4)):
    """Rows of silence after each piece: pause[0] after a sentence, pause[1] after a clause, 0 after a text's last."""
    sent, clause = _check_pause(pause)
    return np.array([{"sentence": sent, "clause": clause, "none": 0}[k] for k in kinds], np.int32)


def _check_pause(pause):
    try:
        sent, clause = (int(p) for p in pause)
    except (TypeError, ValueError):
        raise ValueError("pause must be two integers (after a sentence, after a clause), got %r" % (pause,)) from None
    if sent < 0 or clause < 0:
        raise ValueError("pause must be >= 0 rows, got %r" % (pause,))
    return sent, clause


def plan(texts, pause=(8, 4), max_chars=hp.max_N - 1):
    """Split every text: (pieces [(piece, kind)], piece_text (P,) int32, piece_pause (P,) int32).  A text with no piece is
    refused."""
    pieces, owner = [], []
    for k, t in enumerate(texts):
        ps = split_text(t, max_chars)
        if not ps:
            raise ValueError("text %d has nothing to read after normalisation: %r" % (k, t[:80]))
        pieces += ps
        owner += [k] * len(ps)
    return pieces, np.array(owner, np.int32), pause_rows([k for _, k in pieces], pause)


def synthesize_texts(engine, texts, pause=(8, 4), silence=1e-8, tail=0, momentum=0.0, stop_pos=None, timings=None):
    """One waveform per text of any length.  Returns (wavs, report): wavs a list of trimmed float32 numpy waveforms at
    hp.sr; report one dict per text with its pieces (text, pause kind, frames, whether the attention reached the EOS) and
    its joined frames.  `pause`: rows of silence (after a sentence, after a clause), `silence` their value; `tail` and
    `stop_pos` (one per piece in report order; default each piece's EOS) go to text2mel_generate_until; `momentum` to the
    vocoder.  `timings`: an optional dict that receives the seconds of each stage (the device is synchronised between
    them when it is given)."""
    import time

    import torch

    from .utils import spectrograms2wavs
    texts = list(texts)
    if not texts:
        raise ValueError("synthesize_texts: no texts")
    _check_pause(pause)

    def lap(name, t0):
        if timings is None:
            return t0
        torch.cuda.synchronize(engine.device)
        t = time.perf_counter()
        timings[name] = timings.get(name, 0.0) + t - t0
        return t

    if timings is not None:
        torch.cuda.synchronize(engine.device)
    t0 = time.perf_counter()
    pieces, owner, pauses = plan(texts, pause)
    L = encode_pieces(pieces, engine.hp.max_N)
    t0 = lap("split", t0)
    from .data_load import eos_positions
    sp = eos_positions(L) if stop_pos is None else np.asarray(stop_pos, np.int64).reshape(-1)
    if sp.shape[0] != len(pieces):
        raise ValueError("synthesize_texts: %d stop positions for %d pieces" % (sp.shape[0], len(pieces)))
    Y, P, n = engine.text2mel_generate_until(L, stop_pos=sp, tail=tail)
    t0 = lap("decode", t0)
    M, m = engine.join_rows(Y, n, owner, pauses, len(texts), silence)
    m_host = m.cpu().numpy()
    t0 = lap("join", t0)
    Tmax = int(m_host.max())
    _, Z = engine.ssrn(M[:, :Tmax], want_logits=False, lengths=m)
    t0 = lap("ssrn", t0)
    wavs = spectrograms2wavs(Z, lengths=engine.hp.r * m_host, momentum=momentum, engine=engine)
    lap("vocoder", t0)
    n_host, P_host = n.cpu().numpy(), P.cpu().numpy()
    T = Y.shape[1]
    report = [{"pieces": [], "frames": int(m_host[k])} for k in range(len(texts))]
    for p, (s, kind) in enumerate(pieces):
        k = int(n_host[p])
        eos = bool(k < T or (sp[p] >= 0 and (P_host[p, 1:k] >= sp[p]).any()))
        report[owner[p]]["pieces"].append({"text": s, "pause": kind, "frames": k, "eos": eos})
    return wavs, report


def read_texts(path, header=False):
    """One text per non-empty line of a UTF-8 file.  header=True: the sentences-file convention of load_data (the first
    line is a header and is dropped, and a leading "N. " is removed from each line)."""
    with open(path, encoding="utf-8") as f:
        lines = f.read().splitlines()
    if header:
        lines = [ln.split(" ", 1)[-1] for ln in lines[1:]]
    return [ln for ln in lines if ln.strip()]


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m dc_tts_b200.longform", description="Read texts of any length, one per line.")
    ap.add_argument("infile")
    ap.add_argument("outdir")
    ap.add_argument("--momentum", type=float, default=0.0, help="fast Griffin-Lim momentum (0: the reference's update)")
    a = ap.parse_args(argv)
    from scipy.io.wavfile import write as write_wav

    from .engine import get_engine
    from .synthesize import _restore
    texts = read_texts(a.infile)
    if not texts:
        raise SystemExit("%s holds no text" % a.infile)
    e = get_engine()
    _restore(e, None, 0, False)                  # the latest checkpoints of hp.logdir-1 and hp.logdir-2
    wavs, report = synthesize_texts(e, texts, momentum=a.momentum)
    os.makedirs(a.outdir, exist_ok=True)
    for i, w in enumerate(wavs):
        write_wav(os.path.join(a.outdir, "%d.wav" % (i + 1)), hp.sr, w)
    with open(os.path.join(a.outdir, "report.json"), "w") as f:
        json.dump(report, f, indent=1)
    missed = sum(not p["eos"] for r in report for p in r["pieces"])
    print("%d texts, %d pieces, %d without their EOS in %d frames -> %s" % (
        len(texts), sum(len(r["pieces"]) for r in report), missed, hp.max_T, a.outdir))


if __name__ == "__main__":
    main()
