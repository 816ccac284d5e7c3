"""Time long-form synthesis (dc_tts_b200/longform.py): eight texts of about 1,000 characters each, read by
synthesize_texts, with the time of each stage (split, decode, join, SSRN, vocoder; the device synchronised between
stages), the seconds of audio per second of wall time (runs without the per-stage synchronisation), the join alone, and
the bytes of the full-sequence chains' workspace after the runs, against what SSRN past max_T needs.

SYNTHETIC LENGTHS: no trained model is available and the seeded weights rarely move the attention window to a piece's
EOS, so each piece's stop position is taken from a full run's window history so that its length is the available frame
nearest to (its characters) x max_T / max_N, as tools/bench_until_eos.py does.
   python tools/bench_longform.py [--reps 3] [--momentum 0.99]"""
import argparse
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from dc_tts_b200 import longform as lf  # noqa: E402
from dc_tts_b200.data_load import utterance_lengths  # noqa: E402
from dc_tts_b200.engine import Engine  # noqa: E402
from dc_tts_b200.hyperparams import Hyperparams as hp  # noqa: E402
from dc_tts_b200.params import init_params  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--momentum", type=float, default=0.0)
a = ap.parse_args()
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
except (OSError, IndexError):
    card = "unknown"
print("card:", card, flush=True)

WORDS = ("the birch canoe slid on the smooth planks glue the sheet to the dark blue background it is easy to tell the "
         "depth of a well these days a chicken leg is a rare dish rice is often served in round bowls the juice of "
         "lemons makes fine punch the box was thrown beside the parked truck").split()
rng = np.random.default_rng(0)


def text(n_chars):
    out, sent = [], []
    while sum(len(s) + 1 for s in out) < n_chars:
        sent.append(WORDS[rng.integers(len(WORDS))])
        if len(sent) > 6 and rng.random() < 0.12:
            out.append(" ".join(sent).capitalize() + rng.choice([".", ".", "?", "!"]))
            sent = []
        elif len(sent) > 4 and rng.random() < 0.08:
            sent[-1] += ","
    return " ".join(out)


texts = [text(1000) for _ in range(8)]
e = Engine(0)
e.load_params(init_params(0, "perturbed"))
pieces, owner, _ = lf.plan(texts)
L = lf.encode_pieces(pieces)
_, Pf, _, _ = e.text2mel_generate(L)
m = Pf.cpu().numpy()[:, 1:]
target = np.maximum(np.round((L > 0).sum(1) * hp.max_T / hp.max_N), 2)
sp = np.zeros(len(L), np.int64)
for b in range(len(L)):
    first = [0] + [j for j in range(1, m.shape[1]) if m[b, j] > m[b, j - 1]]
    j = min(first, key=lambda f: abs(f + 1 - target[b]))
    sp[b] = 0 if j == 0 else int(m[b, j])
n = utterance_lengths(m, sp, 0, steps=hp.max_T)
print("%d texts of %s characters, %d pieces (%d..%d characters), piece frames min %d median %d max %d" % (
    len(texts), "/".join(str(len(t)) for t in texts), len(pieces), min(len(p) for p, _ in pieces),
    max(len(p) for p, _ in pieces), n.min(), int(np.median(n)), n.max()), flush=True)

lf.synthesize_texts(e, texts, stop_pos=sp, momentum=a.momentum)            # warm-up: every shape and buffer
torch.cuda.synchronize()
stages = {}
walls = []
for _ in range(a.reps):
    t = {}
    lf.synthesize_texts(e, texts, stop_pos=sp, momentum=a.momentum, timings=t)
    for k, v in t.items():
        stages.setdefault(k, []).append(v)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    wavs, report = lf.synthesize_texts(e, texts, stop_pos=sp, momentum=a.momentum)
    torch.cuda.synchronize()
    walls.append(time.perf_counter() - t0)
frames = [r["frames"] for r in report]
audio = sum(len(w) for w in wavs) / hp.sr
for k, v in stages.items():
    print("%-8s %s ms (median %.2f)" % (k, " ".join("%.2f" % (1e3 * x) for x in v), 1e3 * float(np.median(v))), flush=True)
wall = float(np.median(walls))
print("joined frames per text: %s (max_T = %d)" % (frames, hp.max_T))
print("end to end, no stage syncs: %s s (median %.3f); %.1f s of trimmed audio -> %.1f s of audio per second" % (
    " ".join("%.3f" % w for w in walls), wall, audio, audio / wall))
# the join alone: Engine.join_rows (host checks, one pinned upload, one launch) in a loop, CUDA events, no sync inside
Y, _, n_dev = e.text2mel_generate_until(L, stop_pos=sp)
pauses = lf.pause_rows([k for _, k in pieces])
e.join_rows(Y, n_dev, owner, pauses, len(texts))
ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
ev[0].record()
for _ in range(100):
    e.join_rows(Y, n_dev, owner, pauses, len(texts))
ev[1].record()
torch.cuda.synchronize()
print("join_rows alone (%d pieces -> %d texts): %.1f us per call" % (len(pieces), len(texts),
                                                                   10 * ev[0].elapsed_time(ev[1])))
need = 98688 * len(texts) * max(frames)
print("chain workspace after the run: %d bytes; SSRN at B = %d, T = %d needs 98688 bytes per frame x %d frames = %d "
      "(a workspace that already holds that, e.g. one sized for the decode batch at max_T, does not grow)" % (
          e.reserve_frames(1, 1), len(texts), max(frames), len(texts) * max(frames), need))
f = Engine(0)
f.load_params(init_params(0, "perturbed"))
print("a fresh engine after reserve_frames(%d, %d): %d bytes" % (len(texts), max(frames),
                                                               f.reserve_frames(len(texts), max(frames))))
