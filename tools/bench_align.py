"""Time the aligner with CUDA events, the variants alternated in one run:
  align B          Engine.text2mel_align: the teacher-forced front and the search, T = 210 frames
  search B         Engine.align_search alone on the alignments that call returned
  forward B        align B minus search B
at B = 1 and 32 (texts of 150 characters, U(0, 1) mels), with utterances per second and seconds of audio aligned per
second (one frame is r hop / sr seconds); then align_corpus on a synthetic corpus of noise-burst wavs written to a
temporary directory, features from the wavs (prepro=False), end to end on the wall clock.
   python tools/bench_align.py [--reps 3] [--iters 10] [--corpus 256]"""
import argparse
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from dc_tts_b200.align import align_corpus  # noqa: E402
from dc_tts_b200.engine import Engine  # noqa: E402
from dc_tts_b200.hyperparams import Hyperparams as hp  # noqa: E402
from dc_tts_b200.params import init_params, synthetic_text  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--iters", type=int, default=10)
ap.add_argument("--corpus", type=int, default=256)
a = ap.parse_args()
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
except (OSError, IndexError):
    card = "unknown"
print("card:", card, flush=True)

e = Engine(0)
e.load_params(init_params(0, "perturbed"))
T = hp.max_T
frame_s = hp.r * hp.hop_length / hp.sr


def timed(fn):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(a.iters):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / a.iters


runs = {}
for B in (1, 32):
    L = np.concatenate([synthetic_text(1, 150, seed=900 + b) for b in range(B)])
    mels = torch.rand(B, T, hp.n_mels, device="cuda")
    A = e.text2mel_align(L, mels, want_alignments=True)[4]
    ends = (L == hp.vocab.index("E")).argmax(1)
    n = np.full(B, T)
    runs["align %d" % B] = (lambda L=L, mels=mels: e.text2mel_align(L, mels))
    runs["search %d" % B] = (lambda A=A, n=n, ends=ends: e.align_search(A, n, ends))
for fn in runs.values():
    fn()
torch.cuda.synchronize()
res = {k: [] for k in runs}
for rep in range(a.reps):
    for k, fn in runs.items():
        res[k].append(timed(fn))
for B in (1, 32):
    al, se = float(np.median(res["align %d" % B])), float(np.median(res["search %d" % B]))
    print("B = %2d: align %.3f ms (%s), search %.3f ms (%s), forward %.3f ms; %.0f utterances/s, %.0f s of audio/s"
          % (B, al, " ".join("%.3f" % x for x in res["align %d" % B]), se, " ".join("%.3f" % x for x in res["search %d" % B]),
             al - se, B / al * 1e3, B * T * frame_s / al * 1e3), flush=True)

# align_corpus on noise-burst wavs (1.5 - 9 s), five-field transcript (not "LJ" in the path)
with tempfile.TemporaryDirectory() as d:
    from scipy.io import wavfile
    rng = np.random.default_rng(0)
    lines, secs = [], 0.0
    for i in range(a.corpus):
        s = float(rng.uniform(1.5, 9.0))
        n_s = int(s * hp.sr)
        env = np.repeat(rng.random(n_s // 2205 + 1) < 0.7, 2205)[:n_s] * rng.uniform(0.05, 0.5)
        wav = np.clip(rng.standard_normal(n_s) * env * 32767 * 0.3, -32768, 32767).astype(np.int16)
        wavfile.write(os.path.join(d, "u%04d.wav" % i), hp.sr, wav)
        text = "".join(rng.choice(list("abcdefghijklmnopqrstuvwxyz "), int(s * 12)))
        lines.append("u%04d.wav|x|%s|0|%.2f" % (i, text, s))
        secs += s
    with open(os.path.join(d, "transcript.csv"), "w") as f:
        f.write("\n".join(lines) + "\n")
    out = os.path.join(d, "out")
    align_corpus(d, e, out, B=32, prepro=False)          # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    rows = align_corpus(d, e, out, B=32, prepro=False)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    done = sum(1 for r in rows if not r.get("reason"))
    print("align_corpus: %d utterances (%d aligned, %.0f s of audio) in %.2f s: %.1f utterances/s, %.0f s of audio/s"
          % (len(rows), done, secs, dt, len(rows) / dt, secs / dt), flush=True)
