"""Time the held-out evaluation:
  mcd_dtw B x T    Engine.mcd_dtw with CUDA events (median of --reps windows of --iters calls), at B = 64, T = 210 (the
                   typical held-out shape; the cepstra in shared memory) and B = 8, T = 2000 / 1900 (the global-memory
                   route), next to the float64 numpy reference (tests/ref_mcd.py) on the CPU for the same pairs;
  HeldOut.run      a full evaluation of --corpus synthetic utterances (U(0, 1) mels, 100-210 frames, texts of 40-150
                   characters, mels/ and mags/ in a temporary directory) at random weights, num = 1 and num = 2, on the
                   wall clock after a warm-up run.
   python tools/bench_heldout.py [--reps 5] [--iters 20] [--corpus 64] [--ref-pairs 4]"""
import argparse
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import ref_mcd  # noqa: E402
from dc_tts_b200 import heldout as ho  # noqa: E402
from dc_tts_b200.engine import Engine  # noqa: E402
from dc_tts_b200.hyperparams import Hyperparams as hp  # noqa: E402
from dc_tts_b200.params import init_params  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--iters", type=int, default=20)
ap.add_argument("--corpus", type=int, default=64)
ap.add_argument("--ref-pairs", type=int, default=4, help="pairs of each shape the CPU reference is timed on")
a = ap.parse_args()
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
except (OSError, IndexError):
    card = "unknown"
print("card:", card, flush=True)

e = Engine(0)
e.load_params(init_params(0, "perturbed"))
rng = np.random.default_rng(0)
for B, Tx, Ty in ((64, 210, 210), (8, 2000, 1900)):
    X = rng.uniform(0, 1, (B, Tx, hp.n_mels)).astype(np.float32)
    Y = rng.uniform(0, 1, (B, Ty, hp.n_mels)).astype(np.float32)
    nx, ny = np.full(B, Tx), np.full(B, Ty)
    Xd, Yd = torch.from_numpy(X).cuda(), torch.from_numpy(Y).cuda()
    e.mcd_dtw(Xd, nx, Yd, ny)
    torch.cuda.synchronize()
    times = []
    for _ in range(a.reps):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for _ in range(a.iters):
            e.mcd_dtw(Xd, nx, Yd, ny)
        ev[1].record()
        torch.cuda.synchronize()
        times.append(ev[0].elapsed_time(ev[1]) / a.iters)
    k = min(B, a.ref_pairs)
    t0 = time.perf_counter()
    ref = ref_mcd.mcd_batch(X[:k], nx[:k], Y[:k], ny[:k])
    cpu = (time.perf_counter() - t0) / k
    got = e.mcd_dtw(Xd[:k], nx[:k], Yd[:k], ny[:k])[0].cpu().numpy()
    print("mcd_dtw B = %d, %d x %d: %.3f ms median (%s); %.1f us per pair, %.2f ns per cell; float64 numpy reference "
          "%.3f s per pair (%d pairs), worst relative difference %.1e"
          % (B, Tx, Ty, float(np.median(times)), " ".join("%.3f" % x for x in times), float(np.median(times)) * 1e3 / B,
             float(np.median(times)) * 1e6 / (B * Tx * Ty), cpu, k, float(np.max(np.abs(got - ref["mcd"]) / ref["mcd"]))),
          flush=True)

with tempfile.TemporaryDirectory() as d:
    os.makedirs(os.path.join(d, "mels")); os.makedirs(os.path.join(d, "mags"))
    F = 1 + hp.n_fft // 2
    chars = np.array(list("abcdefghijklmnopqrstuvwxyz "))
    fpaths, lens, texts = [], [], []
    for i in range(a.corpus):
        T = int(rng.integers(100, 211))
        np.save(os.path.join(d, "mels", "u%03d.npy" % i), rng.uniform(0, 1, (T, hp.n_mels)).astype(np.float32))
        np.save(os.path.join(d, "mags", "u%03d.npy" % i), rng.uniform(0, 1, (hp.r * T, F)).astype(np.float32))
        n = int(rng.integers(40, 151))
        ids = np.array([hp.vocab.index(c) for c in rng.choice(chars, n)] + [hp.vocab.index("E")], np.int32)
        fpaths.append(os.path.join(d, "u%03d.wav" % i)); lens.append(len(ids)); texts.append(ids)
    cwd = os.getcwd()
    os.chdir(d)
    try:
        for num in (1, 2):
            if num == 1:
                e.train_init(32)
            else:
                e.train_init_ssrn(32, hp.max_T)
            t0 = time.perf_counter()
            h = ho.HeldOut(e, fpaths, lens, texts, prepro=True, B=32)
            t_read = time.perf_counter() - t0
            h.run(e, num, 0)                                        # warm-up
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            rows, s = h.run(e, num, 0)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            print("HeldOut.run num = %d: %d utterances (%d evaluated) in %.2f s (%.1f utterances/s; reading the features "
                  "took %.2f s); mcd_mean %.3f" % (num, len(rows), s["evaluated"], dt, len(rows) / dt, t_read,
                                                   s.get("mcd_mean", float("nan"))), flush=True)
    finally:
        os.chdir(cwd)
