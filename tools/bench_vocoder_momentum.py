"""Time the Griffin-Lim vocoder with and without momentum, and measure what momentum gains in spectral convergence.

B = 32 utterances of 840 magnitude frames (10.5 s at 22.05 kHz), n_iter = 50; three variants alternated in one run,
CUDA events around `--iters` calls each, all three through dctts_spectrogram2wav_momentum:
  plain          Engine.spectrogram2wav(mag)                              (momentum 0: the plain update)
  momentum       Engine.spectrogram2wav(mag, momentum=0.99)
  momentum+conv  Engine.spectrogram2wav(mag, momentum=0.99, convergence=True)
The magnitudes are the on-device features (Engine.get_spectrograms) of seeded synthetic signals: harmonic tones with
vibrato, chirps and noise bursts, cycled over the batch.  Then, from the convergence histories of plain Griffin-Lim and of
momentum 0.99: the first iteration at which momentum reaches plain Griffin-Lim's 50-iteration spectral convergence, per
utterance.  No trained model is involved: spectral convergence stands in for how the result sounds.
   python tools/bench_vocoder_momentum.py [--reps 5] [--iters 5]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from dc_tts_b200.engine import Engine  # noqa: E402
from dc_tts_b200.hyperparams import Hyperparams as hp  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--iters", type=int, default=5)
ap.add_argument("--momentum", type=float, default=0.99)
a = ap.parse_args()
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
except (OSError, IndexError):
    card = "unknown"
print("card:", card, flush=True)

B, T, N_ITER = 32, 840, 50


def signal(b, seconds=11.0):
    rng = np.random.default_rng(b)
    n = int(seconds * hp.sr)
    t = np.arange(n) / hp.sr
    kind = b % 3
    if kind == 0:                                        # harmonic tone with vibrato and a slow level change
        f0 = rng.uniform(100, 220) * (1 + 0.05 * np.sin(2 * np.pi * rng.uniform(4, 7) * t))
        ph = 2 * np.pi * np.cumsum(f0) / hp.sr
        y = sum(0.3 / h * np.sin(h * ph) for h in range(1, 9)) * (0.6 + 0.4 * np.sin(2 * np.pi * 0.7 * t))
    elif kind == 1:                                      # linear chirp
        f1 = rng.uniform(1000, 5000)
        y = 0.5 * np.sin(2 * np.pi * (150.0 * t + 0.5 * f1 * t * t / seconds))
    else:                                                # noise bursts over a noise floor
        y = 0.02 * rng.standard_normal(n)
        m = int(0.1 * hp.sr)
        for start in rng.uniform(0, seconds - 0.12, 60):
            i = int(start * hp.sr)
            y[i:i + m] += 0.4 * rng.standard_normal(m) * np.hanning(m)
    return np.clip(y, -1, 1).astype(np.float32)


e = Engine(0)
mags = []
for b in range(B):
    _, m, _ = e.get_spectrograms(signal(b))
    assert m.shape[0] >= T, m.shape
    mags.append(m[:T])
mag = torch.stack(mags).contiguous()
torch.cuda.synchronize()


def timed(fn):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(a.iters):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / a.iters


runs = {
    "plain": lambda: e.spectrogram2wav(mag, n_iter=N_ITER),
    "momentum": lambda: e.spectrogram2wav(mag, n_iter=N_ITER, momentum=a.momentum),
    "momentum+conv": lambda: e.spectrogram2wav(mag, n_iter=N_ITER, momentum=a.momentum, convergence=True),
}
for fn in runs.values():
    fn()
torch.cuda.synchronize()
res = {k: [] for k in runs}
for rep in range(a.reps):
    for k, fn in runs.items():
        res[k].append(timed(fn))
for k, v in res.items():
    print("%-14s %s ms (median %.2f)" % (k, " ".join("%.2f" % x for x in v), float(np.median(v))), flush=True)

_, _, plain = e.spectrogram2wav(mag, n_iter=N_ITER, convergence=True)
_, _, fast = e.spectrogram2wav(mag, n_iter=N_ITER, momentum=a.momentum, convergence=True)
plain, fast = plain.cpu().numpy(), fast.cpu().numpy()
reach = [int(np.argmax(fast[b] <= plain[b, -1])) if (fast[b] <= plain[b, -1]).any() else None for b in range(B)]
for kind, name in enumerate(("vibrato", "chirp", "bursts")):
    sel = list(range(kind, B, 3))
    r = [reach[b] for b in sel]
    print("%-8s spectral convergence at 50 iterations: plain %.4f, momentum %.4f (means); momentum reaches plain's "
          "50-iteration value at iteration %s" % (name, plain[sel, -1].mean(), fast[sel, -1].mean(), r), flush=True)
print(json.dumps({"card": card, "B": B, "T": T, "n_iter": N_ITER, "momentum": a.momentum,
                  "ms_median": {k: float(np.median(v)) for k, v in res.items()},
                  "sc50_plain_mean": float(plain[:, -1].mean()), "sc50_momentum_mean": float(fast[:, -1].mean()),
                  "reach_iteration": reach}))
e.close()
