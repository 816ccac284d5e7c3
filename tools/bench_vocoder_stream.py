"""Time the streaming Griffin-Lim vocoder against whole-signal Griffin-Lim on the same magnitudes.

B utterances of 840 magnitude frames (10.5 s at 22.05 kHz), n_iter = 50, plain and with momentum 0.99.  The magnitudes
are the reference features (oracle/ref_features.get_spectrograms) of the seeded synthetic signals of
tests/ref_vocoder_stages.py (vibrato, chirp, noise bursts), cycled over the batch.  The frames are pushed `chunk` at a
time as fast as the stream takes them (a stand-in for a decoder that is never the bottleneck), and for each push:
  first    host clock from the first push to the return of the first push that committed samples
  total    host clock from the first push to the return of the final push, against Engine.spectrogram2wav of the
           whole batch in the same run (host clock around the call, which synchronises)
  underrun whether, at the return of every push, the audio committed so far (per utterance, at hp.sr) is ahead of the
           wall time since the first chunk arrived
Every figure is the median of `--reps` repetitions after one warm-up.
   python tools/bench_vocoder_stream.py [--reps 5] [--B 1 4] [--chunks 16 32 64]"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from dc_tts_b200.engine import Engine  # noqa: E402
from dc_tts_b200.hyperparams import Hyperparams as hp  # noqa: E402
from oracle import ref_features as rf  # noqa: E402
import ref_vocoder_stages as rs  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--B", type=int, nargs="+", default=[1, 4])
ap.add_argument("--chunks", type=int, nargs="+", default=[16, 32, 64])
a = ap.parse_args()
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
except (OSError, IndexError):
    card = "unknown"
print("card:", card, flush=True)

T, N_ITER = 840, 50
mags = [rf.get_spectrograms(rs.signal(k, seconds=11.0))[1][:T] for k in rs.SIGNALS]
eng = Engine(0)


def streamed(mag, chunk, momentum):
    B = mag.shape[0]
    vs = eng.vocoder_stream(B, T, n_iter=N_ITER, momentum=momentum)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    first, committed, ok = None, 0, True
    for s in range(0, T, chunk):
        out = vs.push(mag[:, s:s + chunk], [min(chunk, T - s)] * B, s + chunk >= T)
        now = time.perf_counter()
        n = min(o.size for o in out)
        if first is None and n:
            first = now
        committed += n
        if first is not None:
            ok = ok and committed / hp.sr >= now - first
    vs.close()
    return first - t0, time.perf_counter() - t0, ok


def whole(mag, momentum):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    eng.spectrogram2wav(mag, n_iter=N_ITER, momentum=momentum)
    return time.perf_counter() - t0


rows = []
for B in a.B:
    mag = torch.from_numpy(np.stack([mags[b % 3] for b in range(B)])).cuda()
    for momentum in (0.0, 0.99):
        whole(mag, momentum)
        t_whole = float(np.median([whole(mag, momentum) for _ in range(a.reps)]))
        for chunk in a.chunks:
            streamed(mag, chunk, momentum)
            runs = [streamed(mag, chunk, momentum) for _ in range(a.reps)]
            row = dict(B=B, momentum=momentum, chunk=chunk, first_ms=1e3 * float(np.median([r[0] for r in runs])),
                       total_ms=1e3 * float(np.median([r[1] for r in runs])), whole_ms=1e3 * t_whole,
                       no_underrun=all(r[2] for r in runs), audio_s=(T - 1) * hp.hop_length / hp.sr)
            rows.append(row)
            print(json.dumps(row), flush=True)
print(json.dumps(dict(card=card, rows=rows)))
eng.close()
