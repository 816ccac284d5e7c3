"""Time the decode along a window path (Engine.text2mel_generate_path) on the persistent decode, CUDA events, the
variants alternated in one run:
  free B           text2mel_generate, every frame following its own argmax
  replay B         text2mel_generate_path along the window history of that free run (expected equal within noise); the
                   Engine passes host arrays (dctts_text2mel_generate_path_host)
  replay dev-entry B   the same through dctts_text2mel_generate_path with the arrays on the device, which reads them
                   back to check them and so waits for the previous call's decode before it can queue the next
  stretch 1.25 B   text2mel_generate_path along that history stretched by 1.25 (utils.stretch_path) from 160 frames
at B = 1 and 32.
   python tools/bench_window_path.py [--reps 3] [--iters 5]"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from dc_tts_b200.engine import Engine, _ptr  # noqa: E402
from dc_tts_b200.hyperparams import Hyperparams as hp  # noqa: E402
from dc_tts_b200.params import init_params, synthetic_text  # noqa: E402
from dc_tts_b200.utils import stretch_path  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--iters", type=int, default=5)
a = ap.parse_args()
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
except (OSError, IndexError):
    card = "unknown"
print("card:", card, flush=True)

e = Engine(0)
e.load_params(init_params(0, "perturbed"))
assert e.get_option("decode_available"), "no persistent decode on this device"


def timed(fn):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(a.iters):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / a.iters


def device_entry(L, P):
    """The replay through dctts_text2mel_generate_path, path and lengths already on the device: the entry point reads
    them back to check them, which waits for the stream."""
    Ld, Pd, nd = e._i32(L), e._i32(P), e._i32(np.full(len(L), P.shape[1]))
    Y = e._empty(len(L), hp.max_T, hp.n_mels)
    H, M = e._empty(len(L), hp.max_T, dtype=torch.int32), e._empty(len(L), hp.max_T, dtype=torch.int32)

    def run():
        rc = e._lib.dctts_text2mel_generate_path(e._h, _ptr(Ld), len(L), P.shape[1], _ptr(Pd), _ptr(nd), _ptr(Y),
                                                 _ptr(H), _ptr(M), e._stream())
        assert rc == 0, e._lib.dctts_last_error(e._h)
    return run


runs = {}
for B in (1, 32):
    L = np.concatenate([synthetic_text(1, 100, seed=700 + b) for b in range(B)])
    Yf, Pf, _, _ = e.text2mel_generate(L)
    P = Pf.cpu().numpy()
    Yr, _, _ = e.text2mel_generate_path(L, P)
    assert torch.equal(Yr, Yf), "replay differs from the free run"
    ps, ns = stretch_path(P, np.full(B, 160), 1.25)
    runs["free %d" % B] = (lambda L=L: e.text2mel_generate(L))
    runs["replay %d" % B] = (lambda L=L, P=P: e.text2mel_generate_path(L, P))
    runs["replay dev-entry %d" % B] = device_entry(L, P)
    runs["stretch 1.25 %d" % B] = (lambda L=L, ps=ps, ns=ns: e.text2mel_generate_path(L, ps, ns))
for fn in runs.values():
    fn()
torch.cuda.synchronize()
res = {k: [] for k in runs}
for rep in range(a.reps):
    for k, fn in runs.items():
        res[k].append(timed(fn))
for k, v in res.items():
    print("%-18s %s ms (median %.2f)" % (k, " ".join("%.2f" % x for x in v), float(np.median(v))), flush=True)
