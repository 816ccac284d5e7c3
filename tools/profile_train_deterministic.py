"""Where the time of the option "train_deterministic" goes: torch.profiler over `--steps` Text2Mel (or SSRN) training steps
with the option off and on, on the same batch, and the CUDA time per step of every kernel name in both modes, sorted by
the difference.  Prints a table and one JSON line with the card's name and power limit; writes nothing unless `--out`
names a directory for the two Chrome traces.
    python tools/profile_train_deterministic.py [--net 1 --batch 32 --shape 180,210 --steps 10 --warmup 3 --out DIR]"""
import argparse
import collections
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from dc_tts_b200.engine import Engine  # noqa: E402
from dc_tts_b200.hyperparams import Hyperparams as hp  # noqa: E402
from dc_tts_b200.params import init_params, synthetic_text  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--net", type=int, default=1, choices=[1, 2])
ap.add_argument("--batch", type=int, default=32)
ap.add_argument("--shape", default="%d,%d" % (hp.max_N, hp.max_T))
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--out", default=None, help="directory for the Chrome traces (default: none written)")
a = ap.parse_args()
N, T, B = (*(int(x) for x in a.shape.split(",")), a.batch)

eng = Engine(0)
eng.load_params(init_params(0))
if a.net == 1:
    eng.train_init(B)
else:
    eng.train_init_ssrn(B, hp.max_T)
L = torch.from_numpy(synthetic_text(B, min(100, N - 1), seed=0)[:, :N]).cuda()
mels = torch.from_numpy(np.random.default_rng(0).uniform(0, 1, (B, T, hp.n_mels)).astype(np.float32)).cuda()
mags = torch.from_numpy(np.random.default_rng(1).uniform(0, 1, (B, T * hp.r, 1 + hp.n_fft // 2)).astype(np.float32)).cuda() \
    if a.net == 2 else None


def step(i):
    if a.net == 2:
        eng.train_step_ssrn(mels, mags, global_step=4000 + i, seed=i)
    else:
        eng.train_step(L, mels, global_step=4000 + i, seed=i)


def kernel_ms(det):
    eng.set_option("train_deterministic", det)
    for i in range(a.warmup):
        step(i)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(a.steps):
            step(a.warmup + i)
        torch.cuda.synchronize()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        prof.export_chrome_trace(os.path.join(a.out, "train_det%d.pt.trace.json" % det))
    per = collections.defaultdict(float)
    for ev in prof.key_averages():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            per[ev.key.replace("(anonymous namespace)::", "").split("(")[0][:90]] += ev.device_time_total / 1e3 / a.steps
    return per


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip() or torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ", power limit unknown"


off, on = kernel_ms(0), kernel_ms(1)
rows = sorted(set(off) | set(on), key=lambda k: -(on.get(k, 0.0) - off.get(k, 0.0)))
print("%-90s %9s %9s %9s" % ("kernel (ms per step)", "default", "ordered", "delta"))
for k in rows:
    d = on.get(k, 0.0) - off.get(k, 0.0)
    if abs(d) >= 0.005 or k in on and k not in off:
        print("%-90s %9.3f %9.3f %+9.3f" % (k, off.get(k, 0.0), on.get(k, 0.0), d))
print(json.dumps({"net": a.net, "B": B, "shape": {"N": N, "T": T}, "kernel_ms_default": sum(off.values()),
                  "kernel_ms_ordered": sum(on.values()), "device": card()}))
