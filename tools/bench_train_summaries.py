"""Text2Mel training steps/s through trainer.train with summaries=True (default summary_secs = 120) against
summaries=False, alternated in one process on one engine: B = 32, synthetic (N, T) = (180, 210) batches, no checkpoints.
Prints one JSON line with both rates per round and the card's name and power limit.
    python tools/bench_train_summaries.py [--steps 400 --rounds 3]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from dc_tts_b200 import trainer
from dc_tts_b200.engine import Engine
from dc_tts_b200.hyperparams import Hyperparams as hp
from dc_tts_b200.params import init_params, synthetic_text

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=400)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--batch", type=int, default=32)
a = ap.parse_args()
B = a.batch
L = synthetic_text(B, 100, seed=0)[:, :hp.max_N]
mels = torch.from_numpy(np.random.default_rng(0).uniform(0, 1, (B, hp.max_T, hp.n_mels)).astype(np.float32)).cuda()


def batches():
    while True:
        yield L, mels, None


eng = Engine(0)
eng.load_params(init_params(0))
out = {"off": [], "on": []}
with tempfile.TemporaryDirectory() as tmp:
    trainer.train(1, eng, batches(), num_iterations=20, logdir=os.path.join(tmp, "warm"), save_every=10 ** 9, log=lambda s: None)
    for r in range(a.rounds):
        for mode in ("off", "on"):
            logdir = os.path.join(tmp, "%s%d" % (mode, r))
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            trainer.train(1, eng, batches(), num_iterations=a.steps - 1, logdir=logdir, global_step=0, save_every=10 ** 9,
                          log=lambda s: None, summaries=(mode == "on"))
            torch.cuda.synchronize()
            out[mode].append(a.steps / (time.perf_counter() - t0))
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = torch.cuda.get_device_name() + ", power limit unknown"
print(json.dumps({"metric": "trainer_steps_per_sec", "summaries_off": out["off"], "summaries_on": out["on"], "steps": a.steps,
                  "B": B, "shape": {"N": hp.max_N, "T": hp.max_T}, "summary_secs": 120, "device": card}))
