"""BASELINE config 5: Text2Mel training step, B = 32 per GPU, fixed N = 180 / T = 210, synthetic batch, dropout on,
data-parallel over the launched ranks (gradient all-reduce of the flat arena over NCCL).  Prints one JSON line.
`--shape N,T` steps at a length bucket's own shape instead (the workspace keeps its (max_N, max_T) capacity); with
`--reserve N,T` the workspace is first grown to that capacity (Engine.train_reserve, timed once: "reserve_ms"), so `--shape`
can go past (max_N, max_T).  `--eval` also times the forward-only evaluation of the training graph on the same batch
(what summaries and alignment plots cost: "eval_ms").  The card's name and power limit are part of the JSON line.
`--deterministic` runs the step with the option "train_deterministic" (its sums in a fixed order).
    python tools/bench_train.py [--steps 10 --warmup 3 --batch 32 --net 1 --shape 180,210 --reserve 256,256 --eval --deterministic]
    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tools/bench_train.py"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.distributed as dist

from dc_tts_b200.engine import Engine
from dc_tts_b200.hyperparams import Hyperparams as hp
from dc_tts_b200.params import init_params, synthetic_text

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--batch", type=int, default=32)
ap.add_argument("--probe", type=int, default=0, help="measurement only: 1 = the wgmma GEMMs fetch their operands but issue no MMA (results are garbage)")
ap.add_argument("--net", type=int, default=1, choices=[1, 2], help="1 = Text2Mel trainer (BASELINE config 5), 2 = SSRN trainer (train.py num=2) at T = 210")
ap.add_argument("--shape", default="%d,%d" % (hp.max_N, hp.max_T), help="N,T of every step's batch (text positions, mel frames); SSRN uses T")
ap.add_argument("--reserve", default=None, help="N,T: grow the training workspace to this capacity after init (SSRN uses T)")
ap.add_argument("--eval", action="store_true", help="also time Engine.train_eval / train_eval_ssrn (forward only, no update) on the same batch: eval_ms")
ap.add_argument("--train-tc", type=int, default=7, help="bit mask: 1 forward conv, 2 data gradient, 4 weight gradient on wgmma (default 7 = all), 0 = fp32 CUDA-core kernels")
ap.add_argument("--deterministic", action="store_true", help="option train_deterministic: the step's sums in a fixed order (bit-reproducible)")
a = ap.parse_args()
N, T = (int(x) for x in a.shape.split(","))
rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
torch.cuda.set_device(local)
if world > 1:
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
eng = Engine(local)
eng.load_params(init_params(0))
B = a.batch
eng.set_option("train_tc", a.train_tc)
eng.set_option("train_probe", a.probe)
eng.set_option("train_deterministic", 1 if a.deterministic else 0)
if a.net == 1:
    eng.train_init(B)
else:
    eng.train_init_ssrn(B, hp.max_T)
reserve_ms = None
if a.reserve:
    RN, RT = (int(x) for x in a.reserve.split(","))
    torch.cuda.synchronize()
    w0 = time.perf_counter()
    eng.train_reserve(RN, RT)                       # synchronises the device when it grows
    reserve_ms = (time.perf_counter() - w0) * 1e3


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(local)],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ", power limit unknown"

L = torch.from_numpy(synthetic_text(B, min(100, N - 1), seed=rank)[:, :N]).cuda()
mels = torch.from_numpy(np.random.default_rng(rank).uniform(0, 1, (B, T, hp.n_mels)).astype(np.float32)).cuda()
mags = torch.from_numpy(np.random.default_rng(rank + 100).uniform(0, 1, (B, T * hp.r, 1 + hp.n_fft // 2)).astype(np.float32)).cuda() if a.net == 2 else None
grads = eng.train_grads()


def step(i):
    if a.net == 2:
        out = eng.train_step_ssrn(mels, mags, global_step=4000 + i, seed=i * world + rank, apply=(world == 1))
    else:
        out = eng.train_step(L, mels, global_step=4000 + i, seed=i * world + rank, apply=(world == 1))
    if world > 1:
        dist.all_reduce(grads)
        grads.mul_(1.0 / world)
        eng.train_apply(4000 + i)
    return out


for i in range(a.warmup):
    first = step(i)
torch.cuda.synchronize()
if world > 1:
    dist.barrier()
t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
n0 = eng.launch_count()
t0.record()
for i in range(a.steps):
    last = step(a.warmup + i)
t1.record()
torch.cuda.synchronize()
ms = torch.tensor([t0.elapsed_time(t1) / a.steps], device="cuda")
if world > 1:
    dist.all_reduce(ms, op=dist.ReduceOp.MAX)
eval_ms = None
if a.eval:                                          # the forward-only evaluation of the same batch (summaries, alignment plots)
    def evaluate():
        return eng.train_eval_ssrn(mels, mags, seed=0xffffffff) if a.net == 2 else eng.train_eval(L, mels, seed=0xffffffff)
    for _ in range(a.warmup):
        evaluate()
    torch.cuda.synchronize()
    t0.record()
    for _ in range(a.steps):
        evaluate()
    t1.record()
    torch.cuda.synchronize()
    eval_ms = t0.elapsed_time(t1) / a.steps
if rank == 0:
    ms = float(ms)
    flops = 3 * 2 * B * (N * 17.10e6 + T * (4.08e6 + 2.71e6 + 0.09e6))                    # SURVEY 8(d) config 5: fwd MACs x 2 x 3
    if a.net == 2:
        flops = 3 * 2 * B * T * 93.66e6                                                          # SSRN: 93.7 MMAC per mel frame
    print(json.dumps({"metric": "train_steps_per_sec", "value": 1e3 / ms, "unit": "steps/s", "n_gpus": world, "ms_per_step": ms,
                      "mel_frames_per_sec": world * B * T * 1e3 / ms, "steps": a.steps, "warmup": a.warmup, "shape": {"N": N, "T": T},
                      "capacity": dict(zip(("N", "T"), eng.train_capacity())), "reserve_ms": reserve_ms, "device": card(),
                      "config": {"workload": ("Text2Mel train step (fwd + bwd + clip + Adam), B=%d per GPU, N=%d, T=%d, dropout %.2f" % (B, N, T, hp.dropout_rate)
                                              if a.net == 1 else
                                              "SSRN train step (train.py num=2: fwd + bwd + clip + Adam), B=%d per GPU, T=%d -> %d frames x 1025 bins, dropout %.2f"
                                              % (B, T, T * hp.r, hp.dropout_rate)),
                                 "parallelism": "dp%d (all-reduce of %d gradients)" % (world, grads.numel())},
                      "dtype": ("f32 tensors; GEMMs as split-fp16 x3 on wgmma, fp32 accumulate" if a.train_tc else "f32 (CUDA-core kernels)"), "data": "synthetic", "deterministic": a.deterministic,
                      "achieved_tflops": world * flops / (ms * 1e-3) / 1e12, "gpu_launches_per_step": (eng.launch_count() - n0) // a.steps,
                      "loss_first": first["loss"], "loss_last": last["loss"],
                      "eval_ms": eval_ms, "eval_over_step": None if eval_ms is None else eval_ms / ms}))
if world > 1:
    dist.destroy_process_group()
