"""What synthesis from the weights being trained costs (Engine.refresh_synthesis), on the GPU:

  refresh      one refresh of a trained Text2Mel handle at the stock hyper-parameters (CUDA events around it; it ends in a
               device synchronise), median of 10
  t2m / ssrn   Text2Mel generation at B = 20 (harvard_sentences.txt) and B = 32 (synthetic texts), full length and until
               EOS, and SSRN on the full-length mels, on a trained handle without a refresh (fp32 kernels, graph-per-frame
               decode: what a trained handle ran before refresh_synthesis existed) and after one
  trainer      Text2Mel steps/s through trainer.train with samples at every checkpoint on and off, alternated three times
               (save_every steps per leg; the samples are the 20 Harvard sentences)

Random weights: the decode runs all max_T frames unless an attention window reaches EOS.  Prints one JSON line with the
card's name and power limit, read in the same run.  Run from the repository root: python tools/bench_refresh.py"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception as e:          # the numbers are still printed, marked as such
        return "unknown (%s)" % e, "unknown"


def timed(fn, reps):
    """Median wall time (ms) of fn() over reps runs, each ended by a device synchronise; one warm-up run first."""
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--save-every", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_refresh needs a GPU"
    from dc_tts_b200 import trainer
    from dc_tts_b200.data_load import load_data
    from dc_tts_b200.engine import Engine
    from dc_tts_b200.hyperparams import Hyperparams as hp
    from dc_tts_b200.params import init_params, synthetic_text

    name, power = card()
    P = init_params(0, "perturbed")
    harvard = load_data("synthesize", os.path.join(ROOT, "harvard_sentences.txt"))
    batches = {"harvard20": harvard, "synthetic32": synthetic_text(32, 100, seed=1)}
    L2 = synthetic_text(2, 50, seed=7)
    mels2 = np.random.default_rng(3).uniform(0, 1, (2, hp.max_T, hp.n_mels)).astype(np.float32)

    e = Engine(0)
    e.load_params(P)
    e.train_init(2)
    e.train_step(L2, mels2, global_step=4000, seed=0)
    res = {"card": name, "power_limit": power}

    # one refresh: every call re-packs (a step in between makes the packing stale again)
    ts = []
    for i in range(10):
        e.train_step(L2, mels2, global_step=4001 + i, seed=i)
        torch.cuda.synchronize()
        s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s0.record()
        e.refresh_synthesis()
        s1.record()
        torch.cuda.synchronize()
        ts.append(s0.elapsed_time(s1))
    res["refresh_ms"] = float(np.median(ts))
    e.train_step(L2, mels2, global_step=4100, seed=0)         # stale again

    for refreshed in (False, True):
        if refreshed:
            e.refresh_synthesis()
        leg = "refreshed" if refreshed else "stale"
        for bname, L in batches.items():
            Y = e.text2mel_generate(L)[0]
            res["%s_%s_t2m_full_ms" % (leg, bname)] = timed(lambda: e.text2mel_generate(L), a.reps)
            res["%s_%s_t2m_until_eos_ms" % (leg, bname)] = timed(lambda: e.text2mel_generate_until(L), a.reps)
            res["%s_%s_ssrn_ms" % (leg, bname)] = timed(lambda: e.ssrn(Y, want_logits=False), a.reps)
    e.close()

    # steps/s of the trainer, samples on and off, alternated
    sents = [s for s in open(os.path.join(ROOT, "harvard_sentences.txt"), encoding="utf-8").read().splitlines()[1:] if s.strip()]
    sents = [s.split(" ", 1)[-1] for s in sents]
    rates = {"on": [], "off": []}
    for _ in range(3):
        for mode in ("off", "on"):
            eng = Engine(0)
            eng.load_params(P)
            n = a.save_every
            with tempfile.TemporaryDirectory() as d:
                data = [(L2, mels2, None)] * (n + 2)
                t0 = time.perf_counter()
                trainer.train(1, eng, data, num_iterations=n - 1, logdir=d, save_every=n, log=lambda *_: None,
                              samples=sents if mode == "on" else None)
                torch.cuda.synchronize()
                rates[mode].append(n / (time.perf_counter() - t0))
            eng.close()
    res["trainer_steps_per_s_samples_off"] = rates["off"]
    res["trainer_steps_per_s_samples_on"] = rates["on"]
    res["trainer_save_every"] = a.save_every
    print(json.dumps(res))


if __name__ == "__main__":
    main()
