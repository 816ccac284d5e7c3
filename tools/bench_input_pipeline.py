"""Input pipeline of the trainers: the npy route (prepo.py's mels/ and mags/, hp.prepro = True) against the wav route
(features of each bucket on the device, trainer.bucketed_batches(..., prepro=False)).

Writes a seeded synthetic corpus shaped like LJ Speech into --out (int16 wavs of 1-10 s with silent lead-in and tail,
random transcripts; at --sample-rate, default hp.sr, resampled to hp.sr on the device when it differs), runs prepo,
then measures on cuda:0:
  - wall time per emitted batch at --batch, each ending in a device synchronise:
      npy route: np.load + zero padding + host-to-device copy;  wav route: read the wavs + one copy + features;
  - the device time of the feature call alone (CUDA events around Engine.load_spectrograms_batch on samples already read);
  - trainer steps/s (trainer.train) for num = 1 and num = 2 on each route, --steps steps after --warmup;
  - at another --sample-rate: the resampling kernel alone (CUDA events around dctts_resample_batch on samples already
    on the device) and, for context, the numpy oracle (oracle/ref_resample.py) resampling the first batch on the host.
Prints the card's name and power limit read in the same run, a markdown table, and one JSON line.

    python tools/bench_input_pipeline.py --out /tmp/dctts_input_bench
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from dc_tts_b200 import prepo, trainer  # noqa: E402
from dc_tts_b200.engine import Engine, set_engine  # noqa: E402
from dc_tts_b200.hyperparams import Hyperparams as hp  # noqa: E402
from dc_tts_b200.params import init_params  # noqa: E402
from dc_tts_b200.utils import _read_pcm  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except Exception:
        power = "unknown (nvidia-smi unavailable)"
    return name, power


def write_corpus(root, n, seed, sr):
    """LJ-shaped: LJSpeech-1.0/transcript.csv and wavs/*.wav, int16 at `sr`, speech-like tones with silent edges."""
    from scipy.io import wavfile
    rng = np.random.default_rng(seed)
    d = os.path.join(root, "LJSpeech-1.0")
    os.makedirs(os.path.join(d, "wavs"), exist_ok=True)
    lines = []
    for i in range(n):
        seconds = float(rng.uniform(1.0, 10.0))
        m = int(seconds * sr)
        t = np.arange(m) / sr
        f0 = rng.uniform(90, 250)
        env = 0.5 + 0.5 * np.sin(2 * np.pi * rng.uniform(2, 5) * t)
        y = sum(0.2 / k * np.sin(2 * np.pi * k * f0 * t) for k in range(1, 6)) * env + 0.02 * rng.standard_normal(m)
        lead, tail = int(rng.integers(1000, 8000)) * sr // hp.sr, int(rng.integers(1000, 8000)) * sr // hp.sr
        y[:lead] *= 1e-4
        y[m - tail:] *= 1e-4
        wavfile.write(os.path.join(d, "wavs", "LJ%04d.wav" % i), sr, np.round(np.clip(y, -1, 1) * 32767).astype(np.int16))
        nchar = int(np.clip(seconds * 15 + rng.normal(0, 10), 10, 170))
        lines.append("LJ%04d|raw|%s" % (i, "".join(rng.choice(list("abcdefghijklmnopqrstuvwxyz '.?"), nchar))))
    with open(os.path.join(d, "transcript.csv"), "w", encoding="utf-8") as f:
        f.write("\n".join(lines) + "\n")
    return d


def per_batch_ms(fn, groups, rounds):
    """Median over `rounds` of each group's wall time, averaged over the groups."""
    times = [[] for _ in groups]
    for _ in range(rounds):
        for j, g in enumerate(groups):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn(g)
            torch.cuda.synchronize()
            times[j].append(1e3 * (time.perf_counter() - t0))
    return statistics.mean(statistics.median(t) for t in times)


def steps_per_s(num, P, batches, warmup, steps, logdir):
    eng = Engine(0)
    eng.load_params(P)
    mark = {}

    def timed(it):
        for k, b in enumerate(it):
            if k == warmup:
                torch.cuda.synchronize()
                mark["t0"] = time.perf_counter()
            yield b
    gs = trainer.train(num, eng, timed(batches), num_iterations=warmup + steps - 1, logdir=logdir, global_step=0,
                       save_every=10 ** 9, log=lambda *_: None)
    torch.cuda.synchronize()
    dt = time.perf_counter() - mark["t0"]
    eng.close()
    assert gs == warmup + steps
    return steps / dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="corpus and npy directory (default: a new temporary directory)")
    ap.add_argument("--clips", type=int, default=256)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--sample-rate", type=int, default=None, help="sample rate of the corpus (default hp.sr)")
    ap.add_argument("--json", default=None, help="also write the result here")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_input_pipeline: needs a CUDA device")
    out = a.out or tempfile.mkdtemp(prefix="dctts_input_bench_")
    os.makedirs(out, exist_ok=True)
    name, power = card()
    sr = a.sample_rate or hp.sr
    d = write_corpus(out, a.clips, a.seed, sr)
    eng = set_engine(Engine(0))
    t0 = time.perf_counter()
    prepo.prepo(d, out, engine=eng, resample=True)
    torch.cuda.synchronize()
    prepo_s = time.perf_counter() - t0
    fpaths, lens, texts = trainer.load_train_data(d)
    mels_dir, mags_dir = os.path.join(out, "mels"), os.path.join(out, "mags")
    loader = lambda p: trainer._load_spectrograms_npy(p, mels_dir, mags_dir)
    B = a.batch

    # the utterance groups of one epoch of bucketed batches (routing does not depend on the route)
    groups = [[os.path.join(d, "wavs", nm) for nm in b[3]]
              for b in trainer.bucketed_batches(fpaths, lens, texts, B=B, seed=a.seed, loader=loader, epochs=1)]
    dev = torch.device("cuda", 0)

    def npy_batch(g):
        mels, mags = trainer._pad_spectrograms([loader(p)[1:] for p in g])
        return torch.from_numpy(mels).to(dev), torch.from_numpy(mags).to(dev)

    def wav_batch(g):
        pcms, rates = zip(*[_read_pcm(p) for p in g])
        return eng.load_spectrograms_batch(list(pcms), rates=list(rates))

    for g in groups:                                   # warm the page cache and every shape
        npy_batch(g); wav_batch(g)
    npy_ms = per_batch_ms(npy_batch, groups, a.rounds)
    wav_ms = per_batch_ms(wav_batch, groups, a.rounds)

    pcms = [[_read_pcm(p)[0] for p in g] for g in groups]
    rates = [[sr] * len(g) for g in groups]
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dev_ms = []
    for _ in range(a.rounds):
        for pc, rt in zip(pcms, rates):
            ev0.record()
            eng.load_spectrograms_batch(pc, rates=rt)
            ev1.record()
            ev1.synchronize()
            dev_ms.append(ev0.elapsed_time(ev1))
    feat_dev_ms = statistics.median(dev_ms)
    frames = statistics.mean(sum(1 + (round(len(p) * hp.sr / sr) // hp.hop_length) for p in pc) for pc in pcms)
    resample_ms = oracle_s = None
    if sr != hp.sr:
        packed = [eng._pack(pc, "bench") for pc in pcms]
        buf = None
        for wav, dtype, offsets in packed:                # warm-up, and the output buffer at its largest
            buf, _ = eng._resample(wav, dtype, offsets, [sr] * (len(offsets) - 1), hp.sr, buf)
        rs = []
        for _ in range(a.rounds):
            for wav, dtype, offsets in packed:
                ev0.record()
                eng._resample(wav, dtype, offsets, [sr] * (len(offsets) - 1), hp.sr, buf)
                ev1.record()
                ev1.synchronize()
                rs.append(ev0.elapsed_time(ev1))
        resample_ms = statistics.median(rs)
        from oracle import ref_resample as rr
        t0 = time.perf_counter()
        for p in pcms[0]:
            rr.load(p, sr, hp.sr)
        oracle_s = time.perf_counter() - t0

    P = init_params(1)
    rates = {}
    for num in (1, 2):
        rates["npy_num%d" % num] = steps_per_s(num, P, trainer.bucketed_batches(fpaths, lens, texts, B=B, seed=a.seed, loader=loader),
                                               a.warmup, a.steps, os.path.join(out, "ld_npy%d" % num))
        rates["wav_num%d" % num] = steps_per_s(num, P, trainer.bucketed_batches(fpaths, lens, texts, B=B, seed=a.seed, prepro=False,
                                                                                engine=eng, resample=True),
                                               a.warmup, a.steps, os.path.join(out, "ld_wav%d" % num))
    res = {"device": name, "power_limit": power, "sample_rate": sr, "clips": a.clips, "B": B, "batches_per_epoch": len(groups),
           "resample_kernel_ms": None if resample_ms is None else round(resample_ms, 3),
           "oracle_resample_one_batch_s": None if oracle_s is None else round(oracle_s, 2),
           "prepo_s": round(prepo_s, 2), "npy_batch_ms": round(npy_ms, 2), "wav_batch_ms": round(wav_ms, 2),
           "feature_call_device_ms": round(feat_dev_ms, 3), "untrimmed_frames_per_batch": round(frames),
           "steps_per_s": {k: round(v, 2) for k, v in rates.items()}, "steps": a.steps, "warmup": a.warmup}
    print("%s, power limit %s; %d clips at %d Hz, B = %d, %d batches per epoch" % (name, power, a.clips, sr, B, len(groups)))
    print("| | npy route | wav route |")
    print("|---|---|---|")
    print("| wall time per batch (ms) | %.1f | %.1f |" % (npy_ms, wav_ms))
    print("| feature call, device (ms) | - | %.2f |" % feat_dev_ms)
    if resample_ms is not None:
        print("| of which the resampling kernel (ms) | - | %.3f |" % resample_ms)
        print("| numpy oracle, resampling one batch on the host (s) | - | %.2f |" % oracle_s)
    print("| Text2Mel steps/s | %.2f | %.2f |" % (rates["npy_num1"], rates["wav_num1"]))
    print("| SSRN steps/s | %.2f | %.2f |" % (rates["npy_num2"], rates["wav_num2"]))
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
