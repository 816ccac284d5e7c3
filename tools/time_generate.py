"""Time Text2Mel generation (TextEnc + 210 frames) for a list of batch sizes, persistent cluster decode
(decode_mode 1) next to the graph-per-frame loop (decode_mode 0), and compare their outputs.
   python tools/time_generate.py 1 32 [--steps N] [--modes 1,0]"""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from dc_tts_b200.engine import Engine  # noqa: E402
from dc_tts_b200.params import init_params, synthetic_text  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("batches", type=int, nargs="*", default=[1, 32])
ap.add_argument("--steps", type=int, default=210)
ap.add_argument("--modes", default="1,0", help="decode modes to time: 1 persistent cluster kernel, 0 graph per frame")
ap.add_argument("--iters", type=int, default=5)
ap.add_argument("--prof", action="store_true", help="print the in-kernel lap timers of the persistent decode")
ap.add_argument("--option", action="append", default=[], metavar="NAME=VALUE",
                help="engine option to set first, e.g. decode_force_prepass=1 (the recompute at every frame)")
a = ap.parse_args()
e = Engine(0)
e.load_params(init_params(0, "perturbed"))
for kv in a.option:
    name, val = kv.split("=")
    e.set_option(name, int(val))
print("decode_available", e.get_option("decode_available"), "max co-resident clusters", e.get_option("decode_max_clusters"), flush=True)
for B in a.batches:
    L = synthetic_text(B, 100, seed=0)
    outs = {}
    for mode in [int(m) for m in a.modes.split(",")]:
        e.set_option("decode_mode", 1 if mode else 0)
        for _ in range(2):
            e.text2mel_generate(L, steps=a.steps)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.iters):
            Y, P, _, _ = e.text2mel_generate(L, steps=a.steps)
        torch.cuda.synchronize()
        dt = (time.perf_counter() - t0) / a.iters
        extra = ""
        if mode >= 1:
            fr, ut, cl = e.decode_stats()
            extra = "  clusters %d, cluster-frames with a recompute %d, utterance-frames recomputed %d" % (cl, fr, ut)
        print("generate B=%d mode=%d: %.2f ms (%.1f us/frame)  checksum %.6f%s"
              % (B, mode, dt * 1e3, dt * 1e6 / a.steps, float(Y.double().sum()), extra), flush=True)
        outs[mode] = (Y, P)
        if mode >= 1 and a.prof:
            e.set_option("decode_prof", 1)
            e.text2mel_generate(L, steps=a.steps)
            pr = e.decode_profile()
            e.set_option("decode_prof", 0)
            wg = {k: v for k, v in pr.items() if k.startswith("wg_")}   # the MMA warpgroup's laps overlap thread 0's
            tot = float(sum(v for k, v in pr.items() if k not in wg)) or 1.0
            print("   lap timers (cluster 0, rank 0; %% of %.1f Mcycles): " % (tot / 1e6)
                  + ", ".join("%s %.1f" % (k, 100.0 * v / tot) for k, v in pr.items() if k not in wg), flush=True)
            print("   recompute laps (Mcycles): "
                  + ", ".join("%s %.2f" % (k, v / 1e6) for k, v in pr.items() if k.startswith("re_")) + "; MMA warpgroup: "
                  + ", ".join("%s %.2f" % (k, v / 1e6) for k, v in wg.items()), flush=True)
    ref = outs.get(0, outs.get(1))
    if ref is None:
        continue
    for m, (Y1, P1) in outs.items():
        if (Y1 is ref[0]):
            continue
        same = (ref[1] == P1).all(dim=1)
        print("   mode %d vs mode %d: windows equal for %d/%d utterances; max|dY| over those %.3e"
              % (m, 0 if 0 in outs else 1, int(same.sum()), B, float((ref[0][same] - Y1[same]).abs().max()) if same.any() else float("nan")), flush=True)
e.set_option("decode_mode", 1)
