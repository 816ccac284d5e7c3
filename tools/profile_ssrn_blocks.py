"""Per-block times of SSRN and TextEnc on the tensor path (CUDA events, warm), with achieved TFLOP/s.

    python tools/profile_ssrn_blocks.py [--batch 32] [--frames 210] [--iters 10] [--cycles SSRN/HC_11,SSRN/HC_8,SSRN/C_14]
                                        [--option name=value ...] [--json out.json]

For every block: the per-launch times that dctts_bench_block reports (tensor path: [plane conversion, fused block]), the
algorithmic TFLOP/s of the fused block (2 x rows x taps x cin x cout of the reference layer) and the TFLOP/s the tensor
pipe executes (three fp16 products per k-step over the padded tile: rows to 128, cin to 64, cout to the CTAs' columns).
Then the whole Engine.ssrn at (B, T) and, for the blocks named by --cycles, the cycle split of CTA 0 from one launch with
option tc_debug = 1.  The card's name and power limit are printed with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from dc_tts_b200.engine import Engine  # noqa: E402
from dc_tts_b200.hyperparams import Hyperparams as hp  # noqa: E402
from dc_tts_b200.params import init_params  # noqa: E402


def rup(x, m):
    return (x + m - 1) // m * m


def block_table(F):
    """(scope, kind, cin, cout, taps, L factor over T) of every SSRN block, as build_tables lays them out (api_params.cu)."""
    c = hp.c
    t = [("SSRN/C_1", "C", hp.n_mels, c, 1, 1), ("SSRN/HC_2", "HC", c, c, 3, 1), ("SSRN/HC_3", "HC", c, c, 3, 1),
         ("SSRN/D_4", "D", c, c, 3, 1), ("SSRN/HC_5", "HC", c, c, 3, 2), ("SSRN/HC_6", "HC", c, c, 3, 2),
         ("SSRN/D_7", "D", c, c, 3, 2), ("SSRN/HC_8", "HC", c, c, 3, 4), ("SSRN/HC_9", "HC", c, c, 3, 4),
         ("SSRN/C_10", "C", c, 2 * c, 1, 4), ("SSRN/HC_11", "HC", 2 * c, 2 * c, 3, 4), ("SSRN/HC_12", "HC", 2 * c, 2 * c, 3, 4),
         ("SSRN/C_13", "C", 2 * c, F, 1, 4), ("SSRN/C_14", "C", F, F, 1, 4), ("SSRN/C_15", "C", F, F, 1, 4),
         ("SSRN/C_16", "C", F, F, 1, 4)]
    d2 = 2 * hp.d
    te = [("Text2Mel/TextEnc/C_2", "C", hp.e, d2, 1, None), ("Text2Mel/TextEnc/C_3", "C", d2, d2, 1, None)]
    te += [("Text2Mel/TextEnc/HC_%d" % i, "HC", d2, d2, 3 if i < 14 else 1, None) for i in range(4, 16)]
    return t + te


def tile_cols(kind, cout):
    """Accumulator columns over the cluster (pack_tc in api_params.cu)."""
    if kind == "C":
        maxbn = 64 if (cout <= 256 and cout % 64 == 0) else 256
        n = 1
        while rup((cout + n - 1) // n, 16) > maxbn:
            n *= 2
        return n * rup((cout + n - 1) // n, 16)
    return 2 * cout


def flops(kind, cin, cout, taps, B, L):
    """(algorithmic, executed on the tensor pipe) floating-point operations of one launch at input length L."""
    rows = B * rup(L, 128)
    if kind == "D":
        alg = 2.0 * B * L * 3 * cin * cout                 # three kernel taps, stride 2
        exe = 3 * 2.0 * rows * 2 * rup(cin, 64) * 2 * cout   # two k-taps over both output halves (tap 1's second half is zero)
    else:
        alg = 2.0 * B * L * taps * cin * (2 * cout if kind == "HC" else cout)
        exe = 3 * 2.0 * rows * taps * rup(cin, 64) * tile_cols(kind, cout)
    return alg, exe


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                                   # the numbers are still printed, marked as of an unknown card
        return "unknown (%s)" % e


def cycle_split(eng, scope, B, L):
    """CTA 0's cycle split of one tc_debug launch: the library prints it to stderr, which is captured here."""
    eng.set_option("tc_debug", 1)
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+") as f:
        os.dup2(f.fileno(), 2)
        try:
            eng.bench_block(scope, B, L, iters=1, warmup=0)
        finally:
            os.dup2(saved, 2)
            os.close(saved)
            eng.set_option("tc_debug", 0)
        f.seek(0)
        lines = [ln.strip() for ln in f if "cycles:" in ln or "mode=" in ln]
    return lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--frames", type=int, default=hp.max_T)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--cycles", default="SSRN/HC_11,SSRN/HC_8,SSRN/C_14")
    ap.add_argument("--option", action="append", default=[], help="engine option name=value, applied before timing")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    B, T = args.batch, args.frames
    F = 1 + hp.n_fft // 2

    eng = Engine(0)
    eng.load_params(init_params(0, "perturbed"))
    eng.set_tensor_path(1)
    for o in args.option:
        k, v = o.split("=")
        eng.set_option(k, int(v))
    print("card: %s   B=%d T=%d   options: %s" % (card(), B, T, args.option or "defaults"))
    rows = []
    tot_ms = tot_alg = tot_exe = 0.0
    print("%-24s %6s %8s %10s %8s %8s %8s" % ("scope", "L", "fused_ms", "other_ms", "alg_TF/s", "exe_TF/s", "share"))
    for scope, kind, cin, cout, taps, lf in block_table(F):
        L = hp.max_N if lf is None else T * lf
        kms = eng.bench_block(scope, B, L, iters=args.iters, warmup=2)
        fused = kms[1] if len(kms) > 1 else kms[0]
        alg, exe = flops(kind, cin, cout, taps, B, L)
        rows.append({"scope": scope, "L": L, "kernels_ms": kms, "fused_ms": fused, "alg_tflops": alg / fused / 1e9,
                     "exe_tflops": exe / fused / 1e9})
        if scope.startswith("SSRN"):
            tot_ms += fused; tot_alg += alg; tot_exe += exe
    for r in rows:
        share = r["fused_ms"] / tot_ms if r["scope"].startswith("SSRN") else float("nan")
        print("%-24s %6d %8.3f %10s %8.1f %8.1f %7.1f%%" % (r["scope"], r["L"], r["fused_ms"],
              ",".join("%.3f" % m for m in r["kernels_ms"] if m != r["fused_ms"]) or "-", r["alg_tflops"], r["exe_tflops"],
              100 * share))
    print("SSRN fused blocks: %.3f ms, %.1f TFLOP/s algorithmic, %.1f TFLOP/s executed" % (tot_ms, tot_alg / tot_ms / 1e9,
                                                                                           tot_exe / tot_ms / 1e9))

    Y = torch.from_numpy(np.random.default_rng(0).uniform(0, 1, (B, T, hp.n_mels)).astype(np.float32)).cuda()
    Z = torch.empty((B, T * hp.r, F), device="cuda")
    for _ in range(3):
        eng.ssrn(Y, want_logits=False, out=Z)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(args.iters):
        eng.ssrn(Y, want_logits=False, out=Z)
    b.record()
    torch.cuda.synchronize()
    ssrn_ms = a.elapsed_time(b) / args.iters
    print("Engine.ssrn B=%d T=%d: %.3f ms" % (B, T, ssrn_ms))

    cycles = {}
    for scope in [s for s in args.cycles.split(",") if s]:
        lf = next(x[5] for x in block_table(F) if x[0] == scope)
        cycles[scope] = cycle_split(eng, scope, B, hp.max_N if lf is None else T * lf)
        for ln in cycles[scope]:
            print("%-12s %s" % (scope, ln))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": card(), "B": B, "T": T, "options": args.option, "blocks": rows, "ssrn_ms": ssrn_ms,
                       "cycles": cycles}, f, indent=1)


if __name__ == "__main__":
    main()
