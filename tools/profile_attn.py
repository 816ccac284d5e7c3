"""Times the full-sequence attention (dense and monotonic) on the tensor-core path at a chosen (B, T, N).

    python tools/profile_attn.py --B 32 --T 210 --N 300 [--dump out.npz]

Prints the card's name and power limit with the per-call times (CUDA events over --iters calls, after warm-up).  Each
call is three kernels: Q planes, K / V^T planes, wgmma attention.  --dump writes R, alignments and the argmax of both
modes on the seeded inputs, for comparing two builds bit for bit."""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from dc_tts_b200.engine import Engine  # noqa: E402
from dc_tts_b200.params import init_params  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
        return out or torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ", power limit unknown"


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--B", type=int, default=32)
    ap.add_argument("--T", type=int, default=210)
    ap.add_argument("--N", type=int, default=180)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--dump", default=None, help="write R, alignments and argmax of both modes to this .npz")
    args = ap.parse_args()
    B, T, N = args.B, args.T, args.N

    e = Engine(0)
    e.load_params(init_params(0, "perturbed"))
    e.set_tensor_path(1)
    rng = np.random.default_rng(0)
    Q = torch.from_numpy(rng.uniform(-1, 1, (B, T, 256)).astype(np.float32)).cuda()
    K = torch.from_numpy(rng.uniform(-1, 1, (B, N, 256)).astype(np.float32)).cuda()
    V = torch.from_numpy(rng.uniform(-1, 1, (B, N, 256)).astype(np.float32)).cuda()
    pma = torch.from_numpy(rng.integers(0, N, B).astype(np.int32)).cuda()
    print("card: %s" % card())
    out = {}
    for name, mono in (("dense", False), ("monotonic", True)):
        for _ in range(3):
            e.attention(Q, K, V, mono, pma)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.iters):
            e.attention(Q, K, V, mono, pma)
        b.record()
        torch.cuda.synchronize()
        print("%-9s attention B=%d T=%d N=%d: %.1f us per call" % (name, B, T, N, a.elapsed_time(b) * 1e3 / args.iters))
        R, A, M = e.attention(Q, K, V, mono, pma)
        out.update({name + "_R": R.cpu().numpy(), name + "_A": A.cpu().numpy(), name + "_M": M.cpu().numpy()})
    if args.dump:
        np.savez(args.dump, pma=pma.cpu().numpy(), **out)


if __name__ == "__main__":
    main()
