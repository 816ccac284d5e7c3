"""Runs the full-sequence attention (dense, then monotonic) a few times -- target of ncu."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from dc_tts_b200.engine import Engine  # noqa: E402
from dc_tts_b200.params import init_params  # noqa: E402

B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
e = Engine(0)
e.load_params(init_params(0, "perturbed"))
rng = np.random.default_rng(0)
Q = torch.from_numpy(rng.uniform(-1, 1, (B, 210, 256)).astype(np.float32)).cuda()
K = torch.from_numpy(rng.uniform(-1, 1, (B, 180, 256)).astype(np.float32)).cuda()
V = torch.from_numpy(rng.uniform(-1, 1, (B, 180, 256)).astype(np.float32)).cuda()
pma = torch.zeros(B, dtype=torch.int32).cuda()
for it in range(3):
    e.attention(Q, K, V, False, None)
    e.attention(Q, K, V, True, pma)
torch.cuda.synchronize()
a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
a.record()
for it in range(10):
    e.attention(Q, K, V, False, None)
b.record(); torch.cuda.synchronize()
print("dense attention B=%d: %.1f us per call (3 kernels: planes, K/V^T planes, wgmma attention)" % (B, a.elapsed_time(b) * 100))
