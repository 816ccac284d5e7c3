"""Probe of the wgmma block kernel: one block on both paths, error printed (debugging aid;
run with DCTTS_TC_DEBUG=1 for per-CTA progress markers)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from dc_tts_b200 import arch  # noqa: E402
from dc_tts_b200.engine import Engine  # noqa: E402
from dc_tts_b200.params import init_params  # noqa: E402

cases = sys.argv[1:] or ["Text2Mel/AudioDec/C_11:1:128", "Text2Mel/AudioEnc/C_1:1:128", "Text2Mel/AudioEnc/HC_4:1:128"]
P = init_params(0, "perturbed")
need = set(c.split(":")[0] for c in cases)
e = Engine(0)
e.load_params(P)
for case in cases:
    scope, B, L = case.split(":"); B, L = int(B), int(L)
    net, name = scope.rsplit("/", 1)
    l = [x for x in arch.NETWORKS[net]() if x.scope == name][0]
    x = np.random.default_rng(0).uniform(-1, 1, (B, L, l.cin)).astype(np.float32)
    outs = []
    for mode in (0, 1):
        e.set_tensor_path(mode)
        if l.kind == "C":
            o = e.conv1d(scope, x, l.cout, l.rate, l.pad == "CAUSAL", 1 if l.act == "relu" else 0)
        elif l.kind == "HC":
            o = e.hc(scope, x, l.rate, l.pad == "CAUSAL")
        else:
            o = e.conv1d_transpose(scope, x)
        torch.cuda.synchronize()
        outs.append(o.cpu().numpy())
    d = np.abs(outs[0] - outs[1])
    print("%s B=%d L=%d: max|simt-tc| = %.3e  (mean %.3e, ref max %.3f)" % (scope, B, L, d.max(), d.mean(), np.abs(outs[0]).max()), flush=True)
    if d.max() > 1e-3:
        bad = np.argwhere(d > 1e-3)
        print("   first bad idx", bad[:5].tolist(), "rows bad:", len(set(bad[:, 1].tolist())), "cols bad:", len(set(bad[:, 2].tolist())))
