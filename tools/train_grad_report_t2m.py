"""Per-tensor gradient deviation of the CUDA Text2Mel training step from the autograd oracle (max |g - g_ref| / max |g_ref|),
wgmma GEMMs (train_tc 1) next to the fp32 CUDA-core kernels (train_tc 0)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from dc_tts_b200.engine import Engine
from dc_tts_b200.hyperparams import Hyperparams as hp
from dc_tts_b200.params import init_params, synthetic_text
from oracle import ref_train as rtr

P = init_params(0, "perturbed")
for (B, rate, seed) in [(2, 0.05, 11)]:
    L = synthetic_text(B, 50, seed=7)
    mels = np.random.default_rng(3).uniform(0, 1, (B, hp.max_T, hp.n_mels)).astype(np.float32)
    _, _, info = rtr.train_step(P, L, mels, global_step=7, seed=seed, rate=rate)
    got = {}
    for tc in (1,):
        eng = Engine(0)
        eng.load_params(P)
        eng.set_option("train_tc", tc)
        eng.train_init(B, rate)
        out = eng.train_step(L, mels, global_step=7, seed=seed, apply=False)
        errs = []
        for n, ref in info["grads"].items():
            g = eng.train_tensor(n, "grad")
            got[(tc, n)] = g
            errs.append((float(np.abs(np.clip(g, -1, 1) - ref).max() / max(np.abs(ref).max(), 1e-8)), n))
        order = [n for n in info["grads"] if n.endswith("conv1d/kernel")]
        print("   kernels in graph order:", " ".join("%s=%.0e" % (n.replace("Text2Mel/", "").replace("/conv1d/kernel", ""), e) for e, n in errs if n in order), flush=True)
        errs.sort(reverse=True)
        print("T2M B=%d rate=%.2f tc=%d: loss %.7f vs %.7f; worst:" % (B, rate, tc, out["loss"], info["loss"]),
              ["%s %.1e" % (n.replace("Text2Mel/", ""), e) for e, n in errs[:8]], "median %.1e" % np.median([e for e, _ in errs]), flush=True)
        eng.close()

