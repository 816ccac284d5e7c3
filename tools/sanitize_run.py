"""Small workload for compute-sanitizer (memcheck / racecheck / synccheck; SURVEY section 5, VERDICT r1 item 8): one
block of every wgmma block-kernel variant (two-stage and deeper rings, transposed conv, a narrow conv), the wgmma
attention, and a few frames of both decode loops with a window move.
   compute-sanitizer --tool memcheck python tools/sanitize_run.py [what ...]      what: blocks attention decode graph train overcap
"overcap": one Text2Mel step past (max_N, max_T) on a grown workspace per training kernel set (train_tc 7 and 0): the
guided-attention table is read only inside its (max_N, max_T) corner."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from dc_tts_b200.engine import Engine  # noqa: E402
from dc_tts_b200.hyperparams import Hyperparams as hp  # noqa: E402
from dc_tts_b200.params import init_params, synthetic_bucket, synthetic_text  # noqa: E402

what = set(sys.argv[1:]) or {"blocks", "attention", "decode", "graph"}
e = Engine(0)
e.load_params(init_params(0, "perturbed"))
rng = np.random.default_rng(0)
if "blocks" in what:
    x = rng.uniform(-1, 1, (3, 840, 1024)).astype(np.float32)          # 21 tiles x 8 CTAs: wider than the device
    e.hc("SSRN/HC_11", x, 1, False)
    e.set_option("tc_occ2", 0); e.hc("SSRN/HC_11", x[:1, :256], 1, False); e.set_option("tc_occ2", 1)
    e.conv1d_transpose("SSRN/D_4", rng.uniform(-1, 1, (2, 210, 512)).astype(np.float32))
    e.conv1d("SSRN/C_13", rng.uniform(-1, 1, (1, 70, 1024)).astype(np.float32), 1025, 1, False, 0)
    e.hc("Text2Mel/AudioEnc/HC_7", rng.uniform(-1, 1, (2, 210, 256)).astype(np.float32), 27, True)
    torch.cuda.synchronize(); print("blocks ok", flush=True)
if "attention" in what:
    Q = rng.uniform(-1, 1, (2, hp.max_T, hp.d)).astype(np.float32)
    K = rng.uniform(-1, 1, (2, hp.max_N, hp.d)).astype(np.float32)
    V = rng.uniform(-1, 1, (2, hp.max_N, hp.d)).astype(np.float32)
    e.attention(Q, K, V, monotonic=True, prev_max_attentions=np.array([3, 170], np.int32))
    e.attention(Q, K, V)
    torch.cuda.synchronize(); print("attention ok", flush=True)
L = synthetic_text(3, 60, seed=0)
if "decode" in what:
    e.set_option("decode_mode", 1)
    Y, P, _, _ = e.text2mel_generate(L, steps=8)
    torch.cuda.synchronize(); print("cluster decode ok; windows", P[:, :8].tolist(), e.decode_stats(), flush=True)
if "graph" in what:
    e.set_option("decode_mode", 0)
    Y, P, _, _ = e.text2mel_generate(L, steps=4)
    torch.cuda.synchronize(); print("graph decode ok", flush=True)
    e.set_option("decode_mode", 1)
if "train" in what:
    # the wgmma training GEMMs (kernels_gemm_tc.cu): one Text2Mel step at B = 2 (forward, data gradient, weight gradient)
    t = Engine(0)
    t.load_params(init_params(0))
    t.train_init(2)
    mels = rng.uniform(0, 1, (2, hp.max_T, hp.n_mels)).astype(np.float32)
    out = t.train_step(synthetic_text(2, 60, seed=1), mels, global_step=7, seed=1)
    torch.cuda.synchronize(); print("train step ok", out, flush=True)
if "overcap" in what:
    for tc in (7, 0):
        t = Engine(0)
        t.load_params(init_params(0))
        t.set_option("train_tc", tc)
        t.train_init(2)
        t.train_reserve(256, 256)
        Lb, mels = synthetic_bucket(2, 200, 240, seed=1)
        out = t.train_step(Lb, mels, global_step=7, seed=1)
        torch.cuda.synchronize(); print("over-capacity train step ok, train_tc", tc, out, flush=True)
        t.close()
