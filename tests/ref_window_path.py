"""CPU reference of the decode along a window path: the reference's synthesize.py:45-54 loop with
prev_max_attentions = path[:, j] fed at step j instead of the previous step's argmax, on the oracle's float32
synthesize graph (full recompute per step)."""
import numpy as np
import torch

from dc_tts_b200.hyperparams import Hyperparams as hp
from oracle import ref_torch as rt


@torch.no_grad()
def forced_path(P, L, path):
    """path (B, steps) -> dict(Y (B, max_T, n_mels) with rows >= steps 0, argmax (B, steps) of every step inside its
    forced window, margin (B, steps): the top-2 probability gap of that row, to skip near-ties)."""
    L = np.asarray(L)
    path = np.asarray(path, np.int64)
    B, steps = path.shape
    Y = torch.zeros((B, hp.max_T, hp.n_mels), dtype=torch.float32)
    KV = None
    amax, margin = [], []
    for j in range(steps):
        out = rt.text2mel_forward(P, L, Y, torch.as_tensor(path[:, j]), KV)
        if KV is None:
            KV = (out["K"], out["V"])
        a = out["alignments"][:, :, j]
        top2 = torch.topk(a, 2, dim=-1).values
        margin.append((top2[:, 0] - top2[:, 1]).numpy())
        amax.append(out["max_attentions"][:, j].numpy())
        Y[:, j] = out["Y"][:, j]
    return dict(Y=Y.numpy(), argmax=np.stack(amax, 1), margin=np.stack(margin, 1))
