"""ORACLE (test infrastructure) -- the Text2Mel training step of oracle/ref_train.py at a length-bucketed batch's own shape
(reference data_load.py:122-129, dynamic_pad=True).  Everything is oracle/ref_train.py's except the guided-attention loss:
train.py:91-95 pads the alignments with -1 to (max_N, max_T) and masks the padding out, so with L (B, N_b) and mels
(B, T_b, n_mels) the loss is sum_{n < N_b, t < T_b} |A[n, t] gts[n, t]| / (B N_b T_b), gts being utils.guided_attention()
on the (max_N, max_T) grid, not recomputed at the bucket shape.  At N_b = max_N, T_b = max_T this is ref_train.forward
exactly.  Pinned by the reference's own training graphs at bucket shapes (refshim_train_bucket.npz,
tests/golden/make_golden_refchecks_bucket.py)."""
import numpy as np
import torch

from dc_tts_b200 import arch
from oracle import ref_torch as rt
from oracle import ref_train as rtr


def forward(P, L, mels, seed=0, rate=None):
    """train.py:48-68 + :83-99 in training mode at the batch's own (N_b, T_b).  P: name -> tensor."""
    from dc_tts_b200.hyperparams import Hyperparams as hp
    rate = hp.dropout_rate if rate is None else rate
    mels = torch.as_tensor(mels, dtype=torch.float32)
    S = torch.cat((torch.zeros_like(mels[:, :1, :]), mels[:, :-1, :]), 1)
    c = [0]
    x = rt.embed(P, torch.as_tensor(L), "Text2Mel/TextEnc/embed_1").to(torch.float32)
    x = rtr._chain(P, x, "Text2Mel/TextEnc", arch.textenc_layers(), c, seed, rate)
    K, V = torch.chunk(x, 2, dim=-1)
    Q = rtr._chain(P, S, "Text2Mel/AudioEnc", arch.audioenc_layers(), c, seed, rate)
    R, alignments, _ = rt.Attention(Q, K, V, False, None)
    logits = rtr._chain(P, R, "Text2Mel/AudioDec", arch.audiodec_layers(), c, seed, rate)
    Y = torch.sigmoid(logits)
    loss_mels = (Y - mels).abs().mean()
    loss_bd1 = torch.nn.functional.binary_cross_entropy_with_logits(logits, mels)
    A = alignments[:, :hp.max_N, :hp.max_T]                                      # (B, N_b, T_b): what the mask keeps
    gts = torch.from_numpy(rtr.guided_attention())[:A.shape[1], :A.shape[2]]
    loss_att = (A * gts).abs().sum() / float(A.numel())
    return dict(loss=loss_mels + loss_bd1 + loss_att, loss_mels=loss_mels, loss_bd1=loss_bd1, loss_att=loss_att,
                Y=Y, logits=logits, alignments=alignments, Q=Q, K=K, V=V, R=R)


def train_step(P, L, mels, state=None, global_step=0, seed=0, rate=None, lr=None, beta1=0.9, beta2=0.999, eps=1e-8):
    """One Text2Mel optimiser step (train.py:122-132) at the batch's own shape; same returns as ref_train.train_step."""
    names = rtr.text2mel_names()
    T = {n: torch.tensor(np.asarray(P[n], np.float32), requires_grad=True) for n in names}
    out = forward(T, L, mels, seed, rate)
    out["loss"].backward()
    newP, newstate, grads, lr_now = rtr._adam(P, names, T, state, global_step, lr, beta1, beta2, eps)
    info = {k: float(out[k].detach()) for k in ("loss", "loss_mels", "loss_bd1", "loss_att")}
    info["grads"] = grads
    info["lr"] = lr_now
    return newP, newstate, info
