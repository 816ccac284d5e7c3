"""numpy restatement of the long-form join (Engine.join_rows, csrc/kernels_longform.cu), which the GPU tests hold the
kernel to bit for bit."""
import numpy as np


def join_rows_reference(Y, lengths, piece_text, piece_pause, K, silence=1e-8, T_out=None):
    """numpy restatement of Engine.join_rows: (K, T_out, C) float32 and the (K,) int32 rows of each text."""
    Y = np.asarray(Y, np.float32)
    P, T, C = Y.shape
    n = np.clip(np.asarray(lengths).reshape(-1), 0, T)
    text, pause = np.asarray(piece_text).reshape(-1), np.asarray(piece_pause).reshape(-1)
    seqs = [[] for _ in range(K)]
    for p in range(P):
        seqs[text[p]].append(Y[p, :n[p]])
        seqs[text[p]].append(np.full((pause[p], C), silence, np.float32))
    joined = [np.concatenate(s) for s in seqs]
    out_len = np.array([len(j) for j in joined], np.int32)
    T_out = int(out_len.max()) if T_out is None else int(T_out)
    out = np.zeros((K, T_out, C), np.float32)
    for k, j in enumerate(joined):
        out[k, :len(j)] = j
    return out, out_len
