"""Float64 references of the full-sequence networks' blocks (conv_ln_tc_kernel in csrc/kernels_tc.cu; the fp32 conv-GEMMs
with ln_rows_kernel / ln_row_cta_kernel in csrc/kernels_simt.cu; the dense attention on both kernel sets), for
tests/test_gpu_forward_blocks.py.

Each function computes ONE block of one utterance from that block's float32 input rows as the chain left them
(Engine.chain_history), so that a block is held to its own rounding.  It builds on tests/ref_decode_blocks.py: the same
LayerNorm error scale, highway gate algebra, sigmoid and attention, generalised here to the SAME and causal convs at any
dilation (per-tap shifts, as api_synth.cu run_block / run_block_tc compute them), the stride-2 transposed conv, ragged
batches (utterance b's block i sees only its own live rows) and the dense attention.  S is the first-order float32 error
scale with the rounding unit left out; a kernel is within its noise where |got - ref| <= tau S
(DESIGN.md, "The full-sequence networks one block at a time").  tests/test_forward_blocks_reference.py pins these functions
against oracle/ref_numpy.py in float64.
"""
import numpy as np
import torch

from ref_decode_blocks import attention_rows, hc_epilogue, layer_norm, mel_sigmoid, sigmoid  # noqa: F401

# err / S allowed, 3-4x above the worst measured on an H100 (DESIGN.md, "The full-sequence networks one block at a time"):
# the fp32 conv-GEMMs with their LayerNorm kernels, and the wgmma block kernel on split-fp16 operands
TAU_FP32 = 2e-7
TAU_TC = 3e-7
TAU_ATTN_FP32 = 3e-7
TAU_ATTN_TC = 4e-6
# the alignments (attention probabilities), against their own scale SA
TAU_ATTN_FP32_A = 1e-7
TAU_ATTN_TC_A = 8e-7
# A block output kept as split-fp16 planes (the tensor path's hidden blocks) is hi + lo, and the lo plane cannot resolve
# less than the fp16 subnormal step: 2^-25 of absolute error, 1/2 in the units of S (the rounding unit 2^-24 left out).
# Without it every hidden output near zero would fail; values at that floor are the small-activation limitation DESIGN.md
# section 2 records (tests/test_gpu_input_range.py, xfail).
S_PLANES = 2.0 ** -25 / 2.0 ** -24


def _f(a):
    return np.asarray(a, np.float64)


def block_params(P, net, layer):
    """The float64 variables of block `layer` (arch.Layer) of `net` ("Text2Mel/TextEnc", "SSRN", ...).  W is (taps, cin,
    nconv) for every kind: the transposed conv's (1, 3, cout, cin) kernel is turned to (3, cin, cout)."""
    s = "%s/%s" % (net, layer.scope)
    if layer.kind == "D":
        return {"W": _f(P[s + "/conv2d_transpose/kernel"])[0].transpose(0, 2, 1), "b": _f(P[s + "/conv2d_transpose/bias"]),
                "g1": _f(P[s + "/normalize/gamma"]), "b1": _f(P[s + "/normalize/beta"])}
    out = {"W": _f(P[s + "/conv1d/kernel"]), "b": _f(P[s + "/conv1d/bias"])}
    if layer.kind == "HC":
        out.update(g1=_f(P[s + "/H1/gamma"]), b1=_f(P[s + "/H1/beta"]), g2=_f(P[s + "/H2/gamma"]), b2=_f(P[s + "/H2/beta"]))
    else:
        out.update(g1=_f(P[s + "/normalize/gamma"]), b1=_f(P[s + "/normalize/beta"]))
    return out


def tap_shifts(layer, extra_shift=0):
    """Tap j reads input row t + shifts[j] (api_synth.cu run_block / run_block_tc): left = (k - 1) rate for a causal block,
    half of it (rounded down) for SAME; extra_shift moves every tap (AudioEnc's first block in text2mel_forward: -1)."""
    tot = (layer.size - 1) * layer.rate
    left = tot if layer.pad == "CAUSAL" else tot // 2
    return [j * layer.rate - left + extra_shift for j in range(layer.size)]


def _gather(x, idx):
    """Rows idx of x (torch float64), zero where idx is outside [0, len(x))."""
    ok = (idx >= 0) & (idx < x.shape[0])
    g = x[torch.as_tensor(np.clip(idx, 0, max(x.shape[0] - 1, 0)))]
    return g * torch.as_tensor(ok, dtype=torch.float64)[:, None]


def conv_rows(W, b, x, rows, shifts):
    """y[t] = b + sum_j W[j]^T x[t + shifts[j]] on the rows `rows`, x zero outside its own rows (an utterance's live rows:
    the caller passes them alone).  Returns (y, Sy), Sy = sum |x| |w| + |b|, in float64 numpy."""
    xt = torch.as_tensor(_f(x))
    rows = np.asarray(rows)
    X = torch.cat([_gather(xt, rows + s) for s in shifts], 1)
    Wf = torch.as_tensor(W.reshape(-1, W.shape[2]))
    y = (X @ Wf).numpy() + b
    Sy = (X.abs() @ Wf.abs()).numpy() + np.abs(b)
    return y, Sy


def deconv_rows(W, b, x, rows):
    """The stride-2 transposed conv (api_synth.cu run_deconv, modules.py:232-239) on output rows `rows`:
    out[2t] = W0 x[t] + W2 x[t - 1], out[2t + 1] = W1 x[t], + b; x zero outside its rows.  Returns (y, Sy)."""
    xt = torch.as_tensor(_f(x))
    rows = np.asarray(rows)
    t, odd = rows // 2, (rows % 2).astype(bool)
    Wt = [torch.as_tensor(W[j]) for j in range(3)]
    x0, x1 = _gather(xt, t), _gather(xt, t - 1)
    ev = torch.cat([x0, x1], 1), torch.cat([Wt[0], Wt[2]], 0)
    od = x0, Wt[1]
    y, Sy = np.zeros((len(rows), W.shape[2])), np.zeros((len(rows), W.shape[2]))
    for m, (X, Wm) in ((~odd, ev), (odd, od)):
        if m.any():
            Xm = X[torch.as_tensor(m)]
            y[m] = (Xm @ Wm).numpy() + b
            Sy[m] = (Xm.abs() @ Wm.abs()).numpy() + np.abs(b)
    return y, Sy


def block_rows(p, layer, x, rows, extra_shift=0):
    """Block `layer` of ONE utterance on its output rows `rows`, from x (its input rows, the live ones only).
    Returns (out, S)."""
    if layer.kind == "D":
        y, Sy = deconv_rows(p["W"], p["b"], x, rows)
        z, S, _ = layer_norm(y, Sy, p["g1"], p["b1"])
        return z, S
    y, Sy = conv_rows(p["W"], p["b"], x, rows, tap_shifts(layer, extra_shift))
    if layer.kind == "HC":
        return hc_epilogue(p, y, Sy, _f(x)[np.asarray(rows)])
    z, S, _ = layer_norm(y, Sy, p["g1"], p["b1"])
    return (np.maximum(z, 0.0) if layer.act == "relu" else z), S


def live_rows(layers, n):
    """Ragged mode: the live input and output rows of every block for an utterance of n input rows, n 2^(transposed convs
    before the block) (api_synth.cu run_chain_full: the chain for that utterance alone at L = n)."""
    ins, outs = [], []
    for l in layers:
        ins.append(n)
        n *= 2 if l.kind == "D" else 1
        outs.append(n)
    return ins, outs


def dense_attention(Q, KV, window=None, win=None):
    """The dense attention (monotonic=False): attention_rows with the window [0, N) for every query row; or, given
    `window` (one prev_max_attentions value) and `win`, the monotonic window of text2mel_forward.  Returns the dict of
    attention_rows: R and S, the probabilities A (T, N), argmax, margin, Sp; and the probabilities' own scale SA, which adds
    to the scores' rounding the float32 exponential's (2 + 1.2 |s - max s| ulp, as the gate of hc_epilogue) and the
    normalising division."""
    N, d = KV.shape[0], Q.shape[1]
    if window is None:
        window, win = 0, N
    r = attention_rows(Q, KV, np.full(len(Q), window, np.int64), win)
    s = _f(Q) @ _f(KV)[:, :d].T / np.sqrt(d)
    live = r["A"] > 0
    top = np.where(live, s, -np.inf).max(1, keepdims=True)
    r["SA"] = r["SA"] + np.where(live, r["A"] * (3 + np.abs(s - top)), 0.0)
    return r


def split_f16(x):
    """The split-fp16 planes of float32 x (csrc/numerics.cuh): hi = fp16(x), lo = fp16(x - hi), both round to nearest even."""
    x = np.asarray(x, np.float32)
    hi = x.astype(np.float16)
    lo = (x - hi.astype(np.float32)).astype(np.float16)
    return hi, lo


def input_planes(x, lengths=None):
    """What the tensor path's first block reads for a network input x (B, L, C) float32 (kernels_tc.cu
    f32_to_planes_scaled_kernel): per utterance the power-of-two scale s that puts its abs-max m in [2^14, 2^15) (1 for an
    all-zero utterance), the split planes of x s, joined and times 1 / s (exact); rows past lengths[b] are 0."""
    x = np.asarray(x, np.float32)
    out = np.zeros_like(x)
    for b in range(x.shape[0]):
        n = x.shape[1] if lengths is None else int(lengths[b])
        live = x[b, :n]
        m = float(np.abs(live).max()) if live.size else 0.0
        s = np.float32(1.0) if m == 0 else np.float32(np.ldexp(1.0, min(15 - np.frexp(np.float32(m))[1], 100)))
        hi, lo = split_f16(live * s)
        out[b, :n] = (hi.astype(np.float32) + lo.astype(np.float32)) * (np.float32(1) / s)
    return out
