"""Float64 references of the autoregressive decode's blocks (csrc/kernels_decode.cu, and the graph-per-frame step of
csrc/api_synth.cu), for tests/test_gpu_decode_blocks.py.

Each function computes ONE block of one utterance from that block's float32 input rows as the decode left them, so that a
block is held to its own rounding instead of the accumulated error of the blocks before it.  Next to each value it returns
the error scale S: the first-order float32 error of the block, in the value's units, with the rounding unit left out.  The
GEMV is bounded by sum |x w| + |b|; LayerNorm carries that through its row gain |gamma| rstd, with the (1 + kappa)
sensitivity of recomputed statistics (tests/ref_train_kernels.py); the gate, the highway mix, the softmax and the sigmoid
carry it through their derivatives.  A kernel is within its noise where |got - ref| <= tau S, with tau a small multiple of
2^-24 fitted on the GPU (DESIGN.md, "The decode one block at a time").  tests/test_decode_blocks_reference.py pins these
functions against oracle/ref_numpy.py in float64.
"""
import numpy as np

LN_EPS = 1e-12
# err / S allowed, 3x or more above the worst measured on an H100 (DESIGN.md, "The decode one block at a time"): rows of the
# float32 paths (the one-row pass, the graph-per-frame decode's GEMV and LayerNorm kernels, the SIMT attention); rows of the
# persistent decode's split-fp16 receptive-field pre-pass, whose dropped lo*lo product stays below the float32 GEMV's own
# rounding at these S; rows of the graph-per-frame decode's 128-row split-fp16 tiles (conv_ln_tc_kernel), which reach the
# scheme's usual 1e-6; the full-sequence attention on the tensor cores, whose scores and probabilities are split-fp16 operands
TAU_FP32 = 4e-7
TAU_SPLIT = 4e-7
TAU_TILES = 5e-6
TAU_ATTN_TC = 1e-5


def _f(a):
    return np.asarray(a, np.float64)


def block_params(P, net, layer):
    """The float64 variables of block `layer` (arch.Layer) of `net` ("Text2Mel/AudioEnc" or "Text2Mel/AudioDec")."""
    s = "%s/%s" % (net, layer.scope)
    out = {"W": _f(P[s + "/conv1d/kernel"]), "b": _f(P[s + "/conv1d/bias"])}
    if layer.kind == "HC":
        out.update(g1=_f(P[s + "/H1/gamma"]), b1=_f(P[s + "/H1/beta"]), g2=_f(P[s + "/H2/gamma"]), b2=_f(P[s + "/H2/beta"]))
    else:
        out.update(g1=_f(P[s + "/normalize/gamma"]), b1=_f(P[s + "/normalize/beta"]))
    return out


def causal_conv(x, W, b, rate, rows, xs=None):
    """Output rows `rows` (indices into x's time axis) of the causal dilated conv y[t] = b + sum_j W[j]^T x[t - (k-1-j) rate],
    zero rows before t = 0.  x (T, cin) float32 rows as read; xs (T, cin) an error scale of x itself, or None (x exact).
    Returns (y, S) (n, cout): S = sum (|x| + xs) |w| + |b|."""
    x = _f(x)
    rows = np.asarray(rows)
    k = W.shape[0]
    taps = []
    for j in range(k):
        t = rows - (k - 1 - j) * rate
        taps.append(np.where((t >= 0)[:, None], x[np.clip(t, 0, None)], 0.0))
    X = np.concatenate(taps, 1)
    Wf = W.reshape(-1, W.shape[2])
    y = X @ Wf + b
    A = np.abs(X)
    if xs is not None:
        xs = _f(xs)
        A = A + np.concatenate([np.where((rows - (k - 1 - j) * rate >= 0)[:, None],
                                         xs[np.clip(rows - (k - 1 - j) * rate, 0, None)], 0.0) for j in range(k)], 1)
    return y, A @ np.abs(Wf) + np.abs(b)


def layer_norm(y, Sy, gamma, beta):
    """LayerNorm (biased variance, eps 1e-12) of rows y with error scale Sy: z = (y - mean) rstd gamma + beta.  The scale of z
    is (1 + kappa) |gamma| (rstd (Sy + mean Sy + |yhat| max Sy) + |yhat|) + |beta|, kappa = (|mean| + max |y - mean|) rstd
    the statistics' sensitivity.  A row of equal values is taken as exact (the tests make such rows with a zero kernel, so
    the conv is exactly its bias and the float32 statistics are exact): its scale is |beta|.
    Returns (z, S, yhat)."""
    mean = y.mean(1, keepdims=True)
    dev = y - mean
    rstd = 1.0 / np.sqrt((dev * dev).mean(1, keepdims=True) + LN_EPS)
    yh = dev * rstd
    spread = np.abs(dev).max(1, keepdims=True)
    kappa = np.where(spread == 0, 0.0, (np.abs(mean) + spread) * rstd)
    prop = rstd * (Sy + Sy.mean(1, keepdims=True) + np.abs(yh) * Sy.max(1, keepdims=True))
    prop = np.where(spread == 0, 0.0, prop)                  # an exact constant row (a zero kernel): z = beta exactly
    S = (1 + kappa) * np.abs(gamma) * (prop + np.abs(yh)) + np.abs(beta)
    return yh * gamma + beta, S, yh


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def conv_epilogue(p, layer, y, Sy):
    """LayerNorm (+ ReLU) of conv rows y with error scale Sy (modules.py:91-141).  Returns (out, S)."""
    z, S, _ = layer_norm(y, Sy, p["g1"], p["b1"])
    if layer.act == "relu":
        z = np.maximum(z, 0.0)
    return z, S


def hc_epilogue(p, y, Sy, xr, xsr=0.0):
    """The highway mix of conv rows y (2C wide) with error scale Sy and the residual rows xr (error scale xsr)
    (modules.py:143-197): h1 = sigmoid(LN(y_gate)), h2 = LN(y_info), out = h1 h2 + (1 - h1) x.  The gate's error passes
    through h1 (1 - h1), and the float32 gate (expf or __expf, 2 + 1.2 |z| ulp) adds (3 + |z1|) h1 (1 - h1) of rounding.
    Returns (out, S)."""
    C = y.shape[1] // 2
    z1, S1, _ = layer_norm(y[:, :C], Sy[:, :C], p["g1"], p["b1"])
    z2, S2, _ = layer_norm(y[:, C:], Sy[:, C:], p["g2"], p["b2"])
    h1 = sigmoid(z1)
    dg = h1 * (1 - h1)
    out = h1 * z2 + (1 - h1) * xr
    S = dg * (S1 + 3 + np.abs(z1)) * (np.abs(z2) + np.abs(xr)) + h1 * (S2 + np.abs(z2)) + (1 + h1) * np.abs(xr) + (1 - h1) * xsr
    return out, S


def conv_block(p, layer, x, rows, xs=None):
    """conv1d + LayerNorm (+ ReLU) of block `layer` on the rows `rows` (modules.py:91-141).  Returns (out, S)."""
    y, Sy = causal_conv(x, p["W"], p["b"], layer.rate, rows, xs)
    return conv_epilogue(p, layer, y, Sy)


def hc_block(p, layer, x, rows, xs=None):
    """Highway conv of block `layer` on the rows `rows` (modules.py:143-197, hc_epilogue).  Returns (out, S)."""
    y, Sy = causal_conv(x, p["W"], p["b"], layer.rate, rows, xs)
    xr = _f(x)[np.asarray(rows)]
    xsr = 0.0 if xs is None else _f(xs)[np.asarray(rows)]
    return hc_epilogue(p, y, Sy, xr, xsr)


def block(p, layer, x, rows, xs=None):
    return hc_block(p, layer, x, rows, xs) if layer.kind == "HC" else conv_block(p, layer, x, rows, xs)


def shifted_feed(Y):
    """AudioEnc C_1's input: row j reads Y[j - 1], zeros at j = 0 (train.py:51)."""
    Y = _f(Y)
    return np.concatenate([np.zeros_like(Y[:1]), Y[:-1]], 0)


def window_keys(p, N, win):
    """The live keys of a window at p: [clamp(p, 0, N - 1), min(that + win, N)) (networks.py:146-150)."""
    lo = min(max(int(p), 0), N - 1)
    return lo, min(lo + win, N)


def attention_rows(Q, KV, windows, win):
    """One query row per window: R = [sum_n a_n V_n | Q] over the window's live keys, a = softmax(Q K^T / sqrt(d)).  Q (n, d)
    float32 rows as read, KV (N, 2d), windows (n,) ints.  Returns dict(R (n, 2d), S (n, 2d), A (n, N) the probabilities (0
    outside the window) and SA (n, N) their error scale, argmax (n,) the first index among equal maxima, margin (n,) top-1 minus top-2 probability (inf with one live key), Sp (n,) the error scale of the
    probabilities of the two leading keys, summed)."""
    Q, KV = _f(Q), _f(KV)
    n, d = Q.shape
    N = KV.shape[0]
    R, S = np.zeros((n, 2 * d)), np.zeros((n, 2 * d))
    A, SA = np.zeros((n, N)), np.zeros((n, N))
    amax, margin, Sp = np.zeros(n, np.int64), np.full(n, np.inf), np.zeros(n)
    for i in range(n):
        lo, hi = window_keys(windows[i], N, win)
        K, V = KV[lo:hi, :d], KV[lo:hi, d:]
        s = K @ Q[i] / np.sqrt(d)
        ss = np.abs(K) @ np.abs(Q[i]) / np.sqrt(d)
        e = np.exp(s - s.max())
        a = e / e.sum()
        sa = a * (ss + (a * ss).sum() + 1)                   # scores' rounding through the softmax, and its own
        A[i, lo:hi], SA[i, lo:hi] = a, sa
        R[i, :d] = a @ V
        R[i, d:] = Q[i]
        S[i, :d] = (a + sa) @ np.abs(V)
        S[i, d:] = np.abs(Q[i])
        amax[i] = lo + int(np.argmax(a))
        if hi - lo > 1:
            top = np.argsort(-a, kind="stable")[:2]
            margin[i] = a[top[0]] - a[top[1]]
            Sp[i] = sa[top[0]] + sa[top[1]]
    return dict(R=R, S=S, A=A, SA=SA, argmax=amax, margin=margin, Sp=Sp)


def mel_sigmoid(logits):
    """Y = sigmoid(logits) (networks.py:210) from the decode's float32 logits; S covers the fast sigmoid's (2 + 1.2 |x|) ulp
    exponential and its reciprocal.  Returns (Y, S)."""
    x = _f(logits)
    y = sigmoid(x)
    return y, y * (3 + (1 - y) * (3 + np.abs(x)))


def float32_block(p, layer, x, rows, shifts=None):
    """The same block restated in float32 (numpy, the kernels' operation order aside): the bound tests' stand-in for a kernel.
    shifts: tap j reads x[t + shifts[j]], zero outside x's rows; default the causal taps -(k - 1 - j) rate."""
    f = np.float32
    x = np.asarray(x, f)
    rows = np.asarray(rows)
    k = p["W"].shape[0]
    if shifts is None:
        shifts = [-(k - 1 - j) * layer.rate for j in range(k)]
    y = np.zeros((len(rows), p["W"].shape[2]), f) + p["b"].astype(f)
    for j in range(k):
        t = rows + shifts[j]
        ok = (t >= 0) & (t < len(x))
        y += np.where(ok[:, None], x[np.clip(t, 0, len(x) - 1)], f(0)) @ p["W"][j].astype(f)

    def ln(v, g, b):
        m = v.mean(1, keepdims=True, dtype=f)
        dv = v - m
        return dv * (f(1) / np.sqrt((dv * dv).mean(1, keepdims=True, dtype=f) + f(LN_EPS))) * g.astype(f) + b.astype(f)
    if layer.kind == "HC":
        C = y.shape[1] // 2
        h1 = f(1) / (f(1) + np.exp(-ln(y[:, :C], p["g1"], p["b1"])))
        return h1 * ln(y[:, C:], p["g2"], p["b2"]) + (f(1) - h1) * x[rows]
    z = ln(y, p["g1"], p["b1"])
    return np.maximum(z, f(0)) if layer.act == "relu" else z


def audiodec_rows(layers, T):
    """Rows of each AudioDec block's output the decode recomputes per frame (api_synth.cu audiodec_rows): the receptive field
    of the last block's one row, clamped to T."""
    rows, need = [1] * len(layers), 1
    for i in range(len(layers) - 1, -1, -1):
        rows[i] = min(need, T)
        need += (layers[i].size - 1) * layers[i].rate
    return rows
