"""Float64 references of the training step's non-GEMM kernels (csrc/kernels_train.cu), for tests/test_gpu_train_kernels.py.

Each function takes the kernel's float32 inputs (torch tensors, any device) and computes in float64.  Next to each value it
returns the error scale S: the same computation on absolute values (a - b -> |a| + |b|, a b -> |a| |b|, sum -> sum of |.|),
so that a float32 kernel that rounds each operation is off by a small multiple of 2^-24 S.  The tests pin these functions
against torch.autograd in float64 on the CPU.
"""
import numpy as np
import torch

LN_EPS = 1e-12              # tf.contrib.layers.layer_norm's epsilon, the kernels' too


# --------------------------------------------------------------------------------------------- block backward
_M32 = 0xffffffff


def _mul32(x, c):
    """(x c) mod 2^32 for int64 x in [0, 2^32): the constant is split in 16-bit halves so that no product overflows."""
    lo, hi = c & 0xffff, c >> 16
    return (x * lo + (((x * hi) & 0xffff) << 16)) & _M32


def mix32_torch(idx, layer, seed):
    """oracle.ref_train.mix32 (the step's dropout hash) on an int64 tensor of element indices, on its device."""
    x = _mul32(idx & _M32, 0x9E3779B1)
    x = x ^ ((int(layer) * 0x85EBCA77 + int(seed)) & _M32)
    x = x ^ (x >> 16)
    x = _mul32(x, 0x85EBCA6B)
    x = x ^ (x >> 13)
    x = _mul32(x, 0xC2B2AE35)
    return x ^ (x >> 16)


def drop_multiplier(rows, C, layer, seed, rate, device=None):
    """(rows, C) float64 multiplier of the step's dropout mask at the dense element index row * C + c: 0 where dropped,
    1 / (1 - rate) in float32 where kept (the kernel's DropArgs: threshold rate * 2^32 and scale from the float32 rate)."""
    rate = np.float32(rate)
    if rate <= 0:
        return torch.ones(rows, C, dtype=torch.float64, device=device)
    thresh = int(min(float(rate) * 4294967296.0, 4294967295.0))
    keep = mix32_torch(torch.arange(rows * C, dtype=torch.int64, device=device), layer, seed) >= thresh
    scale = float(np.float32(1.0) / (np.float32(1.0) - rate))
    return keep.reshape(rows, C).double() * scale


def ln_forward(y):
    """y (rows, C) float64 -> (yhat, rstd (rows, 1), mean (rows, 1)); biased variance, eps 1e-12."""
    mean = y.mean(1, keepdim=True)
    d = y - mean
    rstd = 1.0 / torch.sqrt((d * d).mean(1, keepdim=True) + LN_EPS)
    return d * rstd, rstd, mean


def ln_sensitivity(y, yhat, mean, rstd):
    """Per row, kappa = (|mean| + max |y - mean|) rstd: the float32 statistics give y - mean to about 2^-24 (|mean| + |y -
    mean|), i.e. yhat to 2^-24 kappa, and rstd to about 2^-24 kappa relative.  A row of equal values has kappa 0: the
    tests use only 0 and 0.75 there, whose float32 sums are exact, so the kernel also gets y - mean = 0 and yhat = 0."""
    spread = (y - mean).abs().amax(1, keepdim=True)
    kappa = (mean.abs() + spread) * rstd
    return torch.where(spread == 0, torch.zeros_like(kappa), kappa)


def _ln_bwd(yhat, dz, gam, rstd):
    t = dz * gam
    return rstd * (t - t.mean(1, keepdim=True) - yhat * (t * yhat).mean(1, keepdim=True))


def _ln_bwd_abs(yhat, dz, gam, rstd):
    t = dz.abs() * gam.abs()
    return rstd * (t + t.mean(1, keepdim=True) + yhat.abs() * (t * yhat.abs()).mean(1, keepdim=True))


def block_bwd(mode, act, pre, gout, ln, keep, X=None):
    """The backward of out = keep * act(LN(pre)) (mode 0) or keep * (h1 h2 + (1 - h1) X) (mode 1, h1 = sigmoid(LN(pre[:, :C]; g1,
    b1)), h2 = LN(pre[:, C:]; g2, b2)) given gout = d loss / d out.  pre (rows, nconv), gout (rows, C), ln (4, C), keep (rows,
    C) float64 multiplier.  ReLU passes the gradient where z > 0.  Returns (ref, scale): dicts of dy (rows, nconv), gin (rows,
    C, mode 1), dg1, db1, dg2, db2 (C,), dbias (nconv,), kappa (rows, 1).  The scales of per-row outputs carry (1 + kappa)."""
    f = lambda t: t.double()                                  # noqa: E731
    C = ln.shape[1]
    g1, b1, g2, b2 = (f(ln[i]) for i in range(4))
    y1 = f(pre[:, :C])
    yh1, r1, m1 = ln_forward(y1)
    k = 1 + ln_sensitivity(y1, yh1, m1, r1)
    g = f(gout) * keep
    ref, sc = {}, {}
    if mode == 0:
        z = yh1 * g1 + b1
        if act == 1:
            g = torch.where(z > 0, g, torch.zeros_like(g))
        ga = g.abs()
        ref["dg1"], sc["dg1"] = (g * yh1).sum(0), (ga * yh1.abs() * k).sum(0)
        ref["db1"], sc["db1"] = g.sum(0), (ga * k).sum(0)
        dy = _ln_bwd(yh1, g, g1, r1)
        s_dy = _ln_bwd_abs(yh1, g, g1, r1) * k
        ref["dy"], sc["dy"] = dy, s_dy
        ref["dbias"], sc["dbias"] = dy.sum(0), s_dy.sum(0)
    else:
        y2 = f(pre[:, C:2 * C])
        yh2, r2, m2 = ln_forward(y2)
        k = torch.maximum(k, 1 + ln_sensitivity(y2, yh2, m2, r2))
        x = f(X)
        h1 = torch.sigmoid(yh1 * g1 + b1)
        h2 = yh2 * g2 + b2
        h2a = yh2.abs() * g2.abs() + b2.abs()
        d1, d2 = g * (h2 - x) * h1 * (1 - h1), g * h1
        s1 = g.abs() * (h2a + x.abs()) * h1 * (1 + h1)        # 1 - h1 in float32: absolute error 2^-24, not relative
        s2 = g.abs() * h1
        ref["gin"], sc["gin"] = g * (1 - h1), g.abs() * (1 + h1) * k
        ref["dg1"], sc["dg1"] = (d1 * yh1).sum(0), (s1 * yh1.abs() * k).sum(0)
        ref["db1"], sc["db1"] = d1.sum(0), (s1 * k).sum(0)
        ref["dg2"], sc["dg2"] = (d2 * yh2).sum(0), (s2 * yh2.abs() * k).sum(0)
        ref["db2"], sc["db2"] = d2.sum(0), (s2 * k).sum(0)
        dy = torch.cat([_ln_bwd(yh1, d1, g1, r1), _ln_bwd(yh2, d2, g2, r2)], 1)
        s_dy = torch.cat([_ln_bwd_abs(yh1, s1, g1, r1), _ln_bwd_abs(yh2, s2, g2, r2)], 1) * k
        ref["dy"], sc["dy"] = dy, s_dy
        ref["dbias"], sc["dbias"] = dy.sum(0), s_dy.sum(0)
    ref["kappa"] = k - 1
    return ref, sc


def block_forward(mode, act, pre, ln, keep, X=None):
    """The forward the backward above differentiates (float64, autograd-able): LN -> ReLU / highway -> dropout."""
    C = ln.shape[1]
    yh1 = torch.nn.functional.layer_norm(pre[:, :C], (C,), ln[0], ln[1], eps=LN_EPS)
    if mode == 0:
        out = torch.relu(yh1) if act == 1 else yh1
    else:
        h1 = torch.sigmoid(yh1)
        h2 = torch.nn.functional.layer_norm(pre[:, C:2 * C], (C,), ln[2], ln[3], eps=LN_EPS)
        out = h1 * h2 + (1 - h1) * X
    return out * keep


def block_forward_scale(mode, act, pre, ln, keep, X=None):
    """block_forward in float64 with its error scale S, built like block_bwd's: the same computation on absolute values, the
    LayerNorm terms carrying (1 + kappa) per row, and kappa absolute (the float32 mean is off by 2^-24 (|mean| + spread),
    which moves yhat by 2^-24 kappa however small yhat is: a near-constant row's middle values); the highway gate's error passes through h1 (1 - h1) with the float32
    sigmoid's own (3 + |z1|) ulp, as the synthesis blocks' (tests/ref_decode_blocks.py hc_epilogue).  The dropout multiplier
    scales both (a dropped element is exactly 0).  Returns (out, S), (rows, C) float64."""
    f = lambda t: t.double()                                  # noqa: E731
    C = ln.shape[1]
    g1, b1, g2, b2 = (f(ln[i]) for i in range(4))
    y1 = f(pre[:, :C])
    yh1, r1, m1 = ln_forward(y1)
    z1 = yh1 * g1 + b1
    k1 = ln_sensitivity(y1, yh1, m1, r1)
    s1 = ((1 + k1) * yh1.abs() + k1) * g1.abs() + b1.abs()
    if mode == 0:
        out, S = (torch.relu(z1) if act == 1 else z1), s1
    else:
        y2 = f(pre[:, C:2 * C])
        yh2, r2, m2 = ln_forward(y2)
        z2 = yh2 * g2 + b2
        k2 = ln_sensitivity(y2, yh2, m2, r2)
        s2 = ((1 + k2) * yh2.abs() + k2) * g2.abs() + b2.abs()
        x = f(X)
        h1 = torch.sigmoid(z1)
        out = h1 * z2 + (1 - h1) * x
        S = h1 * (1 - h1) * (s1 + 3 + z1.abs()) * (z2.abs() + x.abs()) + h1 * (s2 + z2.abs()) + (1 + h1) * x.abs()
    return out * keep, S * keep.abs()


# --------------------------------------------------------------------------------------------- attention backward
def attn_bwd(gR, Q, KV, align, gts, n_lim, t_lim):
    """The softmax attention backward of the step with the guided-attention term, from the GIVEN alignments (not a
    recomputed softmax).  gR (B,T,2d) = [dctx | dQ direct], Q (B,T,d), KV (B,N,2d) = [K | V], align (B,N,T), gts (>= n_lim,
    >= t_lim).  The guided term is att_scale sign(A g) g on the (n_lim, t_lim) corner, att_scale = 1 / (B n_lim t_lim).
    Returns (ref, scale) dicts of gQ (B,T,d), gKV (B,N,2d) and att (the corner's sum |A gts|)."""
    f = lambda t: t.double()                                  # noqa: E731
    B, N, T = align.shape
    d = Q.shape[2]
    dctx, dq = f(gR[..., :d]), f(gR[..., d:])
    Qd, K, V = f(Q), f(KV[..., :d]), f(KV[..., d:])
    A = f(align).transpose(1, 2)                                # (B, T, N)
    G = torch.zeros(T, N, dtype=torch.float64, device=A.device)
    G[:t_lim, :n_lim] = f(gts[:n_lim, :t_lim]).t()
    scale = 1.0 / (B * n_lim * t_lim)
    AG = A * G
    dA = dctx @ V.transpose(1, 2) + torch.sign(AG) * G * scale
    dA_abs = dctx.abs() @ V.abs().transpose(1, 2) + G.abs() * scale
    dot = (A * dA).sum(2, keepdim=True)
    dS = A * (dA - dot)
    dS_abs = A * (dA_abs + (A * dA_abs).sum(2, keepdim=True))
    rs = d ** -0.5
    ref = {"gQ": dq + (dS @ K) * rs,
           "gKV": torch.cat([(dS.transpose(1, 2) @ Qd) * rs, A.transpose(1, 2) @ dctx], 2),
           "att": AG.abs().sum()}
    sc = {"gQ": dq.abs() + (dS_abs @ K.abs()) * rs,
          "gKV": torch.cat([(dS_abs.transpose(1, 2) @ Qd.abs()) * rs, A.transpose(1, 2) @ dctx.abs()], 2),
          "att": AG.abs().sum()}
    return ref, sc


def attn_forward_loss(Q, K, V, gR, gts, n_lim, t_lim):
    """What attn_bwd differentiates, for autograd: S = Q K^T / sqrt(d), A = softmax over keys, R = [A V | Q];
    loss = sum(R gR) + sum over the corner |A gts| / (B n_lim t_lim).  Returns (loss, align (B,N,T))."""
    B, T, d = Q.shape
    A = torch.softmax(Q @ K.transpose(1, 2) / d ** 0.5, dim=2)     # (B, T, N)
    R = torch.cat([A @ V, Q], 2)
    att = (A[:, :t_lim, :n_lim] * gts[:n_lim, :t_lim].t()).abs().sum() / (B * n_lim * t_lim)
    return (R * gR).sum() + att, A.transpose(1, 2)


# --------------------------------------------------------------------------------------------- losses
def train_loss(logits, target):
    """L1 + sigmoid cross-entropy of the step (train.py:83-89): y = sigmoid(x), sums |y - t| and BCE, and the gradient of
    mean |y - t| + mean BCE w.r.t. x, (sign(y - t) y (1 - y) + y - t) / n.  The sign is taken of sigmoid(x) ROUNDED TO
    FLOAT32 minus t, as the float32 graph sees it: where t is the float32 sigmoid the L1 term has no slope (sign(0) = 0);
    elsewhere this is the sign of the exact difference.  Returns (ref, scale) dicts of dlogits, Y, l1, bce."""
    x, t = logits.double(), target.double()
    n = x.numel()
    y = torch.sigmoid(x)
    sg = torch.sign(y.float().double() - t)
    bce = x.clamp(min=0) - x * t + torch.log1p(torch.exp(-x.abs()))
    ref = {"dlogits": (sg * y * (1 - y) + y - t) / n, "Y": y, "l1": (y - t).abs().sum(), "bce": bce.sum()}
    sc = {"dlogits": (sg.abs() * y * (1 + y) + y + t.abs()) / n, "Y": y,
          "l1": (y + t.abs()).sum(), "bce": (x.clamp(min=0) + x.abs() * t.abs() + torch.log1p(torch.exp(-x.abs()))).sum()}
    return ref, sc


# --------------------------------------------------------------------------------------------- Adam
BETA1, BETA2, EPS = (float(np.float32(v)) for v in (0.9, 0.999, 1e-8))     # the constants the kernel is handed


def adam_lr_t(global_step, lr, warmup=4000.0, beta1=0.9, beta2=0.999):
    """The step size of train.py:122-132: the Noam schedule (utils.py:141-145) at global_step + 1 times Adam's bias
    correction sqrt(1 - beta2^t) / (1 - beta1^t), t = global_step + 1."""
    t = float(global_step + 1)
    lr_now = lr * warmup ** 0.5 * min(t * warmup ** -1.5, t ** -0.5)
    return lr_now * np.sqrt(1.0 - beta2 ** t) / (1.0 - beta1 ** t)


def adam(p, g, m, v, lr_t):
    """One Adam update of the step (float64; the kernel's float32 constants beta1, beta2, eps; lr_t as handed to the kernel):
    g clipped to [-1, 1] as min(max(g, -1), 1) with fmaxf's rule that a NaN operand loses (a NaN gradient clips to -1),
    m' = b1 m + (1 - b1) g, v' = b2 v + (1 - b2) g^2, p' = p - lr_t m' / (sqrt(v') + eps).  Returns (ref, scale) dicts of
    p, m, v."""
    p, g, m, v = (torch.as_tensor(a).double() for a in (p, g, m, v))
    g = torch.where(torch.isnan(g), -torch.ones_like(g), g.clamp(-1, 1))
    m1 = BETA1 * m + (1 - BETA1) * g
    v1 = BETA2 * v + (1 - BETA2) * g * g
    step = lr_t * m1 / (torch.sqrt(v1) + EPS)
    m_abs = BETA1 * m.abs() + (1 - BETA1) * g.abs()
    ref = {"p": p - step, "m": m1, "v": v1}
    sc = {"p": p.abs() + lr_t * m_abs / (torch.sqrt(v1) + EPS), "m": m_abs, "v": v1}
    return ref, sc
