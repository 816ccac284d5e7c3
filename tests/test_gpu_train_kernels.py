"""The training step's non-GEMM kernels one launch group at a time, against float64 (tests/ref_train_kernels.py).

  block backward  dctts_block_bwd (Engine.block_bwd): dropout mask, ReLU mask, highway gate and LayerNorm backward of one
                  block, with the gamma / beta / bias reductions
  attention       dctts_attn_bwd (Engine.attn_bwd): softmax backward with the guided-attention term, and its loss sum
  losses          dctts_train_loss (Engine.train_loss): L1 + BCE on the sigmoid, the logits' gradient, sigmoid_rows
  Adam            train_apply on the gradient arena (Engine.train_grads / train_set_tensor / train_tensor): clipping, the
                  Noam schedule and bias correction of the host, every element of every variable of both trainers

An element passes when |got - ref| <= TAU[kernel] * S + floor, S the reference's computation on absolute values.  A float32
kernel that rounds each operation once is off by a few 2^-24 (6e-8) S per operation in its chain; TAU is about 3-4x the
worst err / S seen on an H100 (DESIGN.md, "The training step's other kernels one launch at a time").  For the LayerNorm
backward S also carries (1 + kappa) per row, kappa = (|mean| + max |y - mean|) rstd: the float32 statistics leave yhat off
by 2^-24 kappa, which a plain |.| chain does not see on near-constant rows (offset >> spread).  The reductions (dgamma,
dbeta, dbias over up to 26880 rows, float atomics in no fixed order) get their own TAU.  Floors: none, except where the
float32 sigmoid underflows (losses: 2^-126 per term, the absolute error of a sigmoid that is 0 instead of ~1e-39).
"""
import collections

import numpy as np
import pytest
import torch

from dc_tts_b200 import arch
from dc_tts_b200.hyperparams import Hyperparams as hp

import ref_train_kernels as rk
from sample_rates import at_rate

# worst err / S over this file on an H100 80GB HBM3 at 700 W (DESIGN.md 8e): block backward per-row outputs 2.4e-7, its
# column reductions 1.55e-5 (float atomics over up to 840 CTAs), attention 1.75e-6, losses 1.9e-7, Adam 3.3e-7; the block
# forward (dctts_block_fwd) 1.75e-7
TAU = {"block": 1e-6, "block_sum": 6e-5, "attn": 6e-6, "loss": 8e-7, "adam": 1e-6, "block_fwd": 6e-7}
SENTINEL = -1234.5
_WORST = collections.defaultdict(lambda: [0.0, 0.0])            # kernel -> [max err / S, max err / tolerance]


def _r4(x):
    return (x + 3) // 4 * 4


def check(kernel, got, ref, scale, what, floor=0.0):
    """got (float32, any device) vs ref / scale (float64): finite, and |got - ref| <= TAU[kernel] scale + floor."""
    got = got.double()
    assert bool(torch.isfinite(got).all()), "NaN/inf in %s" % what
    err = (got - ref).abs()
    tol = TAU[kernel] * scale + floor
    ratio = float(torch.where(err > 0, err / tol, torch.zeros_like(err)).max()) if err.numel() else 0.0
    pos = TAU[kernel] * scale > floor                            # the elements S governs, not the floor
    rel = float((err[pos] / scale[pos]).max()) if bool(pos.any()) else 0.0
    w = _WORST[kernel]
    w[0], w[1] = max(w[0], rel), max(w[1], ratio)
    assert ratio <= 1.0, "%s: max err / tolerance %.3g (max err / S %.3g, tau %.1e)" % (what, ratio, rel, TAU[kernel])


@pytest.fixture(scope="module")
def eng():
    from dc_tts_b200.engine import Engine
    e = Engine(0)
    yield e
    print("\ntraining kernels, worst err/S and err/tolerance: " +
          ", ".join("%s %.3g %.3g" % (k, v[0], v[1]) for k, v in sorted(_WORST.items())))
    e.close()


# ============================================================================================= CPU: the references
def test_dropout_hash_matches_the_oracle():
    """The torch restatement of the step's dropout hash is oracle.ref_train's, bit for bit (the kernels share it)."""
    from oracle import ref_train
    idx = np.concatenate([np.arange(5000), np.array([2 ** 31 - 1, 2 ** 31, 2 ** 32 - 1, 55_000_000])]).astype(np.uint64)
    for layer, seed in ((0, 0), (37, 123456789), (15, 0xffffffff)):
        want = ref_train.mix32(idx, layer, seed).astype(np.int64)
        got = rk.mix32_torch(torch.from_numpy(idx.astype(np.int64)), layer, seed).numpy()
        assert np.array_equal(got, want)
    keep = rk.drop_multiplier(7, 13, 5, 99, 0.5).numpy()
    assert np.array_equal(keep.astype(np.float32), ref_train.dropout_keep((7, 13), 5, 99, float(np.float32(0.5))))


@pytest.mark.parametrize("mode,act", [(0, 0), (0, 1), (1, 0)])
def test_block_reference_matches_autograd(mode, act):
    """LN -> ReLU / highway -> dropout in float64 through torch.autograd: the hand-written backward agrees to 1e-12."""
    g = torch.Generator().manual_seed(10 * mode + act)
    rows, C = 9, 11
    nconv = 2 * C if mode else C
    pre = torch.randn(rows, nconv, generator=g, dtype=torch.float64) * 2 + 0.3
    ln = torch.cat([1 + 0.2 * torch.randn(1, C, generator=g, dtype=torch.float64),
                    0.3 * torch.randn(1, C, generator=g, dtype=torch.float64),
                    1 + 0.2 * torch.randn(1, C, generator=g, dtype=torch.float64),
                    0.3 * torch.randn(1, C, generator=g, dtype=torch.float64)])
    X = torch.randn(rows, C, generator=g, dtype=torch.float64)
    gout = torch.randn(rows, C, generator=g, dtype=torch.float64)
    keep = rk.drop_multiplier(rows, C, 3, 7, 0.3)
    ref, _ = rk.block_bwd(mode, act, pre, gout, ln, keep, X)
    pre_, ln_, X_ = (t.clone().requires_grad_(True) for t in (pre, ln, X))
    out = rk.block_forward(mode, act, pre_, ln_, keep, X_)
    gp, gl, gx = torch.autograd.grad((out * gout).sum(), (pre_, ln_, X_), allow_unused=True)
    close = lambda a, b: torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-12)    # noqa: E731
    close(ref["dy"], gp)
    close(ref["dbias"], gp.sum(0))
    close(ref["dg1"], gl[0])
    close(ref["db1"], gl[1])
    if mode == 1:
        close(ref["dg2"], gl[2])
        close(ref["db2"], gl[3])
        close(ref["gin"], gx)


def test_attention_reference_matches_autograd():
    """Softmax attention plus att_scale sum |A gts| over the (n_lim, t_lim) corner, through autograd in float64; the
    reference is handed the forward's alignments."""
    g = torch.Generator().manual_seed(3)
    B, T, N, d, n_lim, t_lim = 2, 6, 5, 8, 3, 4
    Q, K, V = (torch.randn(B, n, d, generator=g, dtype=torch.float64, requires_grad=True) for n in (T, N, N))
    gR = torch.randn(B, T, 2 * d, generator=g, dtype=torch.float64)
    gts = torch.rand(N + 1, T + 2, generator=g, dtype=torch.float64)
    loss, A = rk.attn_forward_loss(Q, K, V, gR, gts, n_lim, t_lim)
    gQ, gK, gV = torch.autograd.grad(loss, (Q, K, V))
    ref, _ = rk.attn_bwd(gR, Q.detach(), torch.cat([K, V], 2).detach(), A.detach(), gts, n_lim, t_lim)
    close = lambda a, b: torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-12)    # noqa: E731
    close(ref["gQ"], gQ)
    close(ref["gKV"], torch.cat([gK, gV], 2))
    att = (A.detach()[:, :n_lim, :t_lim] * gts[:n_lim, :t_lim]).abs().sum()
    close(ref["att"], att)


def test_loss_reference_matches_autograd():
    """mean |sigmoid(x) - t| + mean BCE-with-logits through autograd in float64, x = 0 at t = 0.5 (no slope: sign(0))
    included."""
    g = torch.Generator().manual_seed(4)
    x = torch.randn(7, 9, generator=g, dtype=torch.float64) * 4
    t = torch.rand(7, 9, generator=g, dtype=torch.float64)
    x[0, 0], t[0, 0] = 0.0, 0.5
    x_ = x.clone().requires_grad_(True)
    y = torch.sigmoid(x_)
    loss = (y - t).abs().mean() + torch.nn.functional.binary_cross_entropy_with_logits(x_, t)
    gx, = torch.autograd.grad(loss, x_)
    ref, _ = rk.train_loss(x, t)
    torch.testing.assert_close(ref["dlogits"], gx, rtol=1e-12, atol=1e-15)
    assert float(ref["dlogits"][0, 0]) == 0.0
    torch.testing.assert_close(ref["l1"] / x.numel() + ref["bce"] / x.numel(), loss.detach(), rtol=1e-12, atol=0)


def test_adam_reference_matches_ref_train():
    """The step size is ref_train's Noam schedule times the bias correction (1e-12), and the update is ref_train._adam's
    (which rounds to float32 at each step: 1e-6 of S, and 2^-126 where a subnormal gradient's square underflows) with the
    kernel's float32 constants."""
    from oracle import ref_train
    for step in (0, 3998, 3999, 4000, 10 ** 6):
        for lr in (0.001, 0.02):
            t = step + 1
            want = ref_train.learning_rate(step, lr) * np.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t)
            assert abs(rk.adam_lr_t(step, lr) - want) <= 1e-12 * want
    rng = np.random.default_rng(5)
    shape = (64,)
    g = rng.choice([0.0, 1e-40, 0.5, -0.5, 1.0, -1.0, 1.5, -1.5, 1e3, -1e3], shape).astype(np.float32)
    p = rng.standard_normal(shape).astype(np.float32)
    m = (rng.standard_normal(shape) * 0.1).astype(np.float32)
    v = rng.choice([0.0, 1e-12, 1e-4, 1.0], shape).astype(np.float32)
    step = 3999
    lr_t = rk.adam_lr_t(step, 0.001)
    var = torch.zeros(shape, requires_grad=True)
    var.grad = torch.from_numpy(g)
    newP, state, _, _ = ref_train._adam({"w": p}, ["w"], {"w": var}, {"w": (m, v)}, step, 0.001, rk.BETA1, rk.BETA2, rk.EPS)
    ref, sc = rk.adam(p, g, m, v, lr_t)
    for k, got in (("p", newP["w"]), ("m", state["w"][0]), ("v", state["w"][1])):
        assert bool(((torch.from_numpy(got).double() - ref[k]).abs() <= 1e-6 * sc[k] + 2.0 ** -126).all()), k


# ============================================================================================= block backward
Block = collections.namedtuple("Block", "mode C act name")


def block_cases():
    """Every (mode, C, act) of both trainers (SSRN at n_fft 1024, 2048 and 4096: F = 513, 1025, 2049), conv1d with ReLU on
    and off at every width a block has, highway at every width a highway block has, and the edges of the kernel's MAXV
    instantiations (128, 1056 for both modes, 2080 for conv1d)."""
    blocks = [("Text2Mel/" + n.split("/")[1], l) for n, fn in arch.NETWORKS.items() if n != "SSRN" for l in fn()]
    for sr in (16000, 22050, 44100):
        with at_rate(sr) as h:
            blocks += [("SSRN@%d" % h.n_fft, l) for l in arch.ssrn_layers()]
    cases = collections.OrderedDict()
    for name, l in blocks:
        mode = 1 if l.kind == "HC" else 0
        acts = (0,) if mode else (0, 1)
        for act in acts:
            cases.setdefault((mode, l.cout, act), "%s/%s" % (name, l.scope))
    for key in ((0, 128, 0), (0, 128, 1), (1, 128, 0), (0, 1056, 1), (1, 1056, 0), (0, 2080, 1)):
        cases.setdefault(key, "MAXV edge")
    return [Block(m, C, a, n) for (m, C, a), n in cases.items()]


BLOCKS = block_cases()


def _block_id(c):
    return "%s-C%d%s" % ("hc" if c.mode else "conv", c.C, "-relu" if c.act else "")


def test_block_cases_cover_every_instantiation():
    widths = {c.C for c in BLOCKS}
    assert {80, 256, 512, 513, 1024, 1025, 2049} <= widths
    assert {c.C for c in BLOCKS if c.mode == 1} >= {256, 512, 1024, 1056}
    bounds = (128, 256, 512, 1024, 1056, 2080)                   # MAXV 4, 8, 16, 32, 33 (both modes), 65 (conv1d)
    for lo, hi in zip((0,) + bounds, bounds):
        assert any(lo < c.C <= hi for c in BLOCKS), (lo, hi)


def _block_inputs(c, rows, gen, dev):
    """Rows by row % 8: 0-3 O(1) with offsets, 4 exactly 0 and 5 exactly 0.75 (the epsilon path: TextEnc's padding with
    zero biases at step 0), 6 near-constant (1 + 1e-3 u: offset >> spread), 7 at 1e-6 scale.  beta1 is exactly 0 in every
    4th column, so a constant row has z = 0 exactly there (the ReLU edge)."""
    C, nconv = c.C, (2 * c.C if c.mode else c.C)
    u = lambda *s: torch.rand(*s, generator=gen, device=dev) * 2 - 1     # noqa: E731
    pre = u(rows, nconv) * 1.5 + u(rows, 1) * 0.5
    kind = torch.arange(rows, device=dev) % 8
    pre = torch.where((kind == 4)[:, None], torch.zeros_like(pre), pre)
    pre = torch.where((kind == 5)[:, None], torch.full_like(pre, 0.75), pre)
    pre = torch.where((kind == 6)[:, None], 1 + 1e-3 * u(rows, nconv), pre)
    pre = torch.where((kind == 7)[:, None], 1e-6 * u(rows, nconv), pre)
    if rows == 1:
        pre = u(rows, nconv)
    ln = torch.stack([1 + 0.2 * u(C), 0.3 * u(C), 1 + 0.2 * u(C), 0.3 * u(C)])
    ln[1, ::4] = 0.0
    gout = 1e-3 * u(rows, C)
    X = u(rows, C)
    return pre, ln, gout, X


def run_block(eng, c, rows, rate, seed):
    dev = eng.device
    gen = torch.Generator(device=dev)
    gen.manual_seed(seed)
    C, nconv = c.C, (2 * c.C if c.mode else c.C)
    pre, ln, gout, X = _block_inputs(c, rows, gen, dev)
    layer = 3 + seed % 40
    keep = rk.drop_multiplier(rows, C, layer, seed, rate, dev)
    if c.act == 1:
        # a pre-activation within rounding of 0 may fall on either side of the mask: its gradient is zeroed, so both
        # sides agree; constant rows (kappa 0, z = beta1 exactly) keep theirs -- they pin the z > 0 edge
        yh, r, m = rk.ln_forward(pre[:, :C].double())
        kap = rk.ln_sensitivity(pre[:, :C].double(), yh, m, r)
        z = yh * ln[0].double() + ln[1].double()
        near = (z.abs() < 1e-4 * (1 + kap)) & (kap > 0)
        gout = torch.where(near, torch.zeros_like(gout), gout)
    ldy, ldg, ldx = _r4(nconv) + 4, _r4(C) + 4, _r4(C) + 8
    nan = float("nan")
    pbuf = torch.full((rows, ldy), nan, device=dev); pbuf[:, :nconv] = pre
    gbuf = torch.full((rows, ldg), nan, device=dev); gbuf[:, :C] = gout
    xbuf = torch.full((rows, ldx), nan, device=dev); xbuf[:, :C] = X
    dy = torch.full((rows, ldy), SENTINEL, device=dev)
    gin = torch.full((rows, ldg), SENTINEL, device=dev)
    dp0 = 1e-3 * (torch.rand(4 * C + nconv, generator=gen, device=dev) * 2 - 1)
    dp = dp0.clone()
    eng.block_bwd(c.mode, c.act, C, pbuf[:, :nconv], gbuf[:, :C], ln, dy[:, :nconv], dp,
                  X=xbuf[:, :C] if c.mode else None, gin=gin[:, :C] if c.mode else None, dropout_rate=rate, layer=layer, seed=seed)
    ref, sc = rk.block_bwd(c.mode, c.act, pre, gout, ln, keep, X)
    where = "%s rows %d rate %g" % (_block_id(c), rows, rate)
    assert bool((dy[:, nconv:] == SENTINEL).all()), "a pad column of dy was written: " + where
    check("block", dy[:, :nconv], ref["dy"], sc["dy"], "dy " + where)
    if c.mode:
        assert bool((gin[:, C:] == SENTINEL).all()), "a pad column of gin was written: " + where
        check("block", gin[:, :C], ref["gin"], sc["gin"], "gin " + where)
    d64, a64 = dp0.double(), dp0.double().abs()
    parts = (("dg1", 0), ("db1", C)) + ((("dg2", 2 * C), ("db2", 3 * C)) if c.mode else ())
    for k, o in parts + (("dbias", 4 * C),):
        n = nconv if k == "dbias" else C
        check("block_sum", dp[o:o + n], d64[o:o + n] + ref[k], a64[o:o + n] + sc[k], "%s %s" % (k, where))
    if not c.mode:
        assert torch.equal(dp[2 * C:4 * C], dp0[2 * C:4 * C]), "a conv1d block wrote dgamma2 / dbeta2: " + where


@pytest.mark.gpu
@pytest.mark.parametrize("case", BLOCKS, ids=_block_id)
def test_block_bwd_vs_float64(eng, case):
    """rows 1, 31, 32, 33 (32 rows per CTA) at dropout 0, 0.05 and 0.5; B L = 32 x 840 rows at 0.05."""
    for rate in (0.0, 0.05, 0.5):
        for rows in (1, 31, 32, 33):
            run_block(eng, case, rows, rate, seed=rows + int(rate * 100))
    run_block(eng, case, 32 * 840, 0.05, seed=11)


# The forward twin: train_fwd's LayerNorm epilogue with the dropout mask (dctts_block_fwd, one launch_ln_rows).  Every MAXV
# instantiation of ln_rows_kernel (C = 80 and 256: 8, 512: 16, 1024: 32, 1025: 33, 2049: 65), both modes, ReLU on and off.
# Rows 1 and 255 run 2 warps per CTA and 2051 runs 8; without dropout, C <= 256 and at most 1024 rows take ln_row_cta_kernel.
FWD = [Block(m, C, a, "forward") for C in (80, 256, 512, 1024, 1025, 2049) for m, a in ((0, 0), (0, 1), (1, 0))]


def _block_fwd_restated(c, pre, ln, keep, X):
    """block_forward restated in float32 (torch, the kernel's operation order aside)."""
    C = c.C
    v = pre[:, :C].float()
    m = v.mean(1, keepdim=True)
    z1 = (v - m) / torch.sqrt(((v - m) ** 2).mean(1, keepdim=True) + rk.LN_EPS) * ln[0] + ln[1]
    if c.mode == 0:
        out = torch.relu(z1) if c.act else z1
    else:
        w = pre[:, C:2 * C].float()
        m2 = w.mean(1, keepdim=True)
        z2 = (w - m2) / torch.sqrt(((w - m2) ** 2).mean(1, keepdim=True) + rk.LN_EPS) * ln[2] + ln[3]
        h1 = torch.sigmoid(z1)
        out = h1 * z2 + (1 - h1) * X
    return out * keep.float()


@pytest.mark.parametrize("mode,act", [(0, 0), (0, 1), (1, 0)])
def test_block_forward_scale(mode, act):
    """CPU: block_forward_scale's value is block_forward's, and a float32 restatement stays below TAU / 4 of its S."""
    c = Block(mode, 512, act, "cpu")
    gen = torch.Generator().manual_seed(mode * 2 + act)
    pre, ln, _, X = _block_inputs(c, 64, gen, "cpu")
    keep = rk.drop_multiplier(64, c.C, 5, 9, 0.05)
    ref, S = rk.block_forward_scale(mode, act, pre, ln, keep, X)
    want = rk.block_forward(mode, act, pre.double(), ln.double(), keep, X.double())
    assert float((ref - want).abs().max()) < 1e-12
    got = _block_fwd_restated(c, pre, ln, keep, X).double()
    r = (got - ref).abs() / S
    assert bool(((S > 0) | (got == ref)).all())
    assert float(torch.where(S > 0, r, torch.zeros_like(r)).max()) < TAU["block_fwd"] / 4


@pytest.mark.gpu
@pytest.mark.parametrize("case", FWD, ids=_block_id)
def test_block_fwd_vs_float64(eng, case):
    """Dropout 0, 0.05 and 0.5 at 1, 255 and 2051 rows; pad columns of out untouched."""
    dev = eng.device
    C, nconv = case.C, (2 * case.C if case.mode else case.C)
    for rate in (0.0, 0.05, 0.5):
        for rows in (1, 255, 2051):
            seed = rows + int(rate * 100)
            gen = torch.Generator(device=dev)
            gen.manual_seed(seed)
            pre, ln, _, X = _block_inputs(case, rows, gen, dev)
            layer = 3 + seed % 40
            keep = rk.drop_multiplier(rows, C, layer, seed, rate, dev)
            nan = float("nan")
            pbuf = torch.full((rows, _r4(nconv) + 4), nan, device=dev); pbuf[:, :nconv] = pre
            xbuf = torch.full((rows, _r4(C) + 8), nan, device=dev); xbuf[:, :C] = X
            out = torch.full((rows, _r4(C) + 4), SENTINEL, device=dev)
            eng.block_fwd(case.mode, case.act, C, pbuf[:, :nconv], ln, out[:, :C], X=xbuf[:, :C] if case.mode else None,
                          dropout_rate=rate, layer=layer, seed=seed)
            ref, S = rk.block_forward_scale(case.mode, case.act, pre, ln, keep, X)
            where = "%s rows %d rate %g" % (_block_id(case), rows, rate)
            assert bool((out[:, C:] == SENTINEL).all()), "a pad column of out was written: " + where
            check("block_fwd", out[:, :C], ref, S, "out " + where)


@pytest.mark.gpu
def test_block_bwd_refuses_widths_without_a_kernel(eng):
    """A highway block wider than 1056 channels and any block wider than 2080 fail with a message, launching nothing."""
    from dc_tts_b200.engine import DcttsError
    dev = eng.device
    for mode, C, msg in ((1, 1057, "no hc kernel"), (1, 2080, "no hc kernel"), (0, 2081, "exceed"), (1, 2081, "exceed")):
        nconv = 2 * C if mode else C
        pre = torch.zeros(4, nconv, device=dev)
        dy = torch.full((4, nconv), SENTINEL, device=dev)
        dp = torch.ones(4 * C + nconv, device=dev)
        X = torch.zeros(4, C, device=dev) if mode else None
        gin = torch.full((4, C), SENTINEL, device=dev) if mode else None
        n0 = eng.launch_count()
        with pytest.raises(DcttsError, match=msg):
            eng.block_bwd(mode, 0, C, pre, torch.zeros(4, C, device=dev), torch.ones(4, C, device=dev), dy, dp, X=X, gin=gin)
        assert eng.launch_count() == n0
        assert bool((dy == SENTINEL).all()) and bool((dp == 1).all())
    with pytest.raises(DcttsError, match="needs X and gin"):
        eng.block_bwd(1, 0, 8, torch.zeros(4, 16, device=dev), torch.zeros(4, 8, device=dev), torch.ones(4, 8, device=dev),
                      torch.zeros(4, 16, device=dev), torch.zeros(48, device=dev))
    with pytest.raises(DcttsError, match="columns"):
        eng.block_bwd(0, 0, 8, torch.zeros(4, 6, device=dev), torch.zeros(4, 8, device=dev), torch.ones(4, 8, device=dev),
                      torch.zeros(4, 6, device=dev), torch.zeros(40, device=dev))
    with pytest.raises(DcttsError, match="bad arguments"):
        eng.block_bwd(0, 0, 8, torch.zeros(4, 8, device=dev), torch.zeros(4, 8, device=dev), torch.ones(4, 8, device=dev),
                      torch.zeros(4, 8, device=dev), torch.zeros(40, device=dev), dropout_rate=1.0)


# ============================================================================================= attention backward
Attn = collections.namedtuple("Attn", "B T N n_lim t_lim")


def attn_cases():
    """N across 1, 2, the 32-key edges, max_N = 180 and past it, 300, and 3072 / 3073 (4 warps x N floats of dA crosses the
    48 KB default of dynamic shared memory at 3073); T from 1 to 211; B 1, 3 and 32; crops with n_lim < N and t_lim < T."""
    cases = []
    for i, N in enumerate((1, 2, 33, 180, 181, 300, 3072, 3073)):
        cases.append(Attn(3, 211, N, N, 211))
        cases.append(Attn(1, (1, 7)[i % 2], N, N, (1, 7)[i % 2]))
    cases += [Attn(32, 210, 180, 180, 210), Attn(32, 7, 3073, 180, 7), Attn(3, 210, 300, 180, 200), Attn(1, 211, 181, 180, 210),
              Attn(3, 7, 33, 1, 1), Attn(32, 211, 33, 20, 210)]
    return cases


ATTN = attn_cases()


def run_attn(eng, c, seed):
    dev = eng.device
    gen = torch.Generator(device=dev)
    gen.manual_seed(seed)
    d = eng.hp.d
    u = lambda *s: torch.rand(*s, generator=gen, device=dev) * 2 - 1     # noqa: E731
    B, T, N = c.B, c.T, c.N
    Q, KV = u(B, T, d), u(B, N, 2 * d)
    gR = 1e-3 * u(B, T, 2 * d)
    # alignments: per utterance a flat, a peaked or an underflowing softmax (exact zeros: the sign(0) branch)
    sharp = torch.tensor([0.0, 8.0, 300.0], device=dev, dtype=torch.float64)[(torch.arange(B, device=dev) + seed) % 3]
    logits = torch.randn(B, T, N, generator=gen, device=dev, dtype=torch.float64) * sharp[:, None, None]
    A = torch.softmax(logits, 2).float()
    A = torch.where(A < 1e-20, torch.zeros_like(A), A)
    align = A.transpose(1, 2).contiguous()
    # the table: finite over (N, T) -- a term past the crop shows as a wrong value -- with exact zeros, NaN past T
    ld_gts = T + 5
    gts = torch.full((N + 2, ld_gts), float("nan"), device=dev)
    gts[:N, :T] = torch.rand(N, T, generator=gen, device=dev)
    gts[:N, :T][torch.rand(N, T, generator=gen, device=dev) < 0.1] = 0.0
    gQ = torch.full((B, T, d), SENTINEL, device=dev)
    gKV = torch.full((B, N, 2 * d), SENTINEL, device=dev)
    s0 = torch.tensor([3.25, -1.5, 0.125], device=dev, dtype=torch.float64)
    sums = s0.clone()
    eng.attn_bwd(gR, Q, KV, align, gts, c.n_lim, c.t_lim, gQ, gKV, sums)
    ref, sc = rk.attn_bwd(gR, Q, KV, align, gts, c.n_lim, c.t_lim)
    where = "B %d T %d N %d crop (%d, %d)" % c
    check("attn", gQ, ref["gQ"], sc["gQ"], "gQ " + where)
    check("attn", gKV, ref["gKV"], sc["gKV"], "gKV " + where)
    assert torch.equal(sums[:2], s0[:2]), "sums[0:2] written: " + where
    check("attn", sums[2:], s0[2:] + ref["att"], s0[2:].abs() + sc["att"], "sum |A gts| " + where)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ATTN, ids=lambda c: "B%d-T%d-N%d-crop%d.%d" % c)
def test_attn_bwd_vs_float64(eng, case):
    for seed in (0, 1, 2):                                     # each utterance under each alignment profile
        run_attn(eng, case, seed)


@pytest.mark.gpu
def test_attn_bwd_refuses_what_the_kernels_cannot_run(eng):
    """A crop outside the step or wider than the table's stride, and d != 256, fail with a message, launching nothing."""
    from dc_tts_b200.engine import DcttsError, Engine
    dev = eng.device
    B, T, N, d = 1, 4, 3, eng.hp.d
    args = lambda dd: [torch.zeros(B, T, 2 * dd, device=dev), torch.zeros(B, T, dd, device=dev),     # noqa: E731
                       torch.zeros(B, N, 2 * dd, device=dev), torch.zeros(B, N, T, device=dev)]
    gts = torch.zeros(N, T, device=dev)
    outs = lambda dd: [torch.full((B, T, dd), SENTINEL, device=dev), torch.full((B, N, 2 * dd), SENTINEL, device=dev),  # noqa: E731
                       torch.zeros(3, device=dev, dtype=torch.float64)]
    for n_lim, t_lim, g in ((0, 4, gts), (4, 4, gts), (3, 5, gts), (3, 0, gts), (3, 4, torch.zeros(N, 3, device=dev))):
        o = outs(d)
        n0 = eng.launch_count()
        with pytest.raises(DcttsError, match="crop|at least n_lim"):
            eng.attn_bwd(*args(d), g, n_lim, t_lim, *o)
        assert eng.launch_count() == n0 and bool((o[0] == SENTINEL).all()) and bool((o[1] == SENTINEL).all())
    with pytest.raises(DcttsError, match="at least n_lim"):                  # a table smaller than the crop
        eng.attn_bwd(*args(d), torch.zeros(N - 1, T, device=dev), N, T, *outs(d))

    class HP128(hp):
        d = 128
    e = Engine(0, hparams=HP128)
    try:
        with pytest.raises(DcttsError, match="d = 256"):
            e.attn_bwd(*args(128), gts, N, T, *outs(128))
    finally:
        e.close()


# ============================================================================================= losses
SPECIAL_X = (0.0, 1e-8, -1e-8, 20.0, -20.0, 88.0, -88.0, 89.0, -89.0, 104.0, -104.0)
SIGMOID_EXACT_X = (0.0, 1e-8, -1e-8, 20.0, 88.0, 89.0, -89.0, 104.0, -104.0)   # float32 sigmoid_acc(x) = fl32(sigmoid(x))


def run_loss(eng, rows, C, seed):
    dev = eng.device
    gen = torch.Generator(device=dev)
    gen.manual_seed(seed)
    n = rows * C
    x = (torch.rand(n, generator=gen, device=dev) * 12 - 6)
    t = torch.rand(n, generator=gen, device=dev)
    i = torch.arange(n, device=dev)
    sx = torch.tensor(SPECIAL_X, device=dev)
    special = i % 3 == 0
    x = torch.where(special, sx[(i // 3) % len(sx)], x)
    tv = torch.tensor([0.0, 1.0, 0.5], device=dev)
    t = torch.where(special & ((i // 3 // len(sx)) % 4 < 3), tv[(i // 3 // len(sx)) % 4 % 3], t)
    # targets equal to the float32 sigmoid where it is exact (d == 0: the sign(0) branch)
    ex = torch.tensor(SIGMOID_EXACT_X, device=dev)
    on = (i % 7 == 1)
    xe = ex[(i // 7) % len(ex)]
    x = torch.where(on, xe, x)
    t = torch.where(on, torch.sigmoid(xe.double()).float(), t)
    # elsewhere keep the target clear of the float32 sigmoid (the sign of y - t is then that of the exact difference)
    y64 = torch.sigmoid(x.double())
    close = ((y64 - t.double()).abs() < 1e-5) & ~on
    t = torch.where(close, torch.where(t > 0.5, t - 3e-5, t + 3e-5), t)
    x, t = x.view(rows, C), t.view(rows, C).contiguous()
    ldl, ldg = _r4(C) + 4, _r4(C) + 8
    lbuf = torch.full((rows, ldl), float("nan"), device=dev); lbuf[:, :C] = x
    gbuf = torch.full((rows, ldg), SENTINEL, device=dev)
    Y = torch.full((rows, C), SENTINEL, device=dev)
    s0 = torch.tensor([0.75, -2.5], device=dev, dtype=torch.float64)
    sums = s0.clone()
    eng.train_loss(lbuf[:, :C], t, gbuf[:, :C], sums, Y=Y)
    ref, sc = rk.train_loss(x, t)
    where = "rows %d C %d" % (rows, C)
    tiny = 2.0 ** -126
    assert bool((gbuf[:, C:] == SENTINEL).all()), "a pad column of dlogits was written: " + where
    check("loss", gbuf[:, :C], ref["dlogits"], sc["dlogits"], "dlogits " + where, floor=4 * tiny / n)
    check("loss", Y, ref["Y"], sc["Y"], "Y " + where, floor=tiny)
    check("loss", sums[0:1], s0[0:1] + ref["l1"], s0[0:1].abs() + sc["l1"], "sum |y - t| " + where, floor=n * tiny)
    check("loss", sums[1:2], s0[1:2] + ref["bce"], s0[1:2].abs() + sc["bce"], "sum BCE " + where)
    dz = on.view(rows, C) & (x == 0)
    assert bool((gbuf[:, :C][dz] == 0).all()), "d == 0 did not give a zero gradient: " + where


@pytest.mark.gpu
@pytest.mark.parametrize("rows,C", [(1, 80), (37, 80), (32 * 210, 80), (3, 513), (5, 1025), (4 * 840, 1025), (2, 2049)])
def test_train_loss_vs_float64(eng, rows, C):
    """rows C not a multiple of 256, pitched logits and gradient (NaN / a sentinel in the pad columns), pre-filled sums;
    logits at 0, +-1e-8, +-20, +-88, +-89, +-104 against targets 0, 1, 0.5 and the float32 sigmoid itself."""
    run_loss(eng, rows, C, seed=rows + C)


# ============================================================================================= Adam
GRAD_VALUES = (0.0, 1e-40, -1e-40, 0.5, -0.5, 1.0, -1.0, 1.5, -1.5, 1e3, -1e3, float("inf"), float("-inf"), float("nan"))
V_VALUES = (0.0, 1e-16, 1e-12, 1e-8, 1e-4, 1e-2, 1.0)


def _adam_setup(eng, names, seed):
    """Random variables (a quarter exactly 0), first moments (a quarter 0) and second moments from V_VALUES (0 included);
    the gradient arena from GRAD_VALUES (a subnormal, values past the clip, +-inf and NaN) and uniform in (-2, 2)."""
    rng = np.random.default_rng(seed)
    shapes = arch.param_shapes()
    state = {}
    for n in names:
        s = shapes[n]
        p = (rng.standard_normal(s) * 0.1).astype(np.float32) * (rng.random(s) > 0.25)
        m = (rng.standard_normal(s) * 0.01).astype(np.float32) * (rng.random(s) > 0.25)
        v = np.asarray(V_VALUES, np.float32)[rng.integers(0, len(V_VALUES), s)]
        for what, a in (("param", p), ("m", m), ("v", v)):
            eng.train_set_tensor(n, a, what)
        state[n] = (p, m, v)
    G = eng.train_grads()
    gen = torch.Generator(device=G.device)
    gen.manual_seed(seed)
    vals = torch.tensor(GRAD_VALUES, device=G.device)
    pick = torch.randint(0, 2 * len(GRAD_VALUES), G.shape, generator=gen, device=G.device)
    uni = torch.rand(G.shape, generator=gen, device=G.device) * 4 - 2
    G.copy_(torch.where(pick < len(GRAD_VALUES), vals[pick.clamp(max=len(GRAD_VALUES) - 1)], uni))
    torch.cuda.synchronize()
    return state, {n: eng.train_tensor(n, "grad") for n in names}


def run_adam(eng, names, state, grads, step, lr, where):
    """One train_apply; every element of every variable, m and v against the float64 update.  Floors: a moment below
    float32's normal range carries 2^-149 of absolute error per operation (and the square of a subnormal gradient
    underflows): 2^-126 for m and v, and that divided by eps times lr_t for the variable.  Returns the new state."""
    eng.train_apply(step, lr)
    lr_t = rk.adam_lr_t(step, float(np.float32(hp.lr if lr is None else lr)))
    new = {}
    for n in names:
        p, m, v = state[n]
        ref, sc = rk.adam(p, grads[n], m, v, lr_t)
        got = {k: eng.train_tensor(n, what) for k, what in (("p", "param"), ("m", "m"), ("v", "v"))}
        for k in ("p", "m", "v"):
            floor = 2.0 ** -126 * (lr_t / rk.EPS if k == "p" else 1.0)
            check("adam", torch.from_numpy(got[k]), ref[k], sc[k], "%s of %s (%s)" % (k, n, where), floor=floor)
        new[n] = (got["p"], got["m"], got["v"])
    return new


@pytest.mark.gpu
def test_adam_every_variable_of_both_trainers(eng):
    """train_apply at global steps 0, 3998, 3999 (the top of the warm-up), 4000 and 10^6, at the default and a custom lr,
    over all 209 Text2Mel and 80 SSRN variables (an Adam table entry of the wrong length shows in the variable after it),
    one step after train_reserve grew the workspace.

    A NaN gradient element clips to -1 (fmaxf returns its non-NaN operand) and takes a full-size step; +-inf clips to +-1
    like any value past the clip.  This pins what the step does.  NaN gradients do reach the clip: the float32 graph's own
    gradients overflow on the first step from the reference's initialisers (test_float32_graph_overflows_at_the_
    reference_initialisation below, DESIGN.md 8e).  Whether tf.clip_by_value passes NaN through on the GPU has not been
    checked here; np.clip, the oracle's stand-in for it, does."""
    from dc_tts_b200.params import init_params
    eng.load_params(init_params(0, "perturbed"))
    eng.train_init(2)
    names = [n for n in arch.param_shapes() if n.startswith("Text2Mel/")]
    assert len(names) == 209
    state, grads = _adam_setup(eng, names, seed=1)
    for step, lr in ((0, None), (3998, None), (3999, None), (3999, 0.02), (4000, None), (10 ** 6, None), (10 ** 6, 0.5)):
        state = run_adam(eng, names, state, grads, step, lr, "Text2Mel step %d lr %s" % (step, lr))
    eng.train_reserve(hp.max_N + 20, hp.max_T + 30)
    state = run_adam(eng, names, state, grads, 4001, None, "Text2Mel after train_reserve")
    eng.train_init_ssrn(1, 8)
    names = [n for n in arch.param_shapes() if n.startswith("SSRN/")]
    assert len(names) == 80
    state, grads = _adam_setup(eng, names, seed=2)
    for step, lr in ((0, None), (4000, 0.003)):
        state = run_adam(eng, names, state, grads, step, lr, "SSRN step %d lr %s" % (step, lr))


# ============================================================================================= non-finite gradients
def _reference_init_batch():
    """The reference's initialisers (biases 0, gamma 1, beta 0) and one utterance of 30 characters padded to max_N."""
    from dc_tts_b200.params import init_params, synthetic_text
    L = synthetic_text(1, 30, seed=7)
    mels = np.random.default_rng(9).uniform(0, 1, (1, hp.max_T, hp.n_mels)).astype(np.float32)
    return init_params(1), L, mels


def _oracle_nonfinite_grads(P, L, mels):
    """Names of the Text2Mel variables whose float32 autograd gradient (oracle.ref_train, no dropout) is not finite."""
    from oracle import ref_train as rtr
    names = rtr.text2mel_names()
    T = {n: torch.tensor(np.asarray(P[n], np.float32), requires_grad=True) for n in names}
    rtr.forward(T, L, mels, 0, 0.0)["loss"].backward()
    return {n for n in names if T[n].grad is not None and not bool(torch.isfinite(T[n].grad).all())}


def test_float32_graph_overflows_at_the_reference_initialisation():
    """With zero biases and beta, a zero input row (TextEnc's padding, AudioEnc's first frame, which reads the zero frame
    the mels are shifted by) stays an exactly zero pre-LN row through every block.  LayerNorm with eps 1e-12 has a gain
    of rstd = 1e6 on such a row, so its backward multiplies the gradient by 1e6 per block; after a few blocks it passes
    float32's 3.4e38 and the gradients of every block below turn inf / NaN.  That is the float32 graph, not a kernel:
    autograd on the oracle shows it (48 variables of TextEnc and AudioEnc here).  Any non-zero beta breaks the chain."""
    from dc_tts_b200.params import init_params
    P, L, mels = _reference_init_batch()
    bad = _oracle_nonfinite_grads(P, L, mels)
    assert len(bad) >= 10 and all(n.startswith(("Text2Mel/TextEnc/", "Text2Mel/AudioEnc/")) for n in bad)
    assert not _oracle_nonfinite_grads(init_params(1, "perturbed"), L, mels)


@pytest.mark.gpu
def test_step_gradients_are_non_finite_where_the_float32_graphs_are():
    """The step on that batch: exactly the variables whose float32 autograd gradient is not finite have a non-finite
    gradient in the arena (Adam then clips NaN to -1: test_adam_every_variable_of_both_trainers)."""
    from dc_tts_b200.engine import Engine
    P, L, mels = _reference_init_batch()
    e = Engine(0)                                              # parameters are committed once per handle
    try:
        e.load_params(P)
        e.train_init(1, 0.0)
        e.train_step(L, mels, apply=False)
        names = [n for n in arch.param_shapes() if n.startswith("Text2Mel/")]
        got = {n for n in names if not np.isfinite(e.train_tensor(n, "grad")).all()}
    finally:
        e.close()
    assert got == _oracle_nonfinite_grads(P, L, mels)


@pytest.mark.gpu
def test_gradient_arena_is_finite_after_an_ordinary_step():
    """Away from that initialisation every element of the gradient arena is finite after a step of either trainer, the
    pad columns of SSRN's 1025-wide variables (pitch 1028) and the gaps between variables included."""
    from dc_tts_b200.engine import Engine
    from dc_tts_b200.params import init_params, synthetic_text
    e = Engine(0)                                              # parameters are committed once per handle
    try:
        e.load_params(init_params(0, "perturbed"))
        rng = np.random.default_rng(4)
        e.train_init(2)
        e.train_step(synthetic_text(2, 40, seed=3), rng.uniform(0, 1, (2, hp.max_T, hp.n_mels)).astype(np.float32),
                     global_step=5, seed=5, apply=False)
        G = e.train_grads()
        assert bool(torch.isfinite(G).all()), "Text2Mel: %d non-finite arena elements" % int((~torch.isfinite(G)).sum())
        T = 12
        e.train_init_ssrn(1, T)
        e.train_step_ssrn(rng.uniform(0, 1, (1, T, hp.n_mels)).astype(np.float32),
                          rng.uniform(0, 1, (1, hp.r * T, e.F)).astype(np.float32), global_step=5, seed=5, apply=False)
        G = e.train_grads()
        assert bool(torch.isfinite(G).all()), "SSRN: %d non-finite arena elements" % int((~torch.isfinite(G)).sum())
    finally:
        e.close()
