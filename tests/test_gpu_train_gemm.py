"""The conv-GEMMs of the training step, one launch at a time (dctts_conv_gemm), against float64, on both kernel sets.

Each block of the two trainers issues a forward conv, a data gradient and a weight gradient (api_train.cu train_fwd /
train_bwd); the transposed-conv blocks of SSRN issue three weight-gradient and two data-gradient launches on the
(B*L, 2*ldw) view of their gradient.  The cases below are generated from `arch`, deduplicated, and every one runs on the
fp32 CUDA-core kernels (impl 0) and, where the step can use them, the wgmma split-fp16 kernels (impl 1).

Reference: a tap loop of float64 matmuls with explicit zero padding per utterance (pinned on the CPU against
torch.nn.functional.conv1d, conv_transpose1d and autograd).  The same loop on |x|, |w| gives S = sum |x| |w| per output
element; with the bias and the tensor added onto (accumulate, the += of the weight gradient), S + |bias| + |out0| is the
error scale, and an element passes when |got - ref| <= TAU[impl] * S + floor.

floor: the wgmma operands are split into fp16 planes against a power-of-two scale PER TENSOR (its largest magnitude lands
in [2^13, 2^14)), so the lo plane of a small element underflows into fp16's subnormals: an operand element carries up to
max|x| * 2^-38 of absolute error whatever its own size, two operands per product, i.e. about max|a| max|b| 2^-37 per
reduction term.  floor = max|a| max|b| 2^-36 * (terms per output), with one bit to spare.  The 'span' magnitude profile
(rows from 1e-6 to 1) is where it matters.
"""
import collections

import pytest
import torch

from dc_tts_b200 import arch
from dc_tts_b200.hyperparams import Hyperparams as hp

# worst err / (S + |bias| + |out0|) over every case of this file on an H100 (DESIGN.md section 8e): 3.8e-7 on the fp32
# CUDA-core kernels, 2.45e-6 on the split-fp16 wgmma kernels (6.4x, inside the 8x the CPU emulation of the scheme
# predicts); TAU is about 4x and 3x of these
TAU = {0: 1.5e-6, 1: 8e-6}
FLOOR_BITS = 36
LENGTHS = (1, 2, 7, 31, 32, 33, 127, 128, 129, 210)
SSRN_LENGTH = 840                      # 4 * max_T: the widths after SSRN's two transposed convs
SENTINEL = -1234.5


# --------------------------------------------------------------------------------------------- float64 reference
def _shift(x, s):
    """x (B, L, C) -> y[b, t] = x[b, t + s], zero outside [0, L) of each utterance."""
    y = torch.zeros_like(x)
    L = x.shape[1]
    lo, hi = max(0, -s), min(L, L - s)
    if lo < hi:
        y[:, lo:hi] = x[:, lo + s:hi + s]
    return y


def ref_conv(X, W, shifts):
    """out[b, t, n] = sum_j sum_k X[b, t + shifts[j], k] W[j, k, n];  X (B, L, K), W (ntaps, K, N)."""
    return sum(_shift(X, s) @ W[j] for j, s in enumerate(shifts))


def ref_wgrad(X, dY, shifts):
    """dW[j, k, n] = sum_b sum_t X[b, t + shifts[j], k] dY[b, t, n];  X (B, L, K), dY (B, L, N)."""
    return torch.stack([torch.einsum("btk,btn->kn", _shift(X, s), dY) for s in shifts])


def layer_shifts(l, extra=0):
    """Source-row offsets of the taps of a conv block (api_train.cu layer_shifts)."""
    tot = (l.size - 1) * l.rate
    left = tot if l.pad == "CAUSAL" else tot // 2
    return tuple(j * l.rate - left + extra for j in range(l.size))


@pytest.mark.parametrize("size,rate,causal", [(1, 1, False), (3, 1, False), (3, 9, False), (3, 27, False), (3, 3, True), (3, 27, True)])
def test_reference_matches_conv1d_and_autograd(size, rate, causal):
    """The reference is a dilated conv1d (SAME or causal zero padding) and its two gradients, in float64; L = 20 < 27
    puts the outer taps of the rate-27 cases entirely in the padding."""
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(size * 100 + rate + causal)
    B, L, K, N = 3, 20, 5, 7
    X = torch.randn(B, L, K, generator=g, dtype=torch.float64, requires_grad=True)
    W = torch.randn(size, K, N, generator=g, dtype=torch.float64, requires_grad=True)
    tot = (size - 1) * rate
    left = tot if causal else tot // 2
    shifts = [j * rate - left for j in range(size)]
    Y = ref_conv(X, W, shifts)
    Yt = F.conv1d(F.pad(X.transpose(1, 2), (left, tot - left)), W.permute(2, 1, 0), dilation=rate).transpose(1, 2)
    torch.testing.assert_close(Y, Yt, rtol=1e-12, atol=1e-12)
    G = torch.randn(B, L, N, generator=g, dtype=torch.float64)
    gX, gW = torch.autograd.grad((Y * G).sum(), (X, W))
    # data gradient = the forward conv of G with transposed taps and negated shifts; weight gradient = ref_wgrad
    torch.testing.assert_close(gX, ref_conv(G, W.detach().transpose(1, 2), [-s for s in shifts]), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(gW, ref_wgrad(X.detach(), G, shifts), rtol=1e-12, atol=1e-12)


def test_reference_decomposes_the_transposed_conv():
    """SSRN's stride-2 transposed conv (kernel 3, 'same': out[2t] = x[t] W0 + x[t-1] W2, out[2t+1] = x[t] W1) and its
    gradients as the step computes them on the (B*L, 2C) view of dY: three single-tap weight gradients (even rows with
    shifts 0 and -1, odd rows with shift 0) and two data-gradient launches (even rows with taps W0^T, W2^T at shifts 0, +1,
    then the odd rows with W1^T added on)."""
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(5)
    B, L, K, N = 2, 9, 4, 6
    X = torch.randn(B, L, K, generator=g, dtype=torch.float64, requires_grad=True)
    W = torch.randn(3, K, N, generator=g, dtype=torch.float64, requires_grad=True)
    Y = torch.stack([ref_conv(X, W[[0, 2]], [0, -1]), ref_conv(X, W[[1]], [0])], dim=2).reshape(B, 2 * L, N)
    Yt = F.conv_transpose1d(X.transpose(1, 2), W.permute(1, 2, 0), stride=2)[..., :2 * L].transpose(1, 2)
    torch.testing.assert_close(Y, Yt, rtol=1e-12, atol=1e-12)
    G = torch.randn(B, 2 * L, N, generator=g, dtype=torch.float64)
    gX, gW = torch.autograd.grad((Y * G).sum(), (X, W))
    Ge, Go = G.reshape(B, L, 2 * N)[..., :N], G.reshape(B, L, 2 * N)[..., N:]
    Xd = X.detach()
    torch.testing.assert_close(gW, torch.cat([ref_wgrad(Xd, Ge, [0]), ref_wgrad(Xd, Go, [0]), ref_wgrad(Xd, Ge, [-1])]),
                               rtol=1e-12, atol=1e-12)
    WT = W.detach().transpose(1, 2)
    torch.testing.assert_close(gX, ref_conv(Ge, WT[[0, 2]], [0, 1]) + ref_conv(Go, WT[[1]], [0]), rtol=1e-12, atol=1e-12)


# --------------------------------------------------------------------------------------------- the step's GEMMs
Gemm = collections.namedtuple("Gemm", "role mode K N shifts ldx ldwd ldo acc xoff woff impls ssrn name")


def _r4(x):
    return (x + 3) // 4 * 4


def step_gemms():
    """Every conv-GEMM launch of the Text2Mel and SSRN trainers, deduplicated by (K, N, shifts, pitches, offsets)."""
    nets = [("Text2Mel/TextEnc", arch.textenc_layers(), hp.e), ("Text2Mel/AudioEnc", arch.audioenc_layers(), hp.n_mels),
            ("Text2Mel/AudioDec", arch.audiodec_layers(), 2 * hp.d), ("SSRN", arch.ssrn_layers(), hp.n_mels)]
    cases = collections.OrderedDict()

    def add(role, mode, K, N, shifts, ldx, ldwd, ldo, acc, impls, ssrn, name, xoff=0, woff=0):
        key = (role, mode, K, N, tuple(shifts), ldx, ldwd, ldo, acc, xoff, woff)
        old = cases.get(key)
        cases[key] = Gemm(role, mode, K, N, tuple(shifts), ldx, ldwd, ldo, acc, xoff, woff,
                          tuple(sorted(set(impls) | set(old.impls if old else ()))), ssrn or bool(old and old.ssrn),
                          old.name if old else name)

    for net, layers, ld_in in nets:
        ssrn = net == "SSRN"
        for i, l in enumerate(layers):
            name = "%s/%s" % (net, l.scope)
            first_of_input = i == 0 and net in ("Text2Mel/AudioEnc", "SSRN")       # no data gradient into the mels
            cin_p = _r4(l.cin)
            if l.kind == "D":
                ldw = _r4(l.cout)
                for sh, off in (((0,), 0), ((-1,), 0), ((0,), ldw)):
                    add("wgrad", 1, l.cin, l.cout, sh, ld_in, 2 * ldw, ldw, 1, (0,), ssrn, name, woff=off)
                add("dgrad", 0, l.cout, l.cin, (0, 1), 2 * ldw, cin_p, cin_p, 0, (0,), ssrn, name)
                add("dgrad", 0, l.cout, l.cin, (0,), 2 * ldw, cin_p, cin_p, 1, (0,), ssrn, name, xoff=ldw)
            else:
                nconv = 2 * l.cout if l.kind == "HC" else l.cout
                ldw = _r4(nconv)
                sh = layer_shifts(l, -1 if (net == "Text2Mel/AudioEnc" and i == 0) else 0)    # AudioEnc reads the mels one frame late
                add("fwd", 0, l.cin, nconv, sh, ld_in, ldw, ldw, 0, (0, 1), ssrn, name)
                add("wgrad", 1, l.cin, nconv, sh, ld_in, ldw, ldw, 1, (0, 1), ssrn, name)
                if not first_of_input:
                    add("dgrad", 0, nconv, l.cin, tuple(-s for s in sh), ldw, cin_p, cin_p, 1 if l.kind == "HC" else 0, (0, 1),
                        ssrn, name)
            ld_in = _r4(l.cout)
    return list(cases.values())


CASES = step_gemms()


def _case_id(c):
    return "%s-%s-K%d-N%d-s%s-ld%d.%d.%d%s%s" % (c.name.replace("Text2Mel/", ""), c.role, c.K, c.N, ",".join(map(str, c.shifts)),
                                               c.ldx, c.ldwd, c.ldo, "-acc" if c.acc and c.mode == 0 else "",
                                               "-off%d" % (c.xoff + c.woff) if c.xoff + c.woff else "")


def test_case_list_covers_the_edges():
    """The generated list has the shapes where GEMM kernels go wrong: the extra -1 shift of AudioEnc C_1, rate-27 taps,
    N and K tails (80, 1025), pitches above the width (1028, 2 * ldw), the transposed-conv view at a column offset,
    the accumulate of the highway data gradients, and both impls wherever the step can use the wgmma set."""
    ids = [_case_id(c) for c in CASES]
    assert len(set(ids)) == len(ids)
    by = lambda **kw: [c for c in CASES if all(getattr(c, k) == v for k, v in kw.items())]      # noqa: E731
    assert by(role="fwd", K=80, N=256, shifts=(-1,))                              # AudioEnc C_1
    assert by(role="fwd", shifts=(-27, 0, 27)) and by(role="fwd", shifts=(-54, -27, 0))
    assert by(role="dgrad", shifts=(54, 27, 0), acc=1)
    assert by(role="fwd", K=1025, N=1025, ldx=1028, ldwd=1028) and by(role="dgrad", K=1025, N=1024, ldx=1028)
    assert by(role="fwd", N=80) and by(role="wgrad", K=80)
    deconv = [c for c in CASES if "/D_" in c.name]
    assert len(deconv) == 5 and all(c.impls == (0,) for c in deconv)           # three weight- and two data-gradient launches
    assert [c.woff for c in deconv if c.role == "wgrad"] == [0, 0, 512] and [c.xoff for c in deconv if c.role == "dgrad"] == [0, 512]
    assert all(c.impls == (0, 1) for c in CASES if "/D_" not in c.name)
    assert sum(c.ssrn for c in CASES) >= 10 and len(CASES) >= 40


# --------------------------------------------------------------------------------------------- one launch
PROFILES = ("step", "unit", "span", "zero_a", "zero_b", "tiny")


def _operand(role, which, shape, prof, gen, dev):
    """Magnitudes: 'step' as in a training step (activations O(1), weights 1e-2, gradients 1e-7), 'unit' O(1), 'span' the
    rows of the first operand from 1e-6 to 1, 'zero_*' one operand all zero, 'tiny' both operands at max ~1e-16."""
    u = torch.rand(shape, generator=gen, device=dev, dtype=torch.float32) * 2 - 1
    if prof == "tiny":
        return u * 1e-16
    if prof == "zero_" + which:
        return torch.zeros_like(u)
    if prof == "unit":
        return u
    if prof == "span" and which == "a":                        # a is (B, L, K): one magnitude per row
        return u * torch.logspace(-6, 0, shape[0] * shape[1], device=dev, dtype=torch.float32).reshape(shape[0], shape[1], 1)
    size = {("fwd", "a"): 1.0, ("fwd", "b"): 1e-2, ("dgrad", "a"): 1e-7, ("dgrad", "b"): 1e-2,
            ("wgrad", "a"): 1.0, ("wgrad", "b"): 1e-7}[(role, which)]
    return u * size


_WORST = {0: [0.0, 0.0], 1: [0.0, 0.0]}           # impl -> [max err / S, max err / tolerance]


def run_case(eng, c, impl, B, L, prof, seed):
    dev = eng.device
    gen = torch.Generator(device=dev)
    gen.manual_seed(seed)
    nt = len(c.shifts)
    a = _operand(c.role, "a", (B, L, c.K), prof, gen, dev)
    b = _operand(c.role, "b", (nt, c.K, c.N) if c.mode == 0 else (B, L, c.N), prof, gen, dev)
    a64, b64 = a.double(), b.double()
    if c.mode == 0:
        P, S = ref_conv(a64, b64, c.shifts), ref_conv(a64.abs(), b64.abs(), c.shifts)
        terms = nt * c.K
    else:
        P, S = ref_wgrad(a64, b64, c.shifts), ref_wgrad(a64.abs(), b64.abs(), c.shifts)
        terms = B * L
    # the bias and the tensor added onto are of the product's own size (at O(1) they would hide its rounding)
    mag = float(P.abs().max()) or 1.0
    adds = prof not in ("tiny",)
    bias = (torch.rand(c.N, generator=gen, device=dev) - 0.5) * mag if (c.mode == 0 and adds) else torch.zeros(c.N, device=dev)
    init = c.acc or c.mode == 1
    out0 = (torch.rand(P.shape, generator=gen, device=dev, dtype=torch.float32) - 0.5) * mag if (init and adds) \
        else torch.zeros(P.shape, device=dev)
    # every pad column of every input is NaN (and the valid part of `out` too when it is overwritten, not added onto);
    # the pad columns of `out` hold a sentinel
    nan = float("nan")
    xbuf = torch.full((B, L, c.ldx), nan, device=dev)
    xbuf[..., c.xoff:c.xoff + c.K] = a
    if c.mode == 0:
        wbuf = torch.full((nt, c.K, c.ldwd), nan, device=dev)
        wbuf[..., :c.N] = b
        Wd = wbuf
        out = torch.full((B, L, c.ldo), SENTINEL, device=dev)
        out[..., :c.N] = out0 if init else nan
        bbuf = torch.full((c.ldwd,), nan, device=dev)
        bbuf[:c.N] = bias
    else:
        wbuf = torch.full((B, L, c.ldwd), nan, device=dev)
        wbuf[..., c.woff:c.woff + c.N] = b
        Wd = wbuf[..., c.woff:]
        out = torch.full((nt, c.K, c.ldo), SENTINEL, device=dev)
        out[..., :c.N] = out0
        bbuf = None
    eng.conv_gemm(impl, c.mode, xbuf[..., c.xoff:], c.K, Wd, c.N, c.shifts, out, bias=bbuf, accumulate=c.acc if c.mode == 0 else 1)
    got = out[..., :c.N].double()
    ref = P + bias.double() + (out0.double() if init else 0)
    scale = S + bias.double().abs() + (out0.double().abs() if init else 0)
    where = "%s impl %d B %d L %d %s" % (_case_id(c), impl, B, L, prof)
    assert bool(torch.isfinite(got).all()), "NaN/inf in a valid element: " + where
    if c.mode == 1 or impl == 1:                  # the fp32 forward kernel writes the whole pitch ldwd (the step's pre-LN rows)
        assert bool((out[..., c.N:] == SENTINEL).all()), "a pad column of out was written: " + where
    if prof == "zero_a" or prof == "zero_b":      # no product: exactly the bias on top of out0, or dW unchanged
        exact = (bias + out0) if c.mode == 0 else out0
        assert torch.equal(out[..., :c.N], exact), "zero operand did not give exactly bias / out0: " + where
    err = (got - ref).abs()
    floor = float(a.abs().max()) * float(b.abs().max()) * 2.0 ** -FLOOR_BITS * terms
    tol = TAU[impl] * scale + floor
    ratio = float(torch.where(err > 0, err / tol, torch.zeros_like(err)).max())
    pos = scale > 0
    rel = float((err[pos] / scale[pos]).max()) if bool(pos.any()) else 0.0
    w = _WORST[impl]
    w[0], w[1] = max(w[0], rel), max(w[1], ratio)
    assert ratio <= 1.0, "%s: max err / tolerance %.3g (max err / S %.3g, tau %.1e)" % (where, ratio, rel, TAU[impl])


@pytest.fixture(scope="module")
def eng():
    from dc_tts_b200.engine import Engine
    e = Engine(0)
    yield e
    print("\nconv-GEMM worst err/S and err/tolerance: fp32 %.3g %.3g, wgmma %.3g %.3g"
          % (_WORST[0][0], _WORST[0][1], _WORST[1][0], _WORST[1][1]))
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_gemm_vs_float64_at_every_length(eng, case):
    """B = 3 (different data per utterance), L from 1 to 210 across the 32-row and 128-row tile edges, and 840 for the
    SSRN widths; step-sized magnitudes."""
    lengths = LENGTHS + ((SSRN_LENGTH,) if case.ssrn else ())
    for L in lengths:
        for impl in case.impls:
            run_case(eng, case, impl, 3, L, "step", seed=L)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_gemm_vs_float64_batch_sizes_and_magnitudes(eng, case):
    """B = 1 and B = 32 (the weight gradient then reduces many ksplit CTAs into one dW), and every magnitude profile."""
    for impl in case.impls:
        run_case(eng, case, impl, 1, 210, "step", seed=1)
        run_case(eng, case, impl, 32, 129, "step", seed=2)
        for i, prof in enumerate(PROFILES[1:]):
            run_case(eng, case, impl, 3, 33, prof, seed=3 + i)


@pytest.mark.gpu
@pytest.mark.parametrize("role", ["fwd", "wgrad"])
def test_wgmma_output_scale_survives_tiny_operands(eng, role):
    """Both operands at max ~1e-16: each per-tensor scale is ~2^66, their product overflowed float32 and the epilogue's
    1 / (s_a s_b) zeroed every output; the inverses are now taken one at a time."""
    c = next(c for c in CASES if c.role == role and c.K == 256 and len(c.shifts) == 3)
    for impl in c.impls:
        run_case(eng, c, impl, 2, 40, "tiny", seed=7)


@pytest.mark.gpu
def test_conv_gemm_refuses_what_the_kernels_cannot_run(eng):
    """A layout the launch functions do not support fails with a message; nothing switches kernel sets."""
    from dc_tts_b200.engine import DcttsError
    dev = eng.device
    X = torch.zeros(2, 8, 8, device=dev)
    W = torch.zeros(1, 8, 8, device=dev)
    bias = torch.zeros(8, device=dev)
    out = torch.zeros(2, 8, 8, device=dev)
    eng.conv_gemm(1, 0, X, 8, W, 8, [0], out, bias=bias)
    with pytest.raises(DcttsError, match="impl"):
        eng.conv_gemm(2, 0, X, 8, W, 8, [0], out, bias=bias)
    with pytest.raises(DcttsError, match="multiples of 4"):
        eng.conv_gemm(0, 0, torch.zeros(2, 8, 6, device=dev), 6, torch.zeros(1, 6, 8, device=dev), 8, [0], out, bias=bias)
    with pytest.raises(DcttsError, match="ldo == ldwd"):
        eng.conv_gemm(1, 0, X, 8, torch.zeros(1, 8, 12, device=dev), 8, [0], out, bias=torch.zeros(12, device=dev))
    with pytest.raises(DcttsError, match="accumulate = 1"):
        eng.conv_gemm(1, 1, X, 8, X, 8, [0], torch.zeros(1, 8, 8, device=dev), accumulate=0)
    with pytest.raises(DcttsError, match="narrower"):
        eng.conv_gemm(0, 1, X, 12, X, 8, [0], torch.zeros(1, 12, 8, device=dev), accumulate=1)
    with pytest.raises(DcttsError, match="bad arguments"):
        eng.conv_gemm(1, 0, X, 8, torch.zeros(4, 8, 8, device=dev), 8, [0, 1, 2, 3], out, bias=bias)
