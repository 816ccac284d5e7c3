"""The number format of the tensor-core kernels, emulated in numpy: an fp32 operand x is carried as two fp16 planes
hi = fp16(s x), lo = fp16(s x - hi) with a power-of-two scale s, and a product is hi*hi' + hi*lo' + lo*hi' accumulated in
fp32 (DESIGN.md section 5 and 8e; csrc/kernels_tc.cu, csrc/kernels_gemm_tc.cu).  These tests pin the claims the design rests
on: the scheme is fp32-grade (2^-22 per operand), single-pass fp16 / bf16 are not, the per-tensor scale of the training
GEMMs keeps 1e-7-sized gradients in fp16's normal range, and the per-utterance scale of a network input's planes keeps
silent frames (1e-8) there."""
import numpy as np


def _pow2_scale(x, top=13):
    m = float(np.abs(x).max())
    return 1.0 if m == 0 else 2.0 ** (top - int(np.floor(np.log2(m))))


def _planes(x, s):
    hi = (x * s).astype(np.float16)
    lo = (x * s - hi.astype(np.float32)).astype(np.float16)
    return hi.astype(np.float32), lo.astype(np.float32)


def _gemm3(a, b):
    """(M,K) x (N,K)^T with the three-product scheme and per-tensor scales, fp32 accumulation."""
    sa, sb = _pow2_scale(a), _pow2_scale(b)
    ah, al = _planes(a, np.float32(sa))
    bh, bl = _planes(b, np.float32(sb))
    acc = ah @ bh.T + ah @ bl.T + al @ bh.T
    return acc * np.float32(1.0 / (sa * sb))


def _bf16(x):
    u = x.astype(np.float32).view(np.uint32)
    r = ((u >> 16) & 1) + 0x7FFF
    return ((u + r) & 0xFFFF0000).view(np.float32)


def test_three_product_scheme_is_fp32_grade_and_single_pass_is_not():
    rng = np.random.default_rng(0)
    a = rng.normal(0, 1, (128, 768)).astype(np.float32)
    b = rng.normal(0, 0.05, (256, 768)).astype(np.float32)
    ref = a.astype(np.float64) @ b.astype(np.float64).T
    scale = np.abs(ref).max()
    err3 = np.abs(_gemm3(a, b) - ref).max() / scale
    err_fp32 = np.abs(a @ b.T - ref).max() / scale
    err_fp16 = np.abs(a.astype(np.float16).astype(np.float32) @ b.astype(np.float16).astype(np.float32).T - ref).max() / scale
    err_bf16 = np.abs(_bf16(a) @ _bf16(b).T - ref).max() / scale
    assert err3 < 2e-6 and err3 < 8 * max(err_fp32, 1e-7)          # within a small factor of fp32 FMA arithmetic
    assert err_fp16 > 20 * err3 and err_bf16 > 100 * err3           # why one pass misses the 1e-3 budget after 25 blocks


def test_per_tensor_scale_keeps_tiny_gradients_in_range():
    rng = np.random.default_rng(1)
    dy = (rng.normal(0, 1, (420, 512)) * 3e-7).astype(np.float32)   # gradient-sized values: unscaled fp16 would flush them
    x = rng.normal(0, 1, (420, 256)).astype(np.float32)
    ref = x.astype(np.float64).T @ dy.astype(np.float64)            # the weight-gradient GEMM: X^T dY
    got = _gemm3(np.ascontiguousarray(x.T), np.ascontiguousarray(dy.T))
    assert np.abs(got - ref).max() / np.abs(ref).max() < 2e-6
    naive = np.ascontiguousarray(x.T).astype(np.float16).astype(np.float32) @ dy.astype(np.float16).astype(np.float32)
    assert np.abs(naive - ref).max() / np.abs(ref).max() > 1e-2     # unscaled fp16: subnormal / flushed


def _first_block_ln(x, W, sx):
    """A zero-bias conv (size 1) + LayerNorm as the wgmma block computes it: input planes of sx * x, weight planes scaled
    into [2^10, 2^11), three products accumulated in fp32, the accumulator times 1 / (sx sw); LayerNorm in fp64 so that
    only the planes' error shows."""
    sw = 2.0 ** (11 - np.frexp(np.abs(W).max())[1])
    xh, xl = _planes(x, np.float32(sx))
    wh, wl = _planes(W, np.float32(sw))
    acc = (xh @ wh + xh @ wl + xl @ wh).astype(np.float32)
    return _ln64(acc.astype(np.float64) / (sx * sw))


def _ln64(y):
    m = y.mean(-1, keepdims=True)
    return (y - m) / np.sqrt(((y - m) ** 2).mean(-1, keepdims=True) + 1e-12)


def _utterance_scale(x):
    """f32_to_planes_scaled_kernel's scale: 2^k with max |x| * 2^k in [2^14, 2^15)."""
    m = float(np.abs(x).max())
    return 1.0 if m == 0 else 2.0 ** (15 - np.frexp(m)[1])


def test_quiet_inputs_need_a_scale_on_the_input_planes():
    """Silent mel frames sit at the 1e-8 floor; a zero-bias first block (the reference initialisers) feeds LayerNorm
    with the input alone, which then magnifies whatever the planes lost.  Unscaled fp16 planes flush 1e-8 and keep a few
    bits of 1e-6 .. 1e-4: beyond the 2e-4 block tolerance.  A power-of-two scale per utterance keeps them in fp16's
    normal range, also when the utterance's own loud frames set the scale."""
    from dc_tts_b200.params import init_params
    P = init_params(0, "tf_default")
    rng = np.random.default_rng(2)
    for scope in ("SSRN/C_1", "Text2Mel/AudioEnc/C_1"):
        W = P[scope + "/conv1d/kernel"][0]
        assert not P[scope + "/conv1d/bias"].any()
        for level in (1e-8, 1e-6, 1e-5, 1e-4):
            x = np.maximum(level * rng.uniform(0, 1, (8, W.shape[0])), 1e-8).astype(np.float32)
            ref = _ln64(x.astype(np.float64) @ W.astype(np.float64))
            unscaled = np.abs(_first_block_ln(x, W, 1.0) - ref).max()
            scaled = np.abs(_first_block_ln(x, W, _utterance_scale(x)) - ref).max()
            loud = np.concatenate([rng.uniform(0, 1, (8, W.shape[0])).astype(np.float32), x])     # voiced rows set the scale
            shared = np.abs(_first_block_ln(loud, W, _utterance_scale(loud))[8:] - ref).max()
            assert unscaled > 2e-4, (scope, level, unscaled)
            assert scaled < 1e-5 and shared < 1e-5, (scope, level, scaled, shared)
        floor = np.full((8, W.shape[0]), 1e-8, np.float32)                                        # the exact floor
        ref = _ln64(floor.astype(np.float64) @ W.astype(np.float64))
        assert np.abs(_first_block_ln(floor, W, 1.0) - ref).max() > 2e-4
        assert np.abs(_first_block_ln(floor, W, _utterance_scale(floor)) - ref).max() < 1e-5


def test_elements_far_below_the_tensor_maximum_lose_bits_gracefully():
    """One scale per tensor: an element 2^-20 below the maximum still has fp16's 11 bits (the hi plane is normal down to
    2^-27 of the maximum), so its contribution is wrong by at most 2^-11 of ITSELF -- negligible against the tensor's max-norm,
    which is what the gradient-parity criterion (2e-3 of the max-norm) measures."""
    a = np.zeros((1, 16), np.float32); b = np.ones((1, 16), np.float32)
    a[0, 0] = 1.0; a[0, 1] = 2.0 ** -20 * 1.2345
    got = _gemm3(a, b)[0, 0]
    ref = float(a.astype(np.float64).sum())
    assert abs(got - ref) <= 2.0 ** -11 * a[0, 1] + 2.0 ** -22
