"""The fused conv + LayerNorm block kernel on full-sequence launches (128-row time tiles, one utterance per tile), at the
accumulator widths the networks use (64, 80, 144 and 256 columns per CTA, one full-width wgmma per product) and with one
k-block of MMAs in flight: every SSRN / TextEnc block kind against the float64 oracle and against the fp32 CUDA-core
kernels on identical inputs, at ragged and exact tile lengths, on grids below one wave and far above the co-resident
clusters, under every value of the tensor-core options."""
import zlib

import numpy as np
import pytest
import torch

from dc_tts_b200 import arch
from dc_tts_b200.hyperparams import Hyperparams as hp
from oracle import ref_torch as rt

pytestmark = pytest.mark.gpu
BLOCK_TOL = 2e-4          # against the oracle (same as test_gpu_tensor.py)
PATH_TOL = 1e-4           # against the fp32 CUDA-core kernels: both are fp32-grade, they differ by summation order
DEFAULTS = dict(tc_occ2=0, tc_mcast=1, tc_resid_tma=1)


@pytest.fixture()
def tc(engine):
    engine.set_tensor_path(1)
    yield engine
    for k, v in DEFAULTS.items():
        engine.set_option(k, v)
    engine.set_tensor_path(1)


def _layer(net, scope):
    return [l for l in arch.NETWORKS[net]() if l.scope == scope][0]


def _run(eng, net, scope, x):
    l = _layer(net, scope)
    full = net + "/" + scope
    if l.kind == "C":
        return eng.conv1d(full, x, l.cout, l.rate, l.pad == "CAUSAL", 1 if l.act == "relu" else 0)
    if l.kind == "HC":
        return eng.hc(full, x, l.rate, l.pad == "CAUSAL")
    return eng.conv1d_transpose(full, x)


def _oracle(params, net, scope, x):
    l = _layer(net, scope)
    full = net + "/" + scope
    xt = torch.from_numpy(x)
    with torch.no_grad():
        if l.kind == "C":
            return rt.conv1d(params, xt, full, l.rate, l.pad, l.act).numpy()
        if l.kind == "HC":
            return rt.hc(params, xt, full, l.rate, l.pad).numpy()
        return rt.conv1d_transpose(params, xt, full).numpy()


def _both_paths(eng, net, scope, x):
    out = _run(eng, net, scope, x).cpu().numpy()
    eng.set_tensor_path(0)
    try:
        out32 = _run(eng, net, scope, x).cpu().numpy()
    finally:
        eng.set_tensor_path(1)
    return out, out32


def _input(net, scope, B, L):
    l = _layer(net, scope)
    seed = zlib.crc32(("%s/%s/%d/%d" % (net, scope, B, L)).encode())
    return np.random.default_rng(seed).uniform(-1, 1, (B, L, l.cin)).astype(np.float32)


KINDS = [
    # net, scope: what the block exercises
    ("Text2Mel/TextEnc", "C_2"),      # relu C 128 -> 512: cluster 2 x 256 columns, K of two k-blocks
    ("Text2Mel/TextEnc", "HC_6"),     # hc 512, dilation 9, SAME padding: cluster 4 x 256
    ("SSRN", "C_10"),                 # C 512 -> 1024: cluster 4 x 256
    ("SSRN", "HC_8"),                 # hc 512 at the upsampled length
    ("SSRN", "HC_11"),                # hc 1024: cluster 8 x 256
    ("SSRN", "D_4"),                  # transposed conv: two k-taps, zero second half on tap 1
    ("SSRN", "C_13"),                 # C 1024 -> 1025: cluster 8 x 144 columns (the last CTA mostly padding)
    ("SSRN", "C_14"),                 # relu C 1025 -> 1025: K tail of one channel
    ("Text2Mel/AudioDec", "C_11"),    # C 256 -> 80: one CTA of 80 columns
    ("Text2Mel/AudioEnc", "C_2"),     # relu C 256 -> 256: cluster 4 x 64 columns
]
LENGTHS = [1, 127, 128, 129, 210, 420, 840]


@pytest.mark.parametrize("L", LENGTHS)
@pytest.mark.parametrize("net,scope", KINDS, ids=[n.split("/")[-1] + "/" + s for n, s in KINDS])
def test_block_full_lengths(tc, params, net, scope, L):
    """One utterance at ragged and exact tile lengths: oracle and fp32 kernels."""
    x = _input(net, scope, 1, L)
    out, out32 = _both_paths(tc, net, scope, x)
    ref = _oracle(params, net, scope, x)
    assert out.shape == ref.shape
    assert np.abs(out - ref).max() < BLOCK_TOL
    assert np.abs(out - out32).max() < PATH_TOL


@pytest.mark.parametrize("L", [129, 420])
@pytest.mark.parametrize("net,scope", KINDS, ids=[n.split("/")[-1] + "/" + s for n, s in KINDS])
def test_block_full_batch3(tc, params, net, scope, L):
    """Three utterances: tiles of different utterances side by side in one launch, below one wave."""
    x = _input(net, scope, 3, L)
    out, out32 = _both_paths(tc, net, scope, x)
    assert np.abs(out - _oracle(params, net, scope, x)).max() < BLOCK_TOL
    assert np.abs(out - out32).max() < PATH_TOL


WIDE = [("SSRN", "HC_11", 840), ("SSRN", "C_14", 840), ("SSRN", "D_7", 420), ("Text2Mel/TextEnc", "HC_4", hp.max_N)]


@pytest.mark.parametrize("net,scope,L", WIDE, ids=[s for _, s, _ in WIDE])
def test_block_full_batch32(tc, params, net, scope, L):
    """B = 32: many times more clusters than fit on the device at once.  Every row against the fp32 kernels, the first and
    the last utterance against the oracle."""
    x = _input(net, scope, 32, L)
    out, out32 = _both_paths(tc, net, scope, x)
    assert np.abs(out - out32).max() < PATH_TOL
    sel = [0, 31]
    assert np.abs(out[sel] - _oracle(params, net, scope, x[sel])).max() < BLOCK_TOL


OPTION_SETS = [dict(tc_occ2=1), dict(tc_mcast=0), dict(tc_resid_tma=0), dict(tc_occ2=1, tc_mcast=0, tc_resid_tma=0),
               dict(tc_occ2=0, tc_mcast=0, tc_resid_tma=0)]


@pytest.mark.parametrize("variant", OPTION_SETS, ids=lambda v: "+".join("%s=%d" % kv for kv in v.items()))
@pytest.mark.parametrize("net,scope,B,L", [("SSRN", "HC_11", 3, 840), ("SSRN", "C_13", 32, 840), ("SSRN", "D_7", 32, 420),
                                           ("SSRN", "HC_8", 1, 129)], ids=["HC_11-B3", "C_13-B32", "D_7-B32", "HC_8-B1"])
def test_block_full_options(tc, params, net, scope, B, L, variant):
    """Each option value on narrow and wide grids: the same results as the default path and the fp32 kernels."""
    x = _input(net, scope, B, L)
    base = _run(tc, net, scope, x).cpu().numpy()
    for k, v in variant.items():
        tc.set_option(k, v)
    out, out32 = _both_paths(tc, net, scope, x)
    assert np.abs(out - base).max() < PATH_TOL
    assert np.abs(out - out32).max() < PATH_TOL
    assert np.abs(out[:1] - _oracle(params, net, scope, x[:1])).max() < BLOCK_TOL


@pytest.mark.parametrize("B,T", [(3, 33), (32, hp.max_T)])
def test_ssrn_chain_full(tc, params, B, T):
    """The whole SSRN on the tensor path, ending in the sigmoid block, against the fp32 kernels (and the oracle on the
    first utterance)."""
    Y = np.random.default_rng(B * 1000 + T).uniform(0, 1, (B, T, hp.n_mels)).astype(np.float32)
    _, Z = tc.ssrn(Y, want_logits=False)
    tc.set_tensor_path(0)
    try:
        _, Z32 = tc.ssrn(Y, want_logits=False)
    finally:
        tc.set_tensor_path(1)
    assert (Z - Z32).abs().max().item() < PATH_TOL
    _, Zr = rt.SSRN(params, torch.from_numpy(Y[:1]))
    assert np.abs(Z[:1].cpu().numpy() - Zr.numpy()).max() < 1e-3
