"""GPU parity tests of the wgmma (tensor-core, split-fp16 3-MMA) path against the oracle
and against the fp32 CUDA-core path.  Same tolerances as the fp32 path: the split-plane
arithmetic is fp32-grade (|err| ~ 1e-5), which is what makes the tensor pipe usable under
the 1e-3 parity budget at all."""
import zlib

import numpy as np
import pytest
import torch

from dc_tts_b200 import arch
from dc_tts_b200.hyperparams import Hyperparams as hp
from dc_tts_b200.params import synthetic_text
from oracle import ref_torch as rt

pytestmark = pytest.mark.gpu
BLOCK_TOL = 2e-4
NET_TOL = 1e-3


@pytest.fixture()
def tc(engine):
    engine.set_tensor_path(1)
    yield engine
    engine.set_tensor_path(0)


def _rand(shape, seed, lo=-1.0, hi=1.0):
    return np.random.default_rng(seed).uniform(lo, hi, shape).astype(np.float32)


def _layer(net, scope):
    return [l for l in arch.NETWORKS[net]() if l.scope == scope][0]


CASES = [
    # net, scope, B, L
    ("Text2Mel/AudioEnc", "HC_4", 1, 128),       # cluster 2, one full tile
    ("Text2Mel/AudioEnc", "HC_7", 2, 210),       # dilation 27, causal, ragged last tile
    ("Text2Mel/TextEnc", "HC_6", 2, 180),        # cluster 4, SAME padding, dilation 9
    ("Text2Mel/TextEnc", "HC_15", 1, 50),        # k=1 highway
    ("SSRN", "HC_11", 1, 300),                   # cluster 8, C=1024
    ("Text2Mel/TextEnc", "C_2", 2, 180),         # conv1d 128->512 relu, cluster 2
    ("Text2Mel/AudioEnc", "C_1", 3, 210),        # K=80 (partial k-block), 256 cols, 1 CTA
    ("Text2Mel/AudioDec", "C_1", 2, 85),
    ("Text2Mel/AudioDec", "C_11", 2, 210),       # 80 columns
    ("SSRN", "C_10", 1, 200),                    # 512 -> 1024, cluster 4
    ("SSRN", "C_13", 1, 70),                     # 1024 -> 1025, cluster 8 x 144 columns
    ("SSRN", "C_15", 1, 130),                    # 1025 -> 1025 (K tail of 1), relu
    ("SSRN", "D_4", 2, 210),                     # transposed conv
    ("SSRN", "D_7", 1, 3),
]


@pytest.mark.parametrize("net,scope,B,L", CASES)
def test_block_tensor_path(tc, params, net, scope, B, L):
    l = _layer(net, scope)
    full = net + "/" + scope
    x = _rand((B, L, l.cin), zlib.crc32(full.encode()) % 1000 + L)
    xt = torch.from_numpy(x)
    if l.kind == "C":
        out = tc.conv1d(full, x, l.cout, l.rate, l.pad == "CAUSAL", 1 if l.act == "relu" else 0)
        ref = rt.conv1d(params, xt, full, l.rate, l.pad, l.act)
    elif l.kind == "HC":
        out = tc.hc(full, x, l.rate, l.pad == "CAUSAL")
        ref = rt.hc(params, xt, full, l.rate, l.pad)
    else:
        out = tc.conv1d_transpose(full, x)
        ref = rt.conv1d_transpose(params, xt, full)
    err = np.abs(out.cpu().numpy() - ref.numpy()).max()
    assert out.shape == ref.shape
    assert err < BLOCK_TOL, err


def test_networks_tensor_path(tc, params):
    L = synthetic_text(3, 70, seed=5)
    K, V = tc.textenc(L)
    Kr, Vr = rt.TextEnc(params, L)
    assert np.abs(K.cpu().numpy() - Kr.numpy()).max() < NET_TOL
    assert np.abs(V.cpu().numpy() - Vr.numpy()).max() < NET_TOL
    S = _rand((2, hp.max_T, hp.n_mels), 9, 0, 1)
    Q = tc.audioenc(S)
    assert np.abs(Q.cpu().numpy() - rt.AudioEnc(params, torch.from_numpy(S)).numpy()).max() < NET_TOL
    R = _rand((2, hp.max_T, 2 * hp.d), 10)
    logits, Y = tc.audiodec(R)
    lr, Yr = rt.AudioDec(params, torch.from_numpy(R))
    assert np.abs(Y.cpu().numpy() - Yr.numpy()).max() < NET_TOL
    assert np.abs(logits.cpu().numpy() - lr.numpy()).max() < NET_TOL


@pytest.mark.parametrize("B,T", [(1, 12), (2, 210)])
def test_ssrn_tensor_path(tc, params, B, T):
    Y = _rand((B, T, hp.n_mels), 12, 0, 1)
    logits, Z = tc.ssrn(Y)
    lr, Zr = rt.SSRN(params, torch.from_numpy(Y))
    assert np.abs(Z.cpu().numpy() - Zr.numpy()).max() < NET_TOL
    assert np.abs(logits.cpu().numpy() - lr.numpy()).max() < 5e-3
    _, Z2 = tc.ssrn(Y, want_logits=False)
    assert torch.equal(Z, Z2)


def test_tensor_path_close_to_fp32_path(engine):
    Y = _rand((1, 60, hp.n_mels), 3, 0, 1)
    engine.set_tensor_path(0)
    _, Z0 = engine.ssrn(Y, want_logits=False)
    engine.set_tensor_path(1)
    try:
        _, Z1 = engine.ssrn(Y, want_logits=False)
    finally:
        engine.set_tensor_path(0)
    assert (Z0 - Z1).abs().max().item() < 1e-4


@pytest.mark.parametrize("decode_mode", [0, 1], ids=["graph", "cluster"])
def test_generate_tensor_pyramid_vs_oracle(tc, params, decode_mode):
    """graph decode: B >= 8 moves the 85..59-row AudioDec pyramid of every AR step onto wgmma (windowed
    128-row tiles ending at row j); free-running 40 steps against the oracle's literal schedule."""
    tc.set_option("decode_mode", decode_mode)
    L = np.concatenate([synthetic_text(1, 40 + 15 * i, seed=60 + i) for i in range(8)])
    steps = 40
    r = rt.synthesize(params, L, steps=steps, literal=False, record=True)
    Y, P, _, _ = tc.text2mel_generate(L, steps=steps)
    Yo, Po = r["Y"].numpy(), r["p_hist"].numpy()
    ok = r["margin_hist"].numpy().min(1) > 1e-4
    assert ok.sum() >= 6
    assert np.array_equal(P.cpu().numpy()[ok, :steps], Po[ok])
    assert np.abs(Y.cpu().numpy()[ok] - Yo[ok]).max() < NET_TOL
    # and the same loop on the fp32 kernels
    tc.set_tensor_path(0)
    Y0, P0, _, _ = tc.text2mel_generate(L, steps=steps)
    tc.set_tensor_path(1)
    tc.set_option("decode_mode", 1)
    assert torch.equal(P0[ok], P[ok]) and (Y0[ok] - Y[ok]).abs().max().item() < 1e-4
