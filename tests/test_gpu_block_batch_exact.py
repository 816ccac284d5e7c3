"""The fused conv + LayerNorm block kernel computes each output row from that row's own accumulators: an utterance's
output in a batch is bit for bit its output alone, whatever its neighbours hold and however many tiles and waves the
launch has.  The batches alternate utterances at very different levels (1e-8, O(1), 1e2), so that statistics or staged
tiles taken from the wrong row would show.

The single-block calls cover every block kind (conv1d, hc, transposed conv) at every accumulator width per CTA the
networks use (64, 80, 144, 256 columns); they write fp32 outputs, and their hidden-block inputs are not scaled per
utterance.  The SSRN chain covers the split-plane outputs between blocks (the quad-transposed 16-byte stores of conv1d
and transposed blocks, the TMA-staged output of hc blocks) and the per-utterance input scale of its first block."""
import numpy as np
import pytest
import torch

from dc_tts_b200 import arch

pytestmark = pytest.mark.gpu

# (network, scope): kind, accumulator columns per CTA
BLOCKS = [
    ("Text2Mel/AudioEnc", "C_2"),      # conv1d, 64
    ("Text2Mel/AudioDec", "C_11"),     # conv1d, 80
    ("SSRN", "C_14"),                  # conv1d, 144 (clusters of 8)
    ("SSRN", "C_10"),                  # conv1d, 256
    ("Text2Mel/AudioEnc", "HC_4"),     # hc, 64 (32 + 32)
    ("SSRN", "HC_11"),                 # hc, 256 (128 + 128), clusters of 8
    ("SSRN", "D_4"),                   # transposed conv, 256
]
LEVELS = [1e-8, 1.0, 1e2]
# (utterances, length): one tile each; a ragged last tile; many tiles per utterance over several waves
SHAPES = [(3, 128), (5, 300), (24, 600)]


@pytest.fixture()
def tc(engine):
    engine.set_tensor_path(1)
    yield engine
    engine.set_tensor_path(1)


def _run(eng, net, scope, x):
    l = [l for l in arch.NETWORKS[net]() if l.scope == scope][0]
    full = net + "/" + scope
    if l.kind == "C":
        return eng.conv1d(full, x, l.cout, l.rate, l.pad == "CAUSAL", 1 if l.act == "relu" else 0)
    if l.kind == "HC":
        return eng.hc(full, x, l.rate, l.pad == "CAUSAL")
    return eng.conv1d_transpose(full, x)


@pytest.mark.parametrize("B,L", SHAPES)
@pytest.mark.parametrize("net,scope", BLOCKS)
def test_batch_rows_equal_each_utterance_alone(tc, net, scope, B, L):
    l = [l for l in arch.NETWORKS[net]() if l.scope == scope][0]
    rng = np.random.default_rng(B * 1000 + L)
    x = rng.standard_normal((B, L, l.cin)).astype(np.float32)
    x *= np.array([LEVELS[b % len(LEVELS)] for b in range(B)], dtype=np.float32)[:, None, None]
    xd = torch.from_numpy(x).cuda()
    batch = _run(tc, net, scope, xd).cpu().numpy()
    assert np.isfinite(batch).all()
    for b in range(B):
        alone = _run(tc, net, scope, xd[b:b + 1].contiguous()).cpu().numpy()[0]
        assert np.array_equal(batch[b], alone), (scope, B, L, b, float(np.abs(batch[b] - alone).max()))


@pytest.mark.parametrize("B", [7, 24])
def test_ssrn_batch_equals_each_utterance_alone(tc, B):
    from dc_tts_b200.hyperparams import Hyperparams as hp
    T = 210
    rng = np.random.default_rng(B)
    Y = rng.uniform(0, 1, (B, T, hp.n_mels)).astype(np.float32)
    Y *= np.array([LEVELS[b % len(LEVELS)] for b in range(B)], dtype=np.float32)[:, None, None]
    Yd = torch.from_numpy(Y).cuda()
    lg, Z = tc.ssrn(Yd)
    lg, Z = lg.cpu().numpy(), Z.cpu().numpy()
    assert np.isfinite(Z).all()
    for b in range(B):
        lg1, Z1 = tc.ssrn(Yd[b:b + 1].contiguous())
        assert np.array_equal(Z[b], Z1.cpu().numpy()[0]), (B, b)
        assert np.array_equal(lg[b], lg1.cpu().numpy()[0]), (B, b)
