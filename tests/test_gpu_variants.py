"""Every kernel variant that dctts_set_option can select is a parity-tested code path (round 1 selected them with
environment variables that froze at first use and had no test): the two-stage ring, unicast activation tiles, the non-TMA
residual path, the fused GEMM + LN decode launch."""
import numpy as np
import pytest
import torch

from dc_tts_b200.hyperparams import Hyperparams as hp
from dc_tts_b200.params import synthetic_text
from oracle import ref_torch as rt

pytestmark = pytest.mark.gpu
BLOCK_TOL = 2e-4
DEFAULTS = dict(tc_occ2=1, tc_mcast=1, tc_resid_tma=1, fused_ln=0, decode_mode=1)


@pytest.fixture()
def tc(engine):
    engine.set_tensor_path(1)
    yield engine
    for k, v in DEFAULTS.items():
        engine.set_option(k, v)
    engine.set_tensor_path(1)


@pytest.fixture(scope="module")
def hc11_case(params):
    """SSRN/HC_11 (C = 1024, cluster 8) on 11 x 840 rows: 77 tiles x 8 CTAs = 616 CTAs, more than the SMs of the device,
    so every variant (including the two-stage ring) is eligible; one oracle evaluation for all."""
    x = np.random.default_rng(5).uniform(-1, 1, (11, 840, 1024)).astype(np.float32)
    with torch.no_grad():
        ref = rt.hc(params, torch.from_numpy(x), "SSRN/HC_11", 1, "SAME").numpy()
    return x, ref


VARIANTS = [dict(), dict(tc_occ2=0), dict(tc_mcast=0), dict(tc_resid_tma=0), dict(tc_occ2=0, tc_mcast=0, tc_resid_tma=0)]


@pytest.mark.parametrize("variant", VARIANTS, ids=lambda v: "+".join("%s=%d" % kv for kv in v.items()) or "default")
def test_hc11_variants(tc, hc11_case, variant):
    x, ref = hc11_case
    for k, v in variant.items():
        tc.set_option(k, v)
        assert tc.get_option(k) == v
    out = tc.hc("SSRN/HC_11", x, 1, False).cpu().numpy()
    assert np.abs(out - ref).max() < BLOCK_TOL


@pytest.mark.parametrize("variant", [dict(), dict(tc_occ2=0)], ids=["default", "occ1"])
def test_deconv_and_c512_variants(tc, params, variant):
    """transposed conv (mode 2) and a C = 512 hc block under both ring depths: D_7 at (24, 420), HC_8 at (24, 840)."""
    for k, v in variant.items():
        tc.set_option(k, v)
    x = np.random.default_rng(6).uniform(-1, 1, (24, 420, 512)).astype(np.float32)
    out = tc.conv1d_transpose("SSRN/D_7", x).cpu().numpy()
    with torch.no_grad():
        ref = rt.conv1d_transpose(params, torch.from_numpy(x), "SSRN/D_7").numpy()
    assert np.abs(out - ref).max() < BLOCK_TOL
    x2 = ref[:, :840]                                    # a realistic activation: the block that follows D_7
    out2 = tc.hc("SSRN/HC_8", x2, 1, False).cpu().numpy()
    with torch.no_grad():
        ref2 = rt.hc(params, torch.from_numpy(x2), "SSRN/HC_8", 1, "SAME").numpy()
    assert np.abs(out2 - ref2).max() < BLOCK_TOL


def test_options_reject_garbage(tc):
    from dc_tts_b200.engine import DcttsError
    with pytest.raises(DcttsError):
        tc.set_option("no_such_option", 1)
    with pytest.raises(DcttsError):
        tc.set_option("tc_mcast", 7)
    with pytest.raises(DcttsError):
        tc.set_option("tc_cg2", 1)                       # CTA pairs need a two-CTA MMA, which sm_90 does not have
    assert tc.get_option("decode_available") == 1


def test_graph_decode_fused_ln_variant(tc, params):
    """graph-per-frame decode with GEMM + LN fused in one launch: same windows, same mels as the two-launch form."""
    L = synthetic_text(2, 70, seed=77)
    tc.set_option("decode_mode", 0)
    Y0, P0, _, _ = tc.text2mel_generate(L, steps=25)
    tc.set_option("fused_ln", 1)
    Y1, P1, _, _ = tc.text2mel_generate(L, steps=25)
    assert torch.equal(P0, P1) and (Y0 - Y1).abs().max().item() < 1e-5
