"""SSRN at the linear-spectrogram widths of the other corpus rates: F = 513 (16 kHz, n_fft 1024) and F = 2049 (44.1 and
48 kHz, n_fft 4096).  The last four blocks (C_13 .. C_16) are F channels wide.  On the tensor path they run the wgmma
block kernel (4 CTAs x 144 columns at F = 513, a 16-CTA cluster of it at F = 2049), on the fp32 path the 2080-channel
LayerNorm kernel; the trainer's backward at F = 2049 runs the conv1d-only 2080-channel block-backward kernel.

Engines are built inside `at_rate`, which patches Hyperparams (sr, n_fft, hop_length, win_length), so that
init_params, the oracles and the engine agree on F."""
import numpy as np
import pytest
import torch

from dc_tts_b200 import arch
from dc_tts_b200.engine import DcttsError
from dc_tts_b200.params import init_params
from oracle import ref_torch as rt
from oracle import ref_train as rtr

from sample_rates import at_rate
from test_train import _compare_grads

pytestmark = pytest.mark.gpu
NET_TOL = 1e-3
SIZES = {513: 16000, 2049: 44100}
_ERR = {}


@pytest.fixture(scope="module")
def nets():
    """{F: (engine, params)} for both widths."""
    from dc_tts_b200.engine import Engine
    out = {}
    for F, sr in SIZES.items():
        with at_rate(sr) as H:
            P = init_params(0, "perturbed")
            e = Engine(0, hparams=H)
            e.load_params(P)
            out[F] = (e, P)
    yield out
    print("\nSSRN at other widths, max |dZ| against the oracle: " +
          ", ".join("F=%d %s B=%d T=%d %.2e" % (k + (v,)) for k, v in sorted(_ERR.items())))
    for e, _ in out.values():
        e.close()


_REF = {}


def _oracle(F, P, B, T):
    if (F, B, T) not in _REF:
        Y = np.random.default_rng(B * 1000 + T).uniform(0, 1, (B, T, 80)).astype(np.float32)
        with at_rate(SIZES[F]):
            with torch.no_grad():
                lr, Zr = rt.SSRN(P, torch.from_numpy(Y))
        _REF[(F, B, T)] = (Y, lr.numpy(), Zr.numpy())
    return _REF[(F, B, T)]


@pytest.mark.parametrize("F", sorted(SIZES))
@pytest.mark.parametrize("path", ["tc", "fp32"])
@pytest.mark.parametrize("B,T", [(1, 9), (3, 210), (32, 9), (32, 210), (1, 210), (3, 9)])
def test_ssrn_vs_oracle(nets, F, path, B, T):
    e, P = nets[F]
    Y, lr, Zr = _oracle(F, P, B, T)
    e.set_tensor_path(1 if path == "tc" else 0)
    try:
        if path == "tc":
            # every SSRN block, the F-wide ones included, has a wgmma kernel: no silent drop to the fp32 kernels
            assert e.get_option("ssrn_tc_available") == 1
        logits, Z = e.ssrn(Y)
    finally:
        e.set_tensor_path(0)
    assert tuple(Z.shape) == (B, 4 * T, F)
    err = float(np.abs(Z.cpu().numpy() - Zr).max())
    _ERR[(F, path, B, T)] = err
    assert err < NET_TOL, err
    assert np.abs(logits.cpu().numpy() - lr).max() < 5e-3


def _relu_clear(P):
    """SSRN's ReLU blocks (C_14, C_15) pushed clear of zero (LayerNorm beta += 8): a pre-activation within the forward
    noise of zero may flip its mask between two correct float32 passes (test_train.py, _RELU_TIE)."""
    P = dict(P)
    for l in arch.ssrn_layers():
        if l.kind == "C" and l.act == "relu":
            n = "SSRN/%s/normalize/beta" % l.scope
            P[n] = (np.asarray(P[n], np.float32) + 8.0).astype(np.float32)
    return P


def _l1_clear(P, mels, mags, seed, rate):
    """The targets moved 1e-3 away wherever the oracle's Z lies within 1e-4 of them.  The L1 loss is discontinuous in
    sign(Z - mags) as ReLU is in its pre-activation: at F = 2049 this batch has |Z - mags| = 3e-8 at one element, within
    the split-fp16 forward's noise, and that one flipped sign moves C_16's gradients by 1.7e-2 of their max-norm."""
    W = {n: torch.tensor(np.asarray(P[n], np.float32)) for n in rtr.ssrn_names()}
    with torch.no_grad():
        Z = rtr.forward_ssrn(W, mels, mags, seed, rate)["Z"].numpy()
    near = np.abs(Z - mags) < 1e-4
    mags = mags.copy()
    mags[near] = np.where(Z[near] > 0.5, Z[near] - 1e-3, Z[near] + 1e-3)
    assert np.abs(Z - mags).min() > 5e-5
    return mags


@pytest.mark.parametrize("F", sorted(SIZES))
@pytest.mark.parametrize("tc", [7, 0])
def test_ssrn_train_step_vs_oracle(F, tc):
    from dc_tts_b200.engine import Engine
    B, T, rate, seed = 2, 12, 0.05, 9
    with at_rate(SIZES[F]) as H:
        P = _relu_clear(init_params(0, "perturbed"))
        eng = Engine(0, hparams=H)
        eng.load_params(P)
        eng.set_option("train_tc", tc)
        eng.train_init_ssrn(B, T, rate)
        mels = np.random.default_rng(3).uniform(0, 1, (B, T, 80)).astype(np.float32)
        mags = np.random.default_rng(4).uniform(0, 1, (B, 4 * T, F)).astype(np.float32)
        mags = _l1_clear(P, mels, mags, seed, rate)
        newP, st, info = rtr.train_step_ssrn(P, mels, mags, global_step=3999, seed=seed, rate=rate)
        out = eng.train_step_ssrn(mels, mags, global_step=3999, seed=seed, apply=False)
        for k in ("loss", "loss_mags", "loss_bd2"):
            assert abs(out[k] - info[k]) <= 1e-5 * max(1.0, abs(info[k])), (k, out[k], info[k])
        assert len(info["grads"]) == 80
        worst = _compare_grads(eng, info["grads"])
        print("F=%d train_tc=%d: worst gradient error / max-norm %.2e" % (F, tc, worst))
        eng.train_apply(3999)
        for n in ("SSRN/C_13/conv1d/kernel", "SSRN/C_14/conv1d/kernel", "SSRN/C_16/conv1d/bias", "SSRN/C_15/normalize/gamma",
                  "SSRN/C_16/normalize/beta", "SSRN/HC_12/conv1d/kernel", "SSRN/D_4/conv2d_transpose/kernel"):
            m, v = st[n]
            np.testing.assert_allclose(eng.train_tensor(n, "m"), m, rtol=2e-3, atol=max(1e-9, 1e-4 * np.abs(m).max()))
            np.testing.assert_allclose(eng.train_tensor(n, "v"), v, rtol=4e-3, atol=max(1e-14, 4e-4 * np.abs(v).max()))
            step = np.abs(newP[n] - P[n]).max()
            assert np.abs(eng.train_tensor(n, "param") - newP[n]).max() <= 0.05 * step + 2.4e-7, n
        eng.close()


def test_ssrn_wider_than_the_layernorm_kernels_is_refused():
    """n_fft = 8192 makes the F-wide blocks 4097 channels: past the widest LayerNorm kernel (2080) and any wgmma cluster.
    The call fails with a message instead of returning Z with channels that were never written."""
    from dc_tts_b200.engine import Engine
    with at_rate(44100, 8192) as H:
        P = init_params(0, "perturbed")
        e = Engine(0, hparams=H)
        e.load_params(P)
        assert e.get_option("ssrn_tc_available") == 0
        Y = np.random.default_rng(0).uniform(0, 1, (1, 5, 80)).astype(np.float32)
        for path in (1, 0):
            e.set_tensor_path(path)
            with pytest.raises(DcttsError, match="2080"):
                e.ssrn(Y)
        e.close()
