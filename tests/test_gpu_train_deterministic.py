"""The training step with the option "train_deterministic" (include/dctts.h): every sum of the step in a fixed order, so that
the same variables, Adam moments, global step, batch, seed, lr, dropout rate and kernel set give the same bits.

  repeatable        two handles, 3 steps each: variables, m, v, the gradient arena and the losses bit for bit, Text2Mel and
                    SSRN (F = 513, 1025, 2049), on train_tc 7, 0 and a mixed mask, and across workspace capacities
  history           evaluations, synthesis from the trained weights, apply = 0 + train_apply and a reserve in between leave
                    the next steps' bits unchanged
  resume            trainer.train(deterministic=True) stopped at step 10 and resumed writes the step-20 bundle of a straight run
  parity            the oracle comparisons of tests/test_train.py and tests/test_train_bucketed.py at their tolerances
  one launch        conv_gemm mode 1 (both kernel sets, split > 1), block_bwd (every MAXV), train_loss and attn_bwd against
                    the float64 references of tests/ref_train_kernels.py, twice from the same inputs with identical bits
  compile           ptxas: no stack and no spills in kernels_ordered.cu
"""
import itertools
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from dc_tts_b200 import build, trainer
from dc_tts_b200.hyperparams import Hyperparams as hp
from dc_tts_b200.params import init_params, synthetic_bucket

import ref_train_kernels as rk
from sample_rates import at_rate

RATE = 0.05
# the tolerances of the one-launch checks (tests/test_gpu_train_kernels.py's, for the same references)
TAU = {"block": 1e-6, "block_sum": 6e-5, "attn": 6e-6, "loss": 8e-7}


def _engine(P, tc, hparams=hp, deterministic=1):
    from dc_tts_b200.engine import Engine
    e = Engine(0, hparams=hparams)
    e.load_params(P)
    e.set_option("train_tc", tc)
    e.set_option("train_deterministic", deterministic)
    return e


def _names(scope):
    from dc_tts_b200.arch import param_shapes
    return [n for n in param_shapes() if n.startswith(scope + "/")]


def _state(eng, names):
    s = {(n, w): eng.train_tensor(n, w) for n in names for w in ("param", "m", "v")}
    s["grads"] = eng.train_grads().cpu().numpy()
    return s


def _differ(x, y):
    return sorted(str(k) for k in x if not np.array_equal(x[k], y[k]))


def _t2m_batches(B, N, T, n=3):
    return [synthetic_bucket(B, N, T, seed=i) for i in range(n)]


def _ssrn_batches(B, T, F, n=3):
    out = []
    for i in range(n):
        rng = np.random.default_rng([i, T, F])
        out.append((rng.uniform(0, 1, (B, T, hp.n_mels)).astype(np.float32), rng.uniform(0, 1, (B, 4 * T, F)).astype(np.float32)))
    return out


def _run_t2m(eng, batches, gs0=0):
    return [eng.train_step(L, m, global_step=gs0 + i, seed=gs0 + i) for i, (L, m) in enumerate(batches)]


def _run_ssrn(eng, batches, gs0=0):
    return [eng.train_step_ssrn(m, g, global_step=gs0 + i, seed=gs0 + i) for i, (m, g) in enumerate(batches)]


# ============================================================================================= repeatable
@pytest.mark.gpu
@pytest.mark.parametrize("B,N,T,tc", [(32, 180, 210, 7), (32, 123, 171, 7), (2, 37, 53, 7), (2, 37, 53, 0), (2, 37, 53, 5),
                                      (32, 123, 171, 0)])
def test_text2mel_steps_repeat_bit_for_bit(B, N, T, tc):
    P = init_params(0, "perturbed")
    batches = _t2m_batches(B, N, T)
    names = _names("Text2Mel")
    runs = []
    for _ in range(2):
        e = _engine(P, tc)
        e.train_init(B, RATE)
        losses = _run_t2m(e, batches)
        runs.append((losses, _state(e, names)))
        e.close()
    assert runs[0][0] == runs[1][0]
    assert _differ(runs[0][1], runs[1][1]) == []


@pytest.mark.gpu
def test_text2mel_steps_do_not_depend_on_the_capacity():
    """(2, 197, 230), past (max_N, max_T): a handle grown in place by the trainer's "grow" against one reserved before step 1"""
    B, N, T = 2, 197, 230
    P = init_params(0, "perturbed")
    batches = _t2m_batches(B, N, T)
    names = _names("Text2Mel")
    a, b = _engine(P, 7), _engine(P, 7)
    a.train_init(B, RATE); b.train_init(B, RATE)
    b.train_reserve(320, 320)
    capa = trainer.Capacity(1, hp, "grow", None)
    capa.initialised(a)
    outs = []
    for i, (L, m) in enumerate(batches):
        assert capa.admit(L, m, lambda s: None)
        capa.prepare(a, L, m, lambda s: None)
        outs.append((a.train_step(L, m, global_step=i, seed=i), b.train_step(L, m, global_step=i, seed=i)))
    assert a.train_capacity() != b.train_capacity()
    assert all(x == y for x, y in outs)
    assert _differ(_state(a, names), _state(b, names)) == []
    a.close(); b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("F,sr,tc", [(1025, hp.sr, 7), (1025, hp.sr, 0), (513, 16000, 7), (2049, 44100, 7)])
def test_ssrn_steps_repeat_bit_for_bit(F, sr, tc):
    B, T = (8, 210) if F == 1025 else (2, 53)
    with at_rate(sr) as H:
        P = init_params(0, "perturbed")
        batches = _ssrn_batches(B, T, F)
        names = _names("SSRN")
        runs = []
        for _ in range(2):
            e = _engine(P, tc, H)
            e.train_init_ssrn(B, hp.max_T, RATE)
            losses = _run_ssrn(e, batches)
            runs.append((losses, _state(e, names)))
            e.close()
    assert runs[0][0] == runs[1][0]
    assert _differ(runs[0][1], runs[1][1]) == []


# ============================================================================================= history
@pytest.mark.gpu
def test_history_does_not_change_the_bits():
    B, N, T = 4, 101, 149
    P = init_params(0, "perturbed")
    batches = _t2m_batches(B, N, T, n=4)
    names = _names("Text2Mel")
    a, b = _engine(P, 7), _engine(P, 7)
    a.train_init(B, RATE); b.train_init(B, RATE)
    L0, m0 = batches[0]
    a.train_eval(L0, m0, seed=123)
    a.train_step(L0, m0, global_step=0, seed=0)
    a.refresh_synthesis()
    Lt = torch.from_numpy(L0[:, :hp.max_N] if L0.shape[1] >= hp.max_N else np.pad(L0, ((0, 0), (0, hp.max_N - L0.shape[1])))).cuda()
    Y, _, lengths = a.text2mel_generate_until(Lt, steps=24)[:3]
    a.ssrn(Y, want_logits=False, lengths=lengths)
    torch.cuda.synchronize()
    a.train_step(*batches[1], global_step=1, seed=1, apply=False)
    a.train_eval(*batches[2], seed=7)
    a.train_apply(1)
    a.train_reserve(192, 256)
    a.train_step(*batches[2], global_step=2, seed=2)
    la = a.train_step(*batches[3], global_step=3, seed=3)
    lb = _run_t2m(b, batches)[-1]
    assert la == lb
    assert _differ(_state(a, names), _state(b, names)) == []
    a.close(); b.close()


# ============================================================================================= resume
def _write_dataset(root, n=12, seed=0):
    rng = np.random.default_rng(seed)
    d = root / "LJSpeech-1.0"
    (d / "wavs").mkdir(parents=True)
    (root / "mels").mkdir(); (root / "mags").mkdir()
    F = 1 + hp.n_fft // 2
    lines = []
    for i in range(n):
        text = "".join(rng.choice(list("abcdefghijklmnopqrstuvwxyz '"), int(rng.integers(20, 60))))
        lines.append("LJ%03d|raw|%s" % (i, text))
        T = int(rng.integers(30, 90))
        np.save(root / "mels" / ("LJ%03d.npy" % i), rng.uniform(0, 1, (T, hp.n_mels)).astype(np.float32))
        np.save(root / "mags" / ("LJ%03d.npy" % i), rng.uniform(0, 1, (T * hp.r, F)).astype(np.float32))
    (d / "transcript.csv").write_text("\n".join(lines) + "\n", encoding="utf-8")
    return str(d)


@pytest.mark.gpu
@pytest.mark.parametrize("num", [1, 2])
def test_resumed_run_writes_the_same_bundle(tmp_path, num):
    from dc_tts_b200.checkpoint import latest_checkpoint, list_variables, load_checkpoint
    from dc_tts_b200.engine import Engine
    d = _write_dataset(tmp_path)
    fpaths, _, texts = trainer.load_train_data(d)
    loader = lambda p: trainer._load_spectrograms_npy(p, str(tmp_path / "mels"), str(tmp_path / "mags"))  # noqa: E731
    P = init_params(1)

    def batches(skip=0):
        return itertools.islice(trainer.fixed_size_batches(fpaths, texts, B=4, seed=0, loader=loader), skip, None)

    def run(logdir, num_iterations, skip=0):
        e = Engine(0)
        e.load_params(P)
        gs = trainer.train(num, e, batches(skip), num_iterations=num_iterations, logdir=logdir, save_every=10,
                           log=lambda s: None, deterministic=True)
        e.close()
        return gs

    straight, split = str(tmp_path / "straight"), str(tmp_path / "split")
    assert run(straight, 19) == 20
    assert run(split, 9) == 10
    assert run(split, 19, skip=10) == 20                     # resumed from model_gs_... at step 10
    a, b = latest_checkpoint(straight), latest_checkpoint(split)
    names = sorted(n for n, _, _ in list_variables(a))
    assert names == sorted(n for n, _, _ in list_variables(b))
    ta, tb = load_checkpoint(a, names), load_checkpoint(b, names)
    assert int(ta["gs/global_step"]) == 20
    assert [n for n in names if not np.array_equal(ta[n], tb[n])] == []


# ============================================================================================= parity with the oracle
# The oracle comparisons of tests/test_train.py and tests/test_train_bucketed.py with the option on, at their tolerances:
# the losses to 1e-5, every gradient tensor to 2e-3 of its own max-norm (_compare_grads), and after train_apply m, v and
# the parameters of the tensors those files check.
T2M_CHECKED = ("Text2Mel/TextEnc/embed_1/lookup_table", "Text2Mel/TextEnc/HC_7/conv1d/kernel", "Text2Mel/AudioEnc/C_1/conv1d/kernel",
               "Text2Mel/AudioDec/HC_3/H2/gamma", "Text2Mel/AudioDec/C_11/conv1d/bias", "Text2Mel/AudioEnc/HC_9/H1/beta")
SSRN_CHECKED = ("SSRN/D_4/conv2d_transpose/kernel", "SSRN/D_7/conv2d_transpose/bias", "SSRN/HC_12/conv1d/kernel", "SSRN/C_13/conv1d/kernel",
                "SSRN/C_16/conv1d/bias", "SSRN/C_15/normalize/gamma", "SSRN/HC_2/H1/beta")


def _check_update(eng, P, newP, st, names, check_v=True):
    for n in names:
        m, v = st[n]
        np.testing.assert_allclose(eng.train_tensor(n, "m"), m, rtol=2e-3, atol=max(1e-9, 1e-4 * np.abs(m).max()))
        if check_v:
            np.testing.assert_allclose(eng.train_tensor(n, "v"), v, rtol=4e-3, atol=max(1e-14, 4e-4 * np.abs(v).max()))
        step = np.abs(newP[n] - P[n]).max()
        assert np.abs(eng.train_tensor(n, "param") - newP[n]).max() <= 0.05 * step + 2.4e-7, n


@pytest.mark.gpu
@pytest.mark.parametrize("B,rate,seed,tc", [(2, 0.05, 11, 7), (2, 0.0, 0, 0), (32, 0.05, 5, 7)])
def test_ordered_text2mel_step_vs_oracle(B, rate, seed, tc):
    """test_train.py's test_cuda_train_step_vs_oracle with the option on: fixed shape (max_N, max_T)."""
    from oracle import ref_train as rtr
    from test_train import _batch, _compare_grads, _tie_free
    P = init_params(0, "perturbed")
    if tc:
        P = _tie_free(P)
    eng = _engine(P, tc)
    eng.train_init(B, rate)
    L, mels = _batch(B)
    newP, st, info = rtr.train_step(P, L, mels, global_step=7, seed=seed, rate=rate)
    out = eng.train_step(L, mels, global_step=7, seed=seed, apply=False)
    for k in ("loss", "loss_mels", "loss_bd1", "loss_att"):
        assert abs(out[k] - info[k]) < 1e-5 * max(1.0, abs(info[k])), (k, out[k], info[k])
    _compare_grads(eng, info["grads"])
    eng.train_apply(7)
    _check_update(eng, P, newP, st, T2M_CHECKED)
    eng.close()


@pytest.mark.gpu
def test_ordered_text2mel_step_at_bucket_shape_vs_oracle():
    """test_train_bucketed.py's test_cuda_train_step_at_bucket_shape_vs_oracle with the option on, at (2, 37, 53)."""
    import ref_train_bucket as rtb
    from test_train import _compare_grads, _tie_free
    B, N, T, seed = 2, 37, 53, 11
    P = _tie_free(init_params(0, "perturbed"))
    L, mels = synthetic_bucket(B, N, T, seed=seed)
    newP, st, info = rtb.train_step(P, L, mels, global_step=7, seed=seed, rate=0.05)
    for tc in (7, 0):
        eng = _engine(P, tc)
        eng.train_init(B, 0.05)
        out = eng.train_step(L, mels, global_step=7, seed=seed, apply=False)
        for k in ("loss", "loss_mels", "loss_bd1", "loss_att"):
            assert abs(out[k] - info[k]) < 1e-5 * max(1.0, abs(info[k])), (tc, k, out[k], info[k])
        _compare_grads(eng, info["grads"])
        eng.train_apply(7)
        _check_update(eng, P, newP, st, T2M_CHECKED)
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("B,T,rate,seed,tc", [(2, 12, 0.05, 9, 7), (2, 14, 0.0, 7, 7), (2, 12, 0.05, 9, 0)])
def test_ordered_ssrn_step_vs_oracle(B, T, rate, seed, tc):
    """test_train.py's _ssrn_step_vs_oracle with the option on."""
    from oracle import ref_train as rtr
    from test_train import _compare_grads
    P = init_params(0, "perturbed")
    eng = _engine(P, tc)
    eng.train_init_ssrn(B, T, rate)
    mels = np.random.default_rng(3).uniform(0, 1, (B, T, hp.n_mels)).astype(np.float32)
    mags = np.random.default_rng(4).uniform(0, 1, (B, 4 * T, 1 + hp.n_fft // 2)).astype(np.float32)
    newP, st, info = rtr.train_step_ssrn(P, mels, mags, global_step=3999, seed=seed, rate=rate)
    out = eng.train_step_ssrn(mels, mags, global_step=3999, seed=seed, apply=False)
    for k in ("loss", "loss_mags", "loss_bd2"):
        assert abs(out[k] - info[k]) < 1e-5 * max(1.0, abs(info[k])), (k, out[k], info[k])
    _compare_grads(eng, info["grads"])
    eng.train_apply(3999)
    _check_update(eng, P, newP, st, SSRN_CHECKED, check_v=False)
    eng.close()


# ============================================================================================= one launch at a time
@pytest.fixture(scope="module")
def eng():
    from dc_tts_b200.engine import Engine
    e = Engine(0)
    e.set_option("train_deterministic", 1)
    yield e
    e.close()


def _twice(fn):
    """fn() -> tuple of output tensors, run twice from the same inputs; the outputs' bits must agree"""
    a = [t.clone() for t in fn()]
    b = fn()
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int8) if x.dtype != torch.float64 else x.view(torch.int64),
                           y.view(torch.int8) if y.dtype != torch.float64 else y.view(torch.int64))
    return a


@pytest.mark.gpu
@pytest.mark.parametrize("impl,B,L,K,N,ntaps", [(1, 32, 100, 256, 512, 3), (1, 8, 60, 128, 256, 1), (0, 32, 100, 256, 512, 3),
                                                (0, 16, 130, 80, 1028, 1)])
def test_conv_gemm_weight_gradient_twice(eng, impl, B, L, K, N, ntaps):
    """Weight gradients whose split count is above 1 in the ordered mode, against tests/test_gpu_train_gemm.py's float64 tap
    loop at its TAU and floor"""
    from test_gpu_train_gemm import FLOOR_BITS, TAU as GEMM_TAU, ref_wgrad
    g = torch.Generator(device="cuda").manual_seed(K + N)
    X = torch.randn(B, L, (K + 3) // 4 * 4, device="cuda", generator=g)
    dY = torch.randn(B, L, (N + 3) // 4 * 4, device="cuda", generator=g)
    shifts = [j - ntaps // 2 for j in range(ntaps)]

    def run():
        out = torch.zeros(ntaps, K, (N + 3) // 4 * 4, device="cuda")
        return (eng.conv_gemm(impl, 1, X, K, dY, N, shifts, out, accumulate=1),)
    got = _twice(run)[0][:, :, :N].double()
    Xd, Dd = X[..., :K].double(), dY[..., :N].double()
    ref, S = ref_wgrad(Xd, Dd, shifts), ref_wgrad(Xd.abs(), Dd.abs(), shifts)
    floor = float(Xd.abs().max()) * float(Dd.abs().max()) * 2.0 ** -FLOOR_BITS * (B * L)
    err = (got - ref).abs()
    assert bool((err <= GEMM_TAU[impl] * S + floor).all()), (impl, float((err / S).max()))


@pytest.mark.gpu
@pytest.mark.parametrize("C,mode", [(128, 1), (256, 1), (512, 1), (1024, 1), (1025, 1), (80, 0), (256, 0), (512, 0), (1024, 0),
                                    (1025, 0), (2049, 0)])
@pytest.mark.parametrize("rows", [1, 33, 32 * 840])
def test_block_bwd_twice(eng, C, mode, rows):
    """Every instantiation, the highway branch (mode 1) and the conv branch (mode 0, with ReLU) of each that has both"""
    g = torch.Generator(device="cuda").manual_seed(C + rows)
    nconv = 2 * C if mode == 1 else C
    pre = torch.randn(rows, nconv, device="cuda", generator=g)
    gout = torch.randn(rows, C, device="cuda", generator=g)
    X = torch.randn(rows, C, device="cuda", generator=g) if mode == 1 else None
    ln = torch.randn(4, C, device="cuda", generator=g) * 0.1 + torch.tensor([1.0, 0.0, 1.0, 0.0], device="cuda")[:, None]
    act = 1 if mode == 0 else 0

    def run():
        dy = torch.zeros(rows, nconv, device="cuda")
        gin = torch.zeros(rows, C, device="cuda") if mode == 1 else None
        dparams = torch.zeros(4 * C + nconv, device="cuda")
        eng.block_bwd(mode, act, C, pre, gout, ln, dy, dparams, X=X, gin=gin, dropout_rate=RATE, layer=3, seed=11)
        return (dy, dparams) + ((gin,) if mode == 1 else ())
    out = _twice(run)
    keep = rk.drop_multiplier(rows, C, 3, 11, RATE, device="cuda")
    ref, sc = rk.block_bwd(mode, act, pre, gout, ln, keep, X)
    dy, dp = out[0].double(), out[1].double()
    assert bool(((dy - ref["dy"]).abs() <= TAU["block"] * sc["dy"]).all())
    if mode == 1:
        assert bool(((out[2].double() - ref["gin"]).abs() <= TAU["block"] * sc["gin"]).all())
    parts = {"dg1": dp[:C], "db1": dp[C:2 * C], "dbias": dp[4 * C:]}
    if mode == 1:
        parts.update(dg2=dp[2 * C:3 * C], db2=dp[3 * C:4 * C])
    for k, v in parts.items():
        assert bool(((v - ref[k]).abs() <= TAU["block_sum"] * sc[k]).all()), k


@pytest.mark.gpu
@pytest.mark.parametrize("rows,C", [(32 * 210, 80), (8 * 840, 1025), (3, 7)])
def test_train_loss_twice(eng, rows, C):
    g = torch.Generator(device="cuda").manual_seed(rows)
    logits = torch.randn(rows, C, device="cuda", generator=g) * 3
    target = torch.rand(rows, C, device="cuda", generator=g)

    def run():
        sums = torch.zeros(2, dtype=torch.float64, device="cuda")
        dl = torch.zeros(rows, C, device="cuda")
        eng.train_loss(logits, target, dl, sums)
        return dl, sums
    dl, sums = _twice(run)
    ref, sc = rk.train_loss(logits, target)
    assert bool(((dl.double() - ref["dlogits"]).abs() <= TAU["loss"] * sc["dlogits"]).all())
    assert abs(float(sums[0]) - float(ref["l1"])) <= TAU["loss"] * float(sc["l1"])
    assert abs(float(sums[1]) - float(ref["bce"])) <= TAU["loss"] * float(sc["bce"])


@pytest.mark.gpu
@pytest.mark.parametrize("B,N,T", [(4, 57, 80), (32, 180, 210)])
def test_attn_bwd_twice(eng, B, N, T):
    d = hp.d
    g = torch.Generator(device="cuda").manual_seed(N)
    Q = torch.randn(B, T, d, device="cuda", generator=g) * 0.1
    KV = torch.randn(B, N, 2 * d, device="cuda", generator=g) * 0.1
    align = torch.softmax(Q @ KV[..., :d].transpose(1, 2), 2).transpose(1, 2).contiguous()
    gR = torch.randn(B, T, 2 * d, device="cuda", generator=g) * 1e-3
    nn, tt = np.meshgrid(np.arange(hp.max_N), np.arange(hp.max_T), indexing="ij")
    gts = torch.tensor(1 - np.exp(-((tt / hp.max_T - nn / hp.max_N) ** 2) / (2 * 0.2 ** 2)), dtype=torch.float32, device="cuda")
    n_lim, t_lim = min(N, hp.max_N), min(T, hp.max_T)

    def run():
        gQ, gKV = torch.zeros(B, T, d, device="cuda"), torch.zeros(B, N, 2 * d, device="cuda")
        sums = torch.zeros(3, dtype=torch.float64, device="cuda")
        eng.attn_bwd(gR, Q, KV, align, gts, n_lim, t_lim, gQ, gKV, sums)
        return gQ, gKV, sums
    gQ, gKV, sums = _twice(run)
    ref, sc = rk.attn_bwd(gR, Q, KV, align, gts, n_lim, t_lim)
    assert bool(((gQ.double() - ref["gQ"]).abs() <= TAU["attn"] * sc["gQ"]).all())
    assert bool(((gKV.double() - ref["gKV"]).abs() <= TAU["attn"] * sc["gKV"]).all())
    assert abs(float(sums[2]) - float(ref["att"])) <= TAU["attn"] * float(sc["att"])


# ============================================================================================= compile
ORDERED = ["ordered_colsum_kernelIf", "ordered_colsum_kernelId", "conv_wgrad_part_kernel", "train_loss_ordered_kernel",
           "attn_loss_ordered_kernel", "embed_bwd_ordered_kernel"] + \
          ["train_block_bwd_ordered_kernelILi%dELb%dE" % b for b in [(4, 1), (8, 1), (16, 1), (32, 1), (33, 1), (65, 0)]]


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    obj = str(tmp_path_factory.mktemp("ptxas") / "kernels_ordered.o")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-c", os.path.join(build.CSRC, "kernels_ordered.cu"), "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stderr


def _report(log, tag):
    lines, cur = [], False
    for line in log.splitlines():
        m = re.search(r"(?:Compiling entry function|Function properties for) '?(\w+)'?", line)
        if m:
            cur = tag in m.group(1)
            continue
        if cur:
            lines.append(line)
    return "\n".join(lines)


@pytest.mark.parametrize("tag", ORDERED)
def test_ordered_kernel_no_stack_no_spills(ptxas_log, tag):
    text = _report(ptxas_log, tag)
    assert "Used" in text, ptxas_log[-4000:]
    assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in text, text


def test_every_ordered_kernel_is_checked(ptxas_log):
    names = set(re.findall(r"Compiling entry function '(\w+)'", ptxas_log))
    assert names == {n for n in names if any(t in n for t in ORDERED)}, names
