"""Fast Griffin-Lim on the GPU (dctts_spectrogram2wav_momentum, Engine.spectrogram2wav(momentum=..., convergence=...)).

  * One momentum phase step (dctts_vocoder_momentum_step) against float64 at n_fft 1024, 2048 and 4096, in the stft_phase
    bound form of tests/ref_vocoder_stages.py with A_t extended by alpha |est_{i-1,k}| (the previous estimate enters c
    with weight alpha); the raw estimate written back to E against float64 STFT within TAU A_t; each frame's
    sum_k (S - |est|)^2 within TAU_PART (2 A_t sum_k |S - |est|| + the sum itself).
  * Momentum 0 reproduces dctts_spectrogram2wav and _ragged, called through the C-ABI, bit for bit, with the convergence
    history on and off.
  * With momentum the whole call equals the stages chained by hand, bit for bit; a ragged call equals each utterance's
    call alone, bit for bit.
  * The history matches the float64 oracle (tests/ref_fast_griffin_lim.py) at small n_iter, and shows the
    gain of momentum 0.99 over plain Griffin-Lim that test_vocoder_momentum.py asserts for the oracle.
Engines are built and run inside `at_rate`, because an engine reads hop and win from Hyperparams at call time.
"""
import contextlib
import warnings

import numpy as np
import pytest
import torch

from dc_tts_b200.engine import DcttsError
from dc_tts_b200.hyperparams import Hyperparams
import ref_fast_griffin_lim as fg
import ref_vocoder_stages as rs
from sample_rates import at_rate

pytestmark = pytest.mark.gpu
SR = {1024: 16000, 2048: 22050, 4096: 44100}
LENGTHS = (2, 3, 5, 60, 840)
MOMENTA = (0.99, 0.5, 3.0)
# worst err / bound scale over this file's cases on an H100 80GB HBM3 at 700 W (DESIGN.md section 8b): step 8.16e-8,
# 8.69e-8, 8.29e-8 and est 6.0e-8, 7.84e-8, 4.03e-8 at n_fft 1024, 2048, 4096; part 2.48e-7; history 2.45e-6 relative.
# Each TAU is about 3x of its worst.
TAU = {1024: dict(step=2.5e-7, est=1.8e-7), 2048: dict(step=2.6e-7, est=2.4e-7), 4096: dict(step=2.5e-7, est=1.2e-7)}
TAU_PART = 7.5e-7
TAU_HIST = 7.5e-6
_WORST = {}


def _record(key, raw):
    _WORST[key] = max(_WORST.get(key, 0.0), float(raw))


@contextlib.contextmanager
def power(p):
    old = Hyperparams.power
    Hyperparams.power = p
    try:
        yield
    finally:
        Hyperparams.power = old


@pytest.fixture(scope="module")
def engines():
    from dc_tts_b200.engine import Engine
    out = {}
    for n in SR:
        with at_rate(SR[n], n) as H:
            out[n] = Engine(0, hparams=H)
    yield out
    print("\nfast Griffin-Lim, worst err / bound scale: " + ", ".join("%s %.3g" % (k, v) for k, v in sorted(_WORST.items())))
    for e in out.values():
        e.close()


# ------------------------------------------------------------------------------------------------ one step vs float64
def check_momentum_step(X, E_out, part, y, S, E_prev, alpha, hop, win, tau, tau_est):
    """-> (ratios, raws) of X (the stft_phase bound at alpha and E_prev), the raw estimate E_out and the per-frame
    partials against float64."""
    est, A = rs.ref_stft(y, 2 * (S.shape[-1] - 1), hop, win, S.shape[1])
    ratio, raw = rs.check_phase(X, est, A, S, E_prev, alpha, tau)
    S = S.astype(np.float64)
    err_e = np.abs(E_out.astype(np.complex128) - est)
    ratio_e = float((err_e / (tau_est * A[..., None] + 1e-37)).max())
    pos = A > 0
    raw_e = float((err_e[pos] / A[pos][:, None]).max()) if pos.any() else 0.0
    d = S - np.abs(est)
    ref_p = (d * d).sum(-1)
    scale_p = 2.0 * A * np.abs(d).sum(-1) + ref_p
    err_p = np.abs(part.astype(np.float64) - ref_p)
    ratio_p = float((err_p / (TAU_PART * scale_p + 1e-37)).max())
    raw_p = float((err_p[scale_p > 0] / scale_p[scale_p > 0]).max()) if (scale_p > 0).any() else 0.0
    return (ratio, ratio_e, ratio_p), (raw, raw_e, raw_p)


def _cases():
    out = []
    for i, (n, T) in enumerate((n, T) for n in SR for T in LENGTHS):
        B = rs.case_batch(i)
        if T * SR[n] // 80 > 120000 and B == 32:
            B = 3
        out.append((n, T, B, MOMENTA[i % 3]))
    return out


CASES = _cases()


@pytest.mark.parametrize("n,T,B,momentum", CASES, ids=["n%d-T%d-B%d-m%g" % c for c in CASES])
def test_momentum_step_vs_float64(engines, n, T, B, momentum):
    eng = engines[n]
    with at_rate(SR[n], n) as H:
        F, hop, win = 1 + n // 2, H.hop_length, H.win_length
        rng = np.random.default_rng(T * n + B)
        Ly = hop * (T - 1)
        lev = np.array(rs.LEVELS * B, np.float32)[:B, None, None]
        y = rs.make_wav(rng, B, Ly)
        S = rng.uniform(0, 2, (B, T, F)).astype(np.float32) * lev
        S[:, :, ::97] = 0.0
        Ep = ((rng.standard_normal((B, T, F)) + 1j * rng.standard_normal((B, T, F))) * 5.0 * lev).astype(np.complex64)
        Ep[:, :, 1::89] = 0.0
        bi, vi = rs.guarded(eng, (B, Ly), torch.float32, y)
        bs, vs_ = rs.guarded(eng, (B, T, F), torch.float32, S)
        be, ve = rs.guarded(eng, (B, T, F), torch.complex64, Ep)
        bo, vo = rs.guarded(eng, (B, T, F), torch.complex64)
        bp, vp = rs.guarded(eng, (B, T), torch.float32)
        eng.vocoder_momentum_step(vi, vs_, ve, vo, momentum, vp, hop=hop, win=win)
        rs.intact(bi, vi)
        rs.intact(bs, vs_)
        alpha = np.float32(momentum / (1.0 + momentum))
        ratios, raws = check_momentum_step(rs.intact(bo, vo), rs.intact(be, ve), rs.intact(bp, vp), y, S, Ep, alpha, hop,
                                           win, TAU[n]["step"], TAU[n]["est"])
    for key, r in zip(("step", "est", "part"), raws):
        _record("n_fft %d %s" % (n, key) if key != "part" else "part", r)
    assert max(ratios) <= 1, (ratios, raws)


# ------------------------------------------------------------------------------------------------ bit-exact compositions
def _c_call(eng, mag, n_iter, lengths=None, momentum=None, convergence=False):
    """spectrogram2wav straight through the C-ABI: dctts_spectrogram2wav_momentum when `momentum` is given, else
    dctts_spectrogram2wav, or dctts_spectrogram2wav_ragged with `lengths`."""
    B, T, _ = mag.shape
    eng._set_vocoder_params()
    wav = torch.empty(B, eng.hp.hop_length * (T - 1), device=eng.device)
    trim = np.zeros((B, 2), np.int32)
    conv = torch.empty(B, n_iter + 1, dtype=torch.float64, device=eng.device) if convergence else None
    n = None if lengths is None else np.ascontiguousarray(lengths, np.int32)
    n_ptr = None if n is None else n.ctypes.data
    if momentum is not None:
        fn, args = "dctts_spectrogram2wav_momentum", (n_ptr, n_iter, float(momentum), wav.data_ptr(), trim.ctypes.data,
                                                      None if conv is None else conv.data_ptr())
    elif n is None:
        fn, args = "dctts_spectrogram2wav", (n_iter, wav.data_ptr(), trim.ctypes.data)
    else:
        fn, args = "dctts_spectrogram2wav_ragged", (n_ptr, n_iter, wav.data_ptr(), trim.ctypes.data)
    eng._check(getattr(eng._lib, fn)(eng._h, mag.data_ptr(), B, T, *args, eng._stream()), fn)
    return wav, trim, conv


@pytest.mark.parametrize("n", sorted(SR))
@pytest.mark.parametrize("T,n_iter", [(5, 2), (60, 4)])
def test_momentum_zero_reproduces_the_existing_calls(engines, n, T, n_iter):
    """The plain and ragged entry points are the reference side; the momentum entry point at momentum 0, directly and
    through Engine.spectrogram2wav, must give their bytes."""
    eng = engines[n]
    with at_rate(SR[n], n):
        B = 3
        mag = torch.from_numpy(rs.make_mag(np.random.default_rng(T + n), B, T, n)).to(eng.device)
        lengths = np.array([T, 2, max(2, T // 2)], np.int32)
        w0, t0, _ = _c_call(eng, mag, n_iter)
        r0, rt0, _ = _c_call(eng, mag, n_iter, lengths)
        for conv in (False, True):
            w1, t1, _ = _c_call(eng, mag, n_iter, momentum=0.0, convergence=conv)
            assert torch.equal(w0, w1) and np.array_equal(t0, t1), conv
            r1, rt1, _ = _c_call(eng, mag, n_iter, lengths, momentum=0.0, convergence=conv)
            assert torch.equal(r0, r1) and np.array_equal(rt0, rt1), conv
        w2, t2 = eng.spectrogram2wav(mag, n_iter=n_iter)
        r2, rt2 = eng.spectrogram2wav(mag, n_iter=n_iter, lengths=lengths)
        assert torch.equal(w0, w2) and np.array_equal(t0, t2) and torch.equal(r0, r2) and np.array_equal(rt0, rt2)
        w3, t3, h3 = eng.spectrogram2wav(mag, n_iter=n_iter, convergence=True)
        assert torch.equal(w0, w3) and np.array_equal(t0, t3) and tuple(h3.shape) == (B, n_iter + 1)


def test_plain_launch_count_is_unchanged(engines):
    eng = engines[2048]
    with at_rate(SR[2048]):
        mag = np.full((2, 5, 1025), 0.5, np.float32)
        for kw, extra in ((dict(), 0), (dict(momentum=0.99), 0), (dict(momentum=0.99, convergence=True), 2)):
            c0 = eng.launch_count()
            eng.spectrogram2wav(mag, n_iter=3, **kw)
            assert eng.launch_count() - c0 == 1 + 3 * 3 + 2 + 3 + 1 + extra, kw


@pytest.mark.parametrize("n", sorted(SR))
@pytest.mark.parametrize("n_iter", [1, 2, 3])
def test_momentum_iterations_are_the_stages_bit_for_bit(engines, n, n_iter):
    eng = engines[n]
    with at_rate(SR[n], n) as H:
        B, T, F, hop, win, mom = 3, 60, 1 + n // 2, H.hop_length, H.win_length, 0.99
        mag = torch.from_numpy(rs.make_mag(np.random.default_rng(n_iter + n), B, T, n)).to(eng.device)
        Ly = hop * (T - 1)
        kw = dict(hop=hop, win=win)
        X = torch.empty(B, T, F, dtype=torch.complex64, device=eng.device)
        eng.vocoder_stage(0, mag, X, **kw)
        S = X.real.contiguous()
        E = torch.zeros_like(X)
        y = torch.empty(B, Ly, device=eng.device)
        parts = []
        for _ in range(n_iter):
            eng.vocoder_stage(1, X, y, **kw)
            parts.append(torch.empty(B, T, device=eng.device))
            eng.vocoder_momentum_step(y, S, E, X, mom, parts[-1], **kw)
        eng.vocoder_stage(1, X, y, **kw)
        parts.append(torch.empty(B, T, device=eng.device))
        eng.vocoder_momentum_step(y, S, E.clone(), torch.empty_like(X), mom, parts[-1], **kw)
        eng.vocoder_stage(3, y, y, **kw)
        trim2 = eng.vocoder_stage(4, y, torch.empty(B, 1 + Ly // 512, device=eng.device), **kw)
        wav, trim, conv = eng.spectrogram2wav(mag, n_iter=n_iter, momentum=mom, convergence=True)
        assert torch.equal(wav, y) and np.array_equal(trim, trim2)
        P = np.stack([p.cpu().numpy().astype(np.float64) for p in parts], 1)        # (B, n_iter + 1, T)
        ref = np.sqrt(np.cumsum(P, -1)[..., -1]) / np.sqrt((S.cpu().numpy().astype(np.float64) ** 2).sum((1, 2)))[:, None]
        np.testing.assert_allclose(conv.cpu().numpy(), ref, rtol=1e-12)


@pytest.mark.parametrize("n", sorted(SR))
@pytest.mark.parametrize("T,lengths", [(60, (60, 2, 3, 31, 59)), (840, (840, 400, 5))])
def test_ragged_momentum_is_each_utterance_alone(engines, n, T, lengths):
    eng = engines[n]
    with at_rate(SR[n], n) as H:
        hop, B = H.hop_length, len(lengths)
        mag = rs.make_mag(np.random.default_rng(T + n + 1), B, T, n)
        wav, trim, conv = eng.spectrogram2wav(mag, n_iter=3, lengths=lengths, momentum=0.99, convergence=True)
        wav, conv = wav.cpu().numpy(), conv.cpu().numpy()
        for b, Tb in enumerate(lengths):
            w1, t1, c1 = eng.spectrogram2wav(mag[b:b + 1, :Tb], n_iter=3, momentum=0.99, convergence=True)
            Lb = hop * (Tb - 1)
            assert np.array_equal(wav[b, :Lb], w1.cpu().numpy()[0]) and not wav[b, Lb:].any(), b
            assert np.array_equal(trim[b], t1[0]) and np.array_equal(conv[b], c1.cpu().numpy()[0]), b


# ------------------------------------------------------------------------------------------------ convergence history
@pytest.mark.parametrize("momentum", [0.0, 0.99])
@pytest.mark.parametrize("kind", rs.SIGNALS)
def test_history_matches_the_float64_oracle(engines, kind, momentum):
    eng = engines[2048]
    with at_rate(SR[2048]) as H:
        mag = rs.magnitude(kind)
        for n_iter in (0, 1, 3):
            _, _, conv = eng.spectrogram2wav(mag[None], n_iter=n_iter, momentum=momentum, convergence=True)
            _, ref = fg.fast_griffin_lim(rs.amplitude(mag, H.power, np.float64), n_iter, momentum, convergence=True)
            rel = np.abs(conv.cpu().numpy()[0] - ref) / ref
            _record("history", rel.max())
            assert rel.max() <= TAU_HIST, (n_iter, rel, conv, ref)


@pytest.mark.parametrize("p", rs.POWERS)
def test_gpu_gains_what_the_oracle_gains(engines, p):
    """The three signals in one call (all have 81 frames): momentum 0.99 ends 50 iterations lower than plain Griffin-Lim,
    and the plain history falls, as test_vocoder_momentum.py asserts for the oracle."""
    eng = engines[2048]
    with at_rate(SR[2048]), power(p):
        mags = np.stack([rs.magnitude(k) for k in rs.SIGNALS])
        _, _, plain = eng.spectrogram2wav(mags, n_iter=50, convergence=True)
        _, _, fast = eng.spectrogram2wav(mags, n_iter=50, momentum=0.99, convergence=True)
        plain, fast = plain.cpu().numpy(), fast.cpu().numpy()
        for b, kind in enumerate(rs.SIGNALS):
            first = int(np.argmax(fast[b] <= plain[b, -1]))
            print("power %.1f %s: plain %.4f -> %.4f, momentum 0.99 -> %.4f, reaches plain's 50-iteration value at %d" %
                  (p, kind, plain[b, 0], plain[b, -1], fast[b, -1], first))
            assert np.all(np.diff(plain[b]) <= 1e-4 * plain[b, :-1]), (kind, plain[b])
            assert fast[b, -1] < plain[b, -1], (kind, fast[b, -1], plain[b, -1])


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals(engines):
    eng = engines[2048]
    with at_rate(SR[2048]):
        mag = np.full((1, 5, 1025), 0.5, np.float32)
        for bad in (-0.5, float("nan"), float("inf")):
            with pytest.raises(DcttsError, match="momentum must be finite and >= 0"):
                eng.spectrogram2wav(mag, n_iter=1, momentum=bad)
        with pytest.warns(UserWarning, match="momentum=2 > 1"):
            eng.spectrogram2wav(mag, n_iter=1, momentum=2.0)
        with warnings.catch_warnings():
            warnings.simplefilter("error")
            eng.spectrogram2wav(mag, n_iter=1, momentum=0.99)     # no warning up to 1, and the handle stays usable
