"""CPU side of the vocoder stage references (tests/ref_vocoder_stages.py) at n_fft 1024, 2048 and 4096: a float32
chain passes each stage's bound at the size's TAU, and degraded ones (fp16-rounded inputs or twiddles, de-emphasis in
float32) fail it.  Also the rate table, and ptxas's report for every kernel instantiation the other sizes added."""
import os
import re
import subprocess

import numpy as np
import pytest
import scipy.signal

import ref_vocoder_stages as rs
from dc_tts_b200 import build
from dc_tts_b200.hyperparams import Hyperparams as hp
from oracle import ref_vocoder as rv
from ref_vocoder_stages import HOP_WIN, TAU
from sample_rates import at_rate, rate_values

# (n_fft, hop, win, T): every (hop, win) of the GPU stage cases, on T frames
CASES = [(n, hop, win, 8 if n == 2048 else 6) for n in (1024, 4096, 2048) for hop, win in HOP_WIN[n]]
IDS = ["%d-%d-%d" % c[:3] for c in CASES]


def test_rate_table():
    assert rate_values(16000) == dict(sr=16000, n_fft=1024, hop_length=200, win_length=800)
    assert rate_values(22050) == dict(sr=22050, n_fft=2048, hop_length=275, win_length=1102)
    assert rate_values(44100) == dict(sr=44100, n_fft=4096, hop_length=551, win_length=2205)
    assert rate_values(48000) == dict(sr=48000, n_fft=4096, hop_length=600, win_length=2400)
    from dc_tts_b200.hyperparams import Hyperparams
    with at_rate(44100) as H:
        assert (H.sr, H.n_fft, H.hop_length, H.win_length) == (44100, 4096, 551, 2205)
    assert (Hyperparams.sr, Hyperparams.n_fft, Hyperparams.hop_length, Hyperparams.win_length) == (22050, 2048, 275, 1102)


@pytest.mark.parametrize("n,hop,win,T", CASES, ids=IDS)
def test_float32_istft_passes_and_fp16_twiddles_fail(n, hop, win, T):
    """fp16-rounded twiddles fail the bound, and so does an fp16-rounded spectrum."""
    X = rs.make_spectrum(np.random.default_rng(hop + win), 3, T, n)
    tau = TAU[n]["istft"]
    r32, _ = rs.check_istft(rs.istft32(X, hop, win), X, hop, win, tau)
    assert r32 < 0.5, r32
    r_in, _ = rs.check_istft(rs.istft32(rs.fp16(X), hop, win), X, hop, win, tau)
    r_tw, _ = rs.check_istft(rs.istft32(X, hop, win, twiddles16=True), X, hop, win, tau)
    assert r_in > 1 and r_tw > 1, (r_in, r_tw)


@pytest.mark.parametrize("n,hop,win,T", CASES, ids=IDS)
def test_float32_stft_phase_passes_and_fp16_fails(n, hop, win, T):
    rng = np.random.default_rng(hop * win)
    y = rs.make_wav(rng, 3, hop * (T - 1))
    S = rng.uniform(0, 2, (3, T, 1 + n // 2)).astype(np.float32)
    got = np.stack([rs.phase_update(S[b], rv.stft(y[b], n, hop, win).T, np.float32) for b in range(3)])
    assert got.dtype == np.complex64
    r32, _ = rs.check_stft_phase(got, y, S, hop, win, TAU[n]["stft"])
    assert r32 < 0.5, r32
    y16 = rs.fp16(y)
    bad = np.stack([rs.phase_update(S[b], rv.stft(y16[b], n, hop, win).T, np.float32) for b in range(3)])
    r16, _ = rs.check_stft_phase(bad, y, S, hop, win, TAU[n]["stft"])
    assert r16 > 1, r16


@pytest.mark.parametrize("power", [1.5, 1.0])
def test_float32_prepare_passes_and_fp16_fails(power):
    """The prepare stage does not depend on n_fft."""
    mag = rs.make_mag(np.random.default_rng(3), 3, 5, 2048)
    m = np.clip(mag, 0, 1) * np.float32(hp.max_db) - np.float32(hp.max_db) + np.float32(hp.ref_db)
    got = np.power(np.power(np.float32(10), m * np.float32(0.05)), np.float32(power))
    assert got.dtype == np.float32
    assert rs.check_prepare(got, mag, power, TAU[2048]["prepare"])[0] < 0.5
    assert rs.check_prepare(rs.fp16(got), mag, power, TAU[2048]["prepare"])[0] > 1


# (Ly, seed): short and chunk-edge lengths at 22.05 kHz, then 59 hops at 16, 44.1 and 48 kHz seeded with the rate
DEEMPH = [(Ly, Ly) for Ly in (275, 512, 1024 + 17, 275 * 512)] + \
         [(rate_values(sr)["hop_length"] * 59, sr) for sr in (16000, 44100, 48000)]


@pytest.mark.parametrize("Ly,seed", DEEMPH, ids=["Ly%d" % Ly for Ly, _ in DEEMPH])
def test_chunked_float64_deemph_passes_and_float32_fails(Ly, seed):
    """The de-emphasis does not depend on n_fft."""
    x = rs.make_deemph_input(np.random.default_rng(seed), 3, Ly)
    ulps, exact = rs.check_deemph(rs.deemph_chunked(x), x)
    assert ulps <= 1 and exact >= 0.999, (ulps, exact)
    if Ly > 512:
        y32 = scipy.signal.lfilter(np.ones(1, np.float32), np.array([1, -hp.preemphasis], np.float32), x, axis=-1)
        assert y32.dtype == np.float32
        ulps32, exact32 = rs.check_deemph(y32, x)
        assert ulps32 > 1 and exact32 < 0.999, (ulps32, exact32)
        c32 = float(np.float32(hp.preemphasis))             # the float64 filter with a float32-rounded coefficient
        ulps_c, exact_c = rs.check_deemph(rs.deemph_chunked(x, c32), x)
        assert ulps_c > 1 or exact_c < 0.999, (ulps_c, exact_c)


def test_float32_energies_pass_and_fp16_fail():
    """The trim energies do not depend on n_fft."""
    y = rs.make_wav(np.random.default_rng(5), 3, 275 * 59)
    got = rs.energies32(y)
    assert got.dtype == np.float32
    assert rs.check_energies(got, y, TAU[2048]["energies"])[0] < 0.5
    assert rs.check_energies(rs.energies32(rs.fp16(y)), y, TAU[2048]["energies"])[0] > 1


def _inverts(n, hop_wins):
    for hop, win in hop_wins:
        y = np.random.default_rng(win).standard_normal((2, hop * 20))
        est, _ = rs.ref_stft(y, n, hop, win, 21)
        back, _ = rs.ref_istft(est, hop, win)
        assert np.abs(back - y).max() < 1e-12, (n, hop, win)


@pytest.mark.parametrize("n", (1024, 4096))
def test_reference_istft_inverts_reference_stft(n):
    """The float64 references invert each other (librosa's perfect reconstruction), at every window of the matrix."""
    _inverts(n, HOP_WIN[n])


def test_reference_istft_inverts_reference_stft_at_2048():
    """The same at n_fft 2048, at every window but (1102, 1102): its Hann windows only abut, so the window sum-square is
    exactly 0 where they meet and those samples cannot be reconstructed."""
    _inverts(2048, [hw for hw in HOP_WIN[2048] if hw != (1102, 1102)])


# ------------------------------------------------------------------------------------------------ ptxas
def _ptxas(src, tmp):
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    obj = str(tmp / (src + ".o"))
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-c", os.path.join(build.CSRC, src + ".cu"), "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    props = {}
    cur = None
    for line in r.stderr.splitlines():
        m = re.search(r"Function properties for (\w+)", line)
        if m:
            cur = m.group(1)
            continue
        if cur and "stack frame" in line:
            props[cur] = line.strip()
            cur = None
    return props


NEW_KERNELS = {
    "kernels_vocoder": ["voc_istft_kernelILi1024E", "voc_istft_kernelILi4096E", "voc_stft_phase_kernelILi1024E",
                        "voc_stft_phase_kernelILi4096E", "feat_stft_mel_kernelILi1024EfE", "feat_stft_mel_kernelILi1024EsE",
                        "feat_stft_mel_kernelILi4096EfE", "feat_stft_mel_kernelILi4096EsE", "voc_ola_kernelILi1024E",
                        "voc_ola_kernelILi4096E", "voc_twiddle_kernelILi1024E", "voc_twiddle_kernelILi4096E"],
    "kernels_simt": ["ln_rows_kernelILi65E"],
    "kernels_train": ["train_block_bwd_kernelILi65ELb0E"],
    "kernels_tc": ["conv_ln_tc_kernelILi32ELi144E", "conv_ln_tc_kernelILi64ELi144E"],
}


@pytest.mark.parametrize("src", sorted(NEW_KERNELS))
def test_new_instantiations_have_no_stack_and_no_spills(src, tmp_path):
    props = _ptxas(src, tmp_path)
    for k in NEW_KERNELS[src]:
        hits = [(name, p) for name, p in props.items() if k in name]
        assert hits, (k, sorted(props))
        for name, p in hits:
            assert p == "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", (name, p)
