"""CPU side of n_fft 1024 and 4096: the float64 stage references and bounds of test_gpu_vocoder_stages.py at the other two
sizes with their own TAU (a float32 chain passes them, fp16 twiddles and float32 de-emphasis fail them), the rate table,
and ptxas's report for every kernel instantiation the other sizes added."""
import os
import re
import subprocess

import numpy as np
import pytest
import scipy.signal

import test_gpu_vocoder_stages as vs
from dc_tts_b200 import build
from test_gpu_vocoder_sizes import TAU
from sample_rates import at_rate, rate_values

SIZES = {1024: [(200, 800), (200, 1024), (200, 1023)], 4096: [(551, 2205), (600, 2400), (551, 4096), (551, 4095)]}
CASES = [(n, hop, win) for n, hws in SIZES.items() for hop, win in hws]


@pytest.fixture
def size(monkeypatch):
    def set_size(n):
        monkeypatch.setattr(vs, "N_FFT", n)
        monkeypatch.setattr(vs, "F", 1 + n // 2)
    return set_size


def test_rate_table():
    assert rate_values(16000) == dict(sr=16000, n_fft=1024, hop_length=200, win_length=800)
    assert rate_values(22050) == dict(sr=22050, n_fft=2048, hop_length=275, win_length=1102)
    assert rate_values(44100) == dict(sr=44100, n_fft=4096, hop_length=551, win_length=2205)
    assert rate_values(48000) == dict(sr=48000, n_fft=4096, hop_length=600, win_length=2400)
    from dc_tts_b200.hyperparams import Hyperparams
    with at_rate(44100) as H:
        assert (H.sr, H.n_fft, H.hop_length, H.win_length) == (44100, 4096, 551, 2205)
    assert (Hyperparams.sr, Hyperparams.n_fft, Hyperparams.hop_length, Hyperparams.win_length) == (22050, 2048, 275, 1102)


@pytest.mark.parametrize("n,hop,win", CASES)
def test_float32_istft_passes_and_fp16_twiddles_fail(size, n, hop, win):
    size(n)
    X = vs.make_spectrum(np.random.default_rng(hop + win), 3, 6)
    tau = TAU[n]["istft"]
    r32, _ = vs.check_istft(vs.istft32(X, hop, win), X, hop, win, tau)
    assert r32 < 0.5, r32
    r_tw, _ = vs.check_istft(vs.istft32(X, hop, win, twiddles16=True), X, hop, win, tau)
    assert r_tw > 1, r_tw


@pytest.mark.parametrize("n,hop,win", CASES)
def test_float32_stft_phase_passes_and_fp16_fails(size, n, hop, win):
    from oracle import ref_vocoder as rv
    size(n)
    rng = np.random.default_rng(hop * win)
    T = 6
    y = vs.make_wav(rng, 3, hop * (T - 1))
    S = rng.uniform(0, 2, (3, T, vs.F)).astype(np.float32)
    got = np.stack([vs.phase_update(S[b], rv.stft(y[b], n, hop, win).T, np.float32) for b in range(3)])
    assert vs.check_stft_phase(got, y, S, hop, win, TAU[n]["stft"])[0] < 0.5
    y16 = vs._fp16(y)
    bad = np.stack([vs.phase_update(S[b], rv.stft(y16[b], n, hop, win).T, np.float32) for b in range(3)])
    assert vs.check_stft_phase(bad, y, S, hop, win, TAU[n]["stft"])[0] > 1


@pytest.mark.parametrize("n", sorted(SIZES))
def test_reference_istft_inverts_reference_stft(size, n):
    size(n)
    for hop, win in SIZES[n]:
        y = np.random.default_rng(win).standard_normal((2, hop * 20))
        est, _ = vs.ref_stft(y, hop, win, 21)
        back, _ = vs.ref_istft(est, hop, win)
        assert np.abs(back - y).max() < 1e-12, (hop, win)


@pytest.mark.parametrize("sr", [16000, 44100, 48000])
def test_chunked_float64_deemph_passes_and_float32_fails(sr):
    hop = rate_values(sr)["hop_length"]
    x = vs.make_deemph_input(np.random.default_rng(sr), 3, hop * 59)
    ulps, exact = vs.check_deemph(vs._deemph_chunked(x), x)
    assert ulps <= 1 and exact >= 0.999, (ulps, exact)
    y32 = scipy.signal.lfilter(np.ones(1, np.float32), np.array([1, -0.97], np.float32), x, axis=-1)
    assert y32.dtype == np.float32
    ulps32, exact32 = vs.check_deemph(y32, x)
    assert ulps32 > 1 and exact32 < 0.999, (ulps32, exact32)


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
