"""ptxas's report for the vocoder kernels that take the streaming vocoder's per-utterance bounds (kernels_vocoder.cu):
every instantiation of prepare, istft, overlap-add, stft_phase and the three de-emphasis kernels, whole-signal and
streaming (STREAM = true), compiles for sm_90a with no stack frame and no spills."""
import os
import re
import subprocess

import pytest

from dc_tts_b200 import build

STREAM_KERNELS = ("voc_prepare_kernel", "voc_istft_kernel", "voc_ola_kernel", "voc_stft_phase_kernel", "voc_deemph_local_kernel",
                  "voc_deemph_carry_kernel", "voc_deemph_apply_kernel")


def test_stream_kernels_have_no_stack_and_no_spills(tmp_path):
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    obj = str(tmp_path / "kernels_vocoder.o")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-c", os.path.join(build.CSRC, "kernels_vocoder.cu"), "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    props, cur = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Function properties for (\w+)", line)
        if m:
            cur = m.group(1)
            continue
        if cur and "stack frame" in line:
            props[cur] = line.strip()
            cur = None
    for k in STREAM_KERNELS:
        hits = [(name, p) for name, p in props.items() if k in name]
        # whole-signal and streaming (STREAM) instantiations: prepare and de-emphasis 2; istft and ola 2 per n_fft; stft_phase
        # 4 whole-signal (momentum x convergence) and 2 streaming (momentum) per n_fft
        assert len(hits) == {"voc_istft_kernel": 6, "voc_ola_kernel": 6, "voc_stft_phase_kernel": 18}.get(k, 2), (k, sorted(props))
        for name, p in hits:
            assert p == "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", (name, p)
