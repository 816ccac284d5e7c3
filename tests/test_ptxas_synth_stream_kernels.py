"""ptxas's report for the synthesis stream's kernels: every instantiation of the progress-publishing decode
(decode_progress_kernel, G = 1 .. 5; kernels_decode.cu) and the window gather (mel_windows_to_planes_kernel; kernels_tc.cu)
compiles for sm_90a with no stack frame and no spills."""
import os
import re
import subprocess

import pytest

from dc_tts_b200 import build


def _props(src, tmp_path):
    obj = str(tmp_path / (src + ".o"))
    r = subprocess.run([build._nvcc()] + build.NVCC_FLAGS + ["-c", os.path.join(build.CSRC, src), "-o", obj],
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
    return props


@pytest.mark.parametrize("src,kernel,count", [("kernels_decode.cu", "decode_progress_kernel", 5),
                                              ("kernels_tc.cu", "mel_windows_to_planes_kernel", 1)])
def test_synth_stream_kernels_have_no_stack_and_no_spills(tmp_path, src, kernel, count):
    try:
        build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    hits = [(name, p) for name, p in _props(src, tmp_path).items() if kernel in name]
    assert len(hits) == count, hits
    for name, p in hits:
        assert p == "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", (name, p)
