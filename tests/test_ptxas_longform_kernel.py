"""ptxas's report for the long-form join kernel (kernels_longform.cu): it compiles for sm_90a with no stack frame and no spills."""
import os
import re
import subprocess

import pytest

from dc_tts_b200 import build


def test_join_kernel_has_no_stack_and_no_spills(tmp_path):
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    assert "kernels_longform.cu" in build.SOURCES
    obj = str(tmp_path / "kernels_longform.o")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-c", os.path.join(build.CSRC, "kernels_longform.cu"), "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    assert "sm_90a" in r.stderr
    blocks = re.split(r"Compiling entry function", r.stderr)[1:]
    found = [b for b in blocks if "join_rows_kernel" in b.splitlines()[0]]
    assert len(found) == 1, r.stderr[-2000:]
    assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in found[0], found[0]
