"""Compiles kernels_pack.cu with the package's nvcc flags and reads ptxas's report for the three weight packers (the
abs-max reduction, the wgmma planes, the persistent decode's stream): no stack frame, no spills."""
import os
import re
import subprocess

import pytest

from dc_tts_b200 import build

KERNELS = ["weight_absmax_kernel", "pack_tc_kernel", "pack_decode_kernel"]


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    obj = str(tmp_path_factory.mktemp("ptxas") / "kernels_pack.o")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-c", os.path.join(build.CSRC, "kernels_pack.cu"), "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stderr


@pytest.mark.parametrize("kernel", KERNELS)
def test_pack_kernel_no_stack_no_spills(ptxas_log, kernel):
    lines, cur = [], False
    for line in ptxas_log.splitlines():
        m = re.search(r"(?:Compiling entry function|Function properties for) '?(\w+)'?", line)
        if m:
            cur = kernel in m.group(1)
            continue
        if cur:
            lines.append(line)
    text = "\n".join(lines)
    assert "Used" in text, ptxas_log[-4000:]
    assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in text, text
