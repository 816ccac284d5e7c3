"""Compiles kernels_attn_tc.cu with the package's nvcc flags and reads ptxas's report for the wgmma attention kernel: no
stack frame, no spills (C holds 128 registers per thread beside one 32-register S block), and none of the wgmma
serialisation warnings (C7510 .. C7520) that mean ptxas waited for the tensor pipe where the code keeps MMAs in flight."""
import os
import re
import subprocess

import pytest

from dc_tts_b200 import build


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    obj = str(tmp_path_factory.mktemp("ptxas") / "kernels_attn_tc.o")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-c", os.path.join(build.CSRC, "kernels_attn_tc.cu"), "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stderr


def _entry(log, kernel):
    lines, cur = [], False
    for line in log.splitlines():
        m = re.search(r"(?:Compiling entry function|Function properties for) '?(\w+)'?", line)
        if m:
            cur = kernel in m.group(1)
            continue
        if cur:
            lines.append(line)
    return "\n".join(lines)


def test_attention_kernel_no_stack_no_spills(ptxas_log):
    text = _entry(ptxas_log, "attention_tc_kernel")
    assert "Used" in text, ptxas_log[-4000:]
    assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in text, text


def test_attention_kernel_no_wgmma_serialisation_warnings(ptxas_log):
    bad = [ln for ln in ptxas_log.splitlines() if re.search(r"C75(1\d|20)", ln) and "attention_tc_kernel" in ln]
    assert not bad, bad
