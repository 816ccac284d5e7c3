"""Compiles kernels_tc.cu with the package's nvcc flags and reads ptxas's report for every instantiation of the fused
block kernel: no stack frame, no spills, and none of the wgmma serialisation warnings (C7510 .. C7520) that mean ptxas
waited for the tensor pipe where the code keeps MMAs in flight."""
import os
import re
import subprocess

import pytest

from dc_tts_b200 import build

WIDTHS = (64, 80, 144, 256)


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    obj = str(tmp_path_factory.mktemp("ptxas") / "kernels_tc.o")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-c", os.path.join(build.CSRC, "kernels_tc.cu"), "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stderr


def _entries(log):
    """{mangled kernel name: the ptxas lines about it} for the conv_ln_tc_kernel instantiations."""
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"(?:Compiling entry function|Function properties for) '?(\w+)'?", line)
        if m:
            cur = m.group(1) if "conv_ln_tc_kernel" in m.group(1) else None
            if cur:
                out.setdefault(cur, [])
            continue
        if cur:
            out[cur].append(line)
    return out


def test_every_width_is_instantiated(ptxas_log):
    names = _entries(ptxas_log)
    for bk in (32, 64):
        for bn in WIDTHS:
            assert any(("ILi%dELi%dE" % (bk, bn)) in n for n in names), (bk, bn, sorted(names))


def test_no_stack_no_spills(ptxas_log):
    for name, lines in _entries(ptxas_log).items():
        text = "\n".join(lines)
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in text, (name, text)


def test_no_wgmma_serialisation_warnings(ptxas_log):
    bad = [ln for ln in ptxas_log.splitlines() if re.search(r"C75(1\d|20)", ln) and "conv_ln_tc_kernel" in ln]
    assert not bad, bad
