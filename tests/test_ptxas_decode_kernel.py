"""Compiles kernels_decode.cu with the package's nvcc flags and reads ptxas's report for every instantiation of the
persistent decode kernel (utterances per cluster 1..5, with and without lap timers): no stack frame (with no L1 left
beside 227 KB of shared memory a stack access is an L2 round trip), no spills, and none of the wgmma serialisation
warnings (C7510 .. C7520) that mean ptxas waited for the tensor pipe where the recompute keeps MMAs in flight."""
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
    obj = str(tmp_path_factory.mktemp("ptxas") / "kernels_decode.o")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-c", os.path.join(build.CSRC, "kernels_decode.cu"), "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stderr


def _entries(log):
    """{mangled kernel name: the ptxas lines about it} for the decode_cluster_kernel instantiations."""
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"(?:Compiling entry function|Function properties for) '?(\w+)'?", line)
        if m:
            cur = m.group(1) if "decode_cluster_kernel" in m.group(1) else None
            if cur:
                out.setdefault(cur, [])
            continue
        if cur:
            out[cur].append(line)
    return out


def test_every_instantiation_is_compiled(ptxas_log):
    names = _entries(ptxas_log)
    for prof in ("Lb0E", "Lb1E"):
        for g in range(1, 6):
            assert any((prof + "Li%dE" % g) in n for n in names), (prof, g, sorted(names))


def test_no_stack_no_spills(ptxas_log):
    names = _entries(ptxas_log)
    assert len(names) == 10, sorted(names)
    for name, lines in names.items():
        text = "\n".join(lines)
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in text, (name, text)


def test_no_wgmma_serialisation_warnings(ptxas_log):
    bad = [ln for ln in ptxas_log.splitlines() if re.search(r"C75(1\d|20)", ln)]
    assert not bad, bad
