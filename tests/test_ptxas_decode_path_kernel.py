"""ptxas's report for every instantiation of the persistent decode along a window path (decode_path_kernel, utterances
per cluster 1..5): no stack frame and no spills, as for the other persistent decode kernels (with 227 KB of shared
memory there is no L1 left, so a stack access is an L2 round trip)."""
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
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"(?:Compiling entry function|Function properties for) '?(\w+)'?", line)
        if m:
            cur = m.group(1) if "decode_path_kernel" in m.group(1) else None
            if cur:
                out.setdefault(cur, [])
            continue
        if cur:
            out[cur].append(line)
    return out


def test_path_kernel_has_no_stack_and_no_spills(ptxas_log):
    names = _entries(ptxas_log)
    assert sorted(int(re.search(r"Li(\d)E", n).group(1)) for n in names) == [1, 2, 3, 4, 5], sorted(names)
    for name, lines in names.items():
        text = "\n".join(lines)
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in text, (name, text)
