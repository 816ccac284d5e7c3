"""Compiles kernels_train.cu with the package's nvcc flags and reads ptxas's report for every kernel of the training step's
backward, losses and optimiser, each instantiation of train_block_bwd_kernel included: no stack frame, no spills.

train_block_bwd_kernel<33, true> (highway blocks up to 1056 channels) holds six 33-float arrays per thread and sits at the
255-register limit; a spill there would turn its register arrays into local-memory traffic on every row."""
import os
import re
import subprocess

import pytest

from dc_tts_b200 import build

KERNELS = ["train_dropout_kernel", "train_loss_kernel", "sigmoid_rows_kernel", "conv_wgrad_kernel", "transpose_w_kernel",
           "attn_bwd_q_kernel", "attn_bwd_kv_kernel", "attn_loss_kernel", "guided_attention_kernel", "embed_bwd_kernel",
           "adam_kernel"]
# MAXV, HC of each train_block_bwd_kernel instantiation launch_train_block_bwd uses (mangled: ILi<MAXV>ELb<HC>E)
BLOCK_BWD = [(4, 1), (8, 1), (16, 1), (32, 1), (33, 1), (65, 0)]


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    obj = str(tmp_path_factory.mktemp("ptxas") / "kernels_train.o")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-c", os.path.join(build.CSRC, "kernels_train.cu"), "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stderr


def _report(log, match):
    lines, cur = [], False
    for line in log.splitlines():
        m = re.search(r"(?:Compiling entry function|Function properties for) '?(\w+)'?", line)
        if m:
            cur = match(m.group(1))
            continue
        if cur:
            lines.append(line)
    return "\n".join(lines)


def _assert_clean(log, text):
    assert "Used" in text, log[-4000:]
    assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in text, text


@pytest.mark.parametrize("kernel", KERNELS)
def test_train_kernel_no_stack_no_spills(ptxas_log, kernel):
    _assert_clean(ptxas_log, _report(ptxas_log, lambda name: re.search(r"\d%s" % kernel, name) is not None))


@pytest.mark.parametrize("maxv,hc", BLOCK_BWD, ids=lambda v: str(v))
def test_block_bwd_instantiation_no_stack_no_spills(ptxas_log, maxv, hc):
    tag = "train_block_bwd_kernelILi%dELb%dE" % (maxv, hc)
    _assert_clean(ptxas_log, _report(ptxas_log, lambda name: tag in name))


def test_every_kernel_of_the_file_is_checked(ptxas_log):
    """A kernel added to kernels_train.cu (or a new instantiation) has to be added above."""
    names = set(re.findall(r"Compiling entry function '(\w+)'", ptxas_log))
    covered = {n for n in names if any(re.search(r"\d%s" % k, n) for k in KERNELS)}
    covered |= {n for n in names if any("train_block_bwd_kernelILi%dELb%dE" % b in n for b in BLOCK_BWD)}
    assert names == covered, names - covered
