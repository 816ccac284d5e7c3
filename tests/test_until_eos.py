"""The end-of-utterance rule (data_load.utterance_lengths / eos_positions) on the host, and the ptxas report of the decode
kernel that applies it in its frame loop."""
import os
import re
import subprocess

import numpy as np
import pytest

from dc_tts_b200.data_load import eos_positions, load_data, text_normalize, utterance_lengths
from dc_tts_b200.hyperparams import Hyperparams as hp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_rule_never_reached():
    m = np.array([[0, 0, 1, 1, 2, 2]])
    assert utterance_lengths(m, [3]).tolist() == [6]
    assert utterance_lengths(m, [-1]).tolist() == [6]                  # < 0: never
    assert utterance_lengths(m, [-1], tail=3).tolist() == [6]


def test_rule_reached_at_first_and_last_frame():
    m = np.array([[0, 1, 1, 2, 3, 4]])
    assert utterance_lengths(m, [0]).tolist() == [1]                   # frame 0 already reaches it
    assert utterance_lengths(m, [4]).tolist() == [6]                   # only the last frame does
    assert utterance_lengths(m, [4], tail=2).tolist() == [6]           # the tail runs past steps: clamped
    assert utterance_lengths(m, [0], tail=2).tolist() == [3]


def test_rule_jump_over_stop_position():
    m = np.array([[0, 0, 2, 4, 4, 5, 5, 5]])
    assert utterance_lengths(m, [1]).tolist() == [3]                   # 0 -> 2 jumps over 1: frame 2 is the first >= 1
    assert utterance_lengths(m, [3]).tolist() == [4]
    assert utterance_lengths(m, [3], tail=7).tolist() == [8]


def test_rule_steps_and_batch():
    m = np.array([[0, 1, 2, 3, 4, 5], [0, 0, 0, 0, 0, 0], [5, 5, 5, 5, 5, 5]])
    assert utterance_lengths(m, [3, 1, 2], tail=1).tolist() == [5, 6, 2]
    assert utterance_lengths(m, [3, 1, 2], tail=1, steps=3).tolist() == [3, 3, 2]   # frames past `steps` do not count
    with pytest.raises(ValueError):
        utterance_lengths(m, [0, 0, 0], tail=-1)


def test_rule_prefix_is_the_stepwise_loop():
    """The step-wise synthesize loop applies the rule to the history fetched so far and stops once every utterance has
    ended: on a prefix that long the rule already gives the lengths of the whole history."""
    rng = np.random.default_rng(0)
    T = 60
    for trial in range(200):
        B = 5
        m = np.cumsum(rng.integers(0, 3, (B, T)) * (rng.random((B, T)) < 0.3), axis=1)
        sp = rng.integers(-1, 12, B)
        tail = int(rng.integers(0, 6))
        full = utterance_lengths(m, sp, tail, steps=T)
        stop = T
        for j in range(T):
            n = utterance_lengths(m[:, :j + 1], sp, tail, steps=T)
            if (n <= j + 1).all():
                stop = j + 1
                assert np.array_equal(n, full), (trial, j)
                break
        assert stop == full.max()


def test_eos_positions_harvard():
    L = load_data("synthesize", os.path.join(ROOT, "harvard_sentences.txt"))
    with open(os.path.join(ROOT, "harvard_sentences.txt"), encoding="utf-8") as f:
        sents = [text_normalize(line.split(" ", 1)[-1]).strip() for line in f.readlines()[1:]]
    eos = eos_positions(L)
    assert eos.dtype == np.int32 and len(eos) == 20
    assert eos.tolist() == [len(s) for s in sents]
    assert (L[np.arange(20), eos] == hp.vocab.index("E")).all()
    assert 33 <= eos.min() + 1 and eos.max() + 1 <= 50                   # 33-50 ids with the EOS
    no_eos = L.copy()
    no_eos[3] = 2
    assert eos_positions(no_eos)[3] == -1


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    from dc_tts_b200 import build
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    obj = str(tmp_path_factory.mktemp("ptxas") / "kernels_decode.o")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-c", os.path.join(build.CSRC, "kernels_decode.cu"), "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stderr


def test_until_kernel_no_stack_no_spills(ptxas_log):
    """Every utterance count of decode_until_kernel: no stack frame and no spills, like decode_cluster_kernel."""
    out, cur = {}, None
    for line in ptxas_log.splitlines():
        m = re.search(r"(?:Compiling entry function|Function properties for) '?(\w+)'?", line)
        if m:
            cur = m.group(1) if "decode_until_kernel" in m.group(1) else None
            if cur:
                out.setdefault(cur, [])
            continue
        if cur:
            out[cur].append(line)
    assert sorted(int(re.search(r"Li(\d)E", n).group(1)) for n in out) == [1, 2, 3, 4, 5], sorted(out)
    for name, lines in out.items():
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in "\n".join(lines), name
