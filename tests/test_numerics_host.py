"""The host side of csrc/numerics.cuh, which both weight packers run: split_f16 / join_f16 bit for bit against numpy's
round-to-nearest-even float16 emulation (the one tests/test_split_fp16_scheme.py rests on), and weight_scale against
2^(11 - frexp(max)[1]).  A host-only program that includes the header is compiled with the package's nvcc flags (no
-gencode: it needs no GPU) and run on generated inputs."""
import subprocess

import numpy as np
import pytest

from dc_tts_b200 import build

PROGRAM = r"""
#include "numerics.cuh"
#include <cmath>
#include <cstdio>
#include <cstring>
// argv[1]: float32 inputs; argv[2]: per input hi bits, lo bits (uint16), join_f16(hi, lo), weight_scale(|x|) (float32)
int main(int argc, char** argv) {
    if (argc != 3) return 2;
    FILE* in = fopen(argv[1], "rb");
    FILE* out = fopen(argv[2], "wb");
    if (!in || !out) return 3;
    float x;
    while (fread(&x, sizeof x, 1, in) == 1) {
        __half hi, lo;
        dctts::split_f16(x, hi, lo);
        unsigned short bits[2];
        memcpy(&bits[0], &hi, 2);
        memcpy(&bits[1], &lo, 2);
        const float r[2] = {dctts::join_f16(hi, lo), dctts::weight_scale(std::fabs(x))};
        fwrite(bits, 2, 2, out);
        fwrite(r, 4, 2, out);
    }
    fclose(in);
    return fclose(out) == 0 ? 0 : 4;
}
"""
RECORD = np.dtype([("hi", "<u2"), ("lo", "<u2"), ("join", "<f4"), ("scale", "<f4")])


@pytest.fixture(scope="module")
def host_numerics(tmp_path_factory):
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    d = tmp_path_factory.mktemp("numerics")
    src, exe = str(d / "numerics_host.cu"), str(d / "numerics_host")
    with open(src, "w") as f:
        f.write(PROGRAM)
    flags, skip = [], False
    for a in build.NVCC_FLAGS:
        if skip or a == "-gencode":
            skip = not skip
            continue
        flags.append(a)
    r = subprocess.run([nvcc] + flags + ["-I", build.CSRC, src, "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]

    def run(x):
        x = np.ascontiguousarray(x, dtype=np.float32)
        x.tofile(str(d / "in.bin"))
        r = subprocess.run([exe, str(d / "in.bin"), str(d / "out.bin")], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        out = np.fromfile(str(d / "out.bin"), dtype=RECORD)
        assert out.shape == x.shape
        return out
    return run


def _inputs():
    rng = np.random.default_rng(0)
    normals = (10.0 ** rng.uniform(-30, 5, 200000)).astype(np.float32)
    normals *= rng.choice(np.float32([-1, 1]), normals.size)
    # exact ties halfway between neighbouring fp16 values: round-to-nearest-even decides hi
    h = rng.uniform(-60000, 60000, 20000).astype(np.float16)
    ties = ((h.astype(np.float64) + np.nextafter(h, np.float16(np.inf)).astype(np.float64)) / 2).astype(np.float32)
    sub_bits = rng.integers(1, 0x800000, 20000, dtype=np.uint32)
    subnormals = np.concatenate([sub_bits, sub_bits | 0x80000000]).view(np.float32)
    special = np.float32([0.0, -0.0, 65504, -65504, 65520, -65520, np.inf, -np.inf, np.nan, 2 ** -24, 2 ** -25, 6.1e-5])
    return np.concatenate([normals, ties[np.isfinite(ties)], subnormals, special])


def _same(got_bits, want_bits, nan_mask):
    return np.array_equal(got_bits[~nan_mask], want_bits[~nan_mask])


def test_split_and_join_match_numpy_float16_rounding(host_numerics):
    x = _inputs()
    out = host_numerics(x)
    with np.errstate(invalid="ignore", over="ignore"):
        hi = x.astype(np.float16)
        lo = (x - hi.astype(np.float32)).astype(np.float16)
        join = hi.astype(np.float32) + lo.astype(np.float32)
    got_hi, got_lo, got_join = out["hi"].view(np.float16), out["lo"].view(np.float16), out["join"]
    for got, want in ((got_hi, hi), (got_lo, lo), (got_join, join)):
        assert np.array_equal(np.isnan(got), np.isnan(want))
        assert _same(got.view(np.uint16 if got.dtype == np.float16 else np.uint32),
                     want.view(np.uint16 if want.dtype == np.float16 else np.uint32), np.isnan(want))
    # the cases the format's edges turn on
    at = {v: i for i, v in enumerate(x[-12:].tolist()) if v == v}
    base = x.size - 12
    assert out["hi"][base + at[65504.0]] == 0x7BFF and out["lo"][base + at[65504.0]] == 0
    assert np.isposinf(got_hi[base + at[65520.0]]) and np.isneginf(got_lo[base + at[65520.0]])
    assert out["hi"][base + 1] == 0x8000 and out["lo"][base + 1] == 0x0000          # -0 -> (-0, +0)
    assert np.isnan(got_hi[base + 8]) and np.isnan(got_join[base + 8])


def test_weight_scale_is_the_power_of_two_below_2_to_the_11(host_numerics):
    x = _inputs()
    x = x[np.isfinite(x)]
    out = host_numerics(x)
    m = np.abs(x)
    with np.errstate(over="ignore"):
        want = np.where(m > 0, 2.0 ** (11 - np.frexp(m)[1].astype(np.float64)), 1.0).astype(np.float32)
    assert np.array_equal(out["scale"].view(np.uint32), want.view(np.uint32))
    normal = (m >= np.finfo(np.float32).tiny) & (m < 2.0 ** 117)
    scaled = m[normal].astype(np.float64) * out["scale"][normal]
    assert scaled.min() >= 2.0 ** 10 and scaled.max() < 2.0 ** 11
