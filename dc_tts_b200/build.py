"""In-tree build of libdctts_b200.so (nvcc, sm_90a only).

`python -m dc_tts_b200.build` or `__graft_entry__.build()`.  The .so is written next to
this file, so that the package is importable from the source tree; it is git-ignored.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libdctts_b200.so")
SOURCES = ["dctts_api.cu", "api_params.cu", "api_synth.cu", "api_train.cu", "api_audio.cu", "kernels_simt.cu", "kernels_tc.cu", "kernels_attn_tc.cu", "kernels_vocoder.cu", "kernels_train.cu", "kernels_ordered.cu", "kernels_decode.cu", "kernels_gemm_tc.cu", "kernels_pack.cu", "kernels_align.cu", "kernels_mcd.cu", "kernels_longform.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--use_fast_math" if False else "-DDCTTS_NO_FAST_MATH",     # accuracy first: no fast-math
    "-Xcompiler", "-fPIC,-O3,-Wall", "-Xptxas", "-v", "--expt-relaxed-constexpr",
]


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    raise RuntimeError("nvcc not found")


def _stale(out, deps):
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hdrs.append(os.path.join(HERE, "..", "include", "dctts.h"))
    objs = []
    log = []
    for s in srcs:
        o = os.path.join(CSRC, os.path.basename(s)[:-3] + ".o")
        if force or _stale(o, [s] + hdrs + [os.path.abspath(__file__)]):
            cmd = [_nvcc()] + NVCC_FLAGS + ["-c", s, "-o", o]
            r = subprocess.run(cmd, capture_output=True, text=True)
            log.append(r.stderr)
            if r.returncode != 0:
                sys.stderr.write(r.stdout + r.stderr)
                raise RuntimeError("nvcc failed for %s" % s)
            if verbose:
                sys.stderr.write(r.stderr)
        objs.append(o)
    if force or _stale(LIB, objs):
        cmd = [_nvcc(), "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a",
                                                         "-cudart", "static", "-Xcompiler", "-fPIC"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    return LIB, "".join(log)


if __name__ == "__main__":
    lib, log = build(force="--force" in sys.argv, verbose=True)
    print(lib)
