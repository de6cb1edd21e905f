"""Builds libstrolle_b200.so (CUDA kernels + host engine + C ABI) in-tree with nvcc for sm_90a (H100).

    python -m strolle_b200.build [--force]

Flags that matter for parity: -fmad=false (device) and -ffp-contract=off (host) keep every
float operation a single IEEE-754 operation in source order.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT_DIR = os.path.join(HERE, "_lib")
LIB = os.path.join(OUT_DIR, "libstrolle_b200.so")
# (source, object stem, extra flags): kernels.cu is built twice — strict IEEE (namespace st) and the fast-shading flavour of the
# ReSTIR kernels (namespace stf: FMA contraction, approximate div/sqrt, SFU transcendentals; traversal stays bit-exact, st_math.cuh)
UNITS = [("kernels.cu", "kernels", ["-fmad=false"]),
         ("kernels.cu", "kernels_fast", ["-DST_FAST=1", "-fmad=true", "-prec-div=false", "-prec-sqrt=false"]),
         ("refit.cu", "refit", ["-fmad=false"]),
         ("engine.cu", "engine", ["-fmad=false"])]
HEADERS = ["st_math.cuh", "st_device.cuh", "st_types.h", "kernels.h", os.path.join("..", "..", "include", "strolle_b200.h")]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O3", "-lineinfo",
         "-Xcompiler", "-fPIC,-ffp-contract=off,-fno-fast-math,-O2", "-Xptxas", "-v"]


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, defines=(), tag=""):
    """tag/defines: tuning builds (e.g. tag="minb8", defines=["ST_MINB_ALL=8"]) -> _lib/libstrolle_b200_<tag>.so."""
    os.makedirs(OUT_DIR, exist_ok=True)
    deps = [os.path.join(CSRC, h) for h in HEADERS] + [os.path.abspath(__file__)]
    objs = []
    procs = []
    suffix = ("_" + tag) if tag else ""
    lib = LIB.replace(".so", suffix + ".so")
    flags = FLAGS + ["-D" + d for d in defines]
    for src, stem, extra in UNITS:
        obj = os.path.join(OUT_DIR, stem + suffix + ".o")
        objs.append(obj)
        if force or _stale(obj, deps + [os.path.join(CSRC, src)]):
            cmd = [NVCC] + flags + extra + ["-c", os.path.join(CSRC, src), "-o", obj]
            procs.append((stem, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for stem, p in procs:
        out, _ = p.communicate()
        with open(os.path.join(OUT_DIR, stem + suffix + ".ptxas.log"), "w") as f:
            f.write(out)
        if p.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError("nvcc failed for " + stem)
        if verbose:
            print(out)
    if force or procs or _stale(lib, objs):
        subprocess.check_call([NVCC, "-shared", "-o", lib] + objs + ["-lcudart_static", "-ldl", "-lrt", "-lpthread", "-Xlinker", "--no-undefined"])
    return lib


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
