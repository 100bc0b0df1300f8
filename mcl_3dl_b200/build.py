"""Build the in-tree CUDA engine: mcl_3dl_b200/libmcl3dl_b200.so (sm_90a, H100, only).

nvcc cross-compiles without a GPU; the .so is a build product (git-ignored).
-fmad=false: the DDA stepping and the SE(3) transform must round exactly like the reference's
x86-64 Release build (no FMA contraction); see csrc/device_math.cuh.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libmcl3dl_b200.so")
SOURCES = [os.path.join(CSRC, "engine.cu")]
DEPS = SOURCES + [os.path.join(CSRC, "kernels.cuh"), os.path.join(CSRC, "device_funcs.cuh"),
                  os.path.join(CSRC, "device_math.cuh"), os.path.join(CSRC, "pf_kernels.cuh"), os.path.join(CSRC, "pf_funcs.cuh"),
                  os.path.join(CSRC, "scan_kernels.cuh"), os.path.join(CSRC, "scan_funcs.cuh"), os.path.join(CSRC, "match_funcs.cuh"),
                  os.path.join(CSRC, "accum_funcs.cuh"), os.path.join(CSRC, "window_funcs.cuh"),
                  os.path.join(os.path.dirname(HERE), "include", "mcl3dl_b200.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-fmad=false", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared"]


def stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(d) > t for d in DEPS)


def build(force=False, verbose=False, defines=(), out=None):
    """defines/out: build an experiment variant (e.g. defines=["MCL_FAST_DIV=0"], out="/tmp/x.so")."""
    if not force and not stale() and out is None:
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = ([nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-D" + d for d in defines]
           + ["-o", out or LIB] + SOURCES)
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n%s\n%s" % (r.stdout, r.stderr))
    if verbose:
        print(r.stderr)
    return out or LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
