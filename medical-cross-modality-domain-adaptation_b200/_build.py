"""In-tree build of the sm_90a (H100) shared library (libpnp_b200.so) with nvcc.

nvcc cross-compiles without a GPU, so the library can be built on a machine without one; the resulting .so and
the objects under build/ are git-ignored build products."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libpnp_b200.so")
SOURCES = ["conv_simt.cu", "elementwise.cu", "conv_tc.cu", "surface.cu", "metrics3d.cu", "resample.cu", "components3d.cu"]
HEADERS = [os.path.join(CSRC, "common.cuh"), os.path.join(os.path.dirname(HERE), "include", "pnp_b200.h")]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + [ "-O3", "-std=c++17", "-lineinfo",
              "-Xcompiler", "-fPIC", "-diag-suppress", "177"]


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=True):
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    nvcc = _nvcc()
    jobs = []
    objs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(objdir, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _stale(o, [s] + HEADERS):
            jobs.append([nvcc] + NVCC_FLAGS + ["-c", s, "-o", o])

    def run(cmd):
        if verbose:
            print("[pnp_b200 build]", " ".join(cmd), file=sys.stderr)
        subprocess.run(cmd, check=True)

    if jobs:
        with ThreadPoolExecutor(max_workers=len(jobs)) as ex:
            list(ex.map(run, jobs))
    if force or jobs or _stale(LIB, objs):
        run([nvcc] + ARCH + ["-shared", "-o", LIB] + objs + ["-cudart", "static"])
    build_io(force, run)
    return LIB


IO_LIB = os.path.join(HERE, "libpnp_io.so")


def build_io(force=False, run=None):
    """libpnp_io.so: the host-side TFRecord decoder (plain C, gcc; no CUDA dependency) -- include/pnp_io.h"""
    src = os.path.join(CSRC, "tfrecord_io.c")
    hdr = os.path.join(os.path.dirname(HERE), "include", "pnp_io.h")
    if force or _stale(IO_LIB, [src, hdr]):
        cmd = [os.environ.get("CC", "gcc"), "-O3", "-std=c11", "-fPIC", "-shared", "-Wall", "-o", IO_LIB, src]
        if run is None:
            subprocess.run(cmd, check=True)
        else:
            run(cmd)
    return IO_LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
