"""Build libsnn_b200.so (hand-written sm_90a CUDA + C++ host engine) in-tree with nvcc.

Objects are cached under shadernn_b200/csrc/build/ keyed on source mtime; the shared library lands at
shadernn_b200/libsnn_b200.so (git-ignored build product).
"""
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(CSRC, "build")
LIB = os.path.join(HERE, "libsnn_b200.so")

SOURCES = [
    "kernels_simt.cu",
    "kernels_umma.cu",
    "pack.cpp",
    "conv_plan.cpp",
    "capi.cpp",
    "engine/modelparser.cpp",
    "engine/layers.cpp",
    "engine/dp.cpp",
    "engine/core.cpp",
    "engine/model_capi.cpp",
]
HEADERS = ["snnb_internal.h", "engine/engine.h", "engine/json.h", "../../include/snnb.h"]

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-std=c++17", "-O3", "-lineinfo", "-Xcompiler", "-fPIC", "-Xcompiler", "-pthread", "-Xcompiler", "-Wall", "-I", os.path.join(ROOT, "include"), "-I", CSRC]


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: libsnn_b200 cannot be built (there is no CPU fallback)")


def _host_cxx():
    # the image exports CXX=/opt/gcc/bin/g++ (a wrapper); the system g++ is what nvcc is validated against
    return "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"


def _newest_header_mtime():
    m = 0.0
    for h in HEADERS:
        p = os.path.join(CSRC, h)
        if os.path.exists(p):
            m = max(m, os.path.getmtime(p))
    return m


def _compile_one(nvcc, src, hdr_mtime, verbose):
    obj = os.path.join(BUILD, src.replace("/", "_") + ".o")
    spath = os.path.join(CSRC, src)
    if os.path.exists(obj) and os.path.getmtime(obj) > max(os.path.getmtime(spath), hdr_mtime):
        return obj
    cmd = [nvcc, "-ccbin", _host_cxx()] + ARCH + COMMON + ["-c", spath, "-o", obj]
    if src.endswith(".cu"):
        cmd += ["-Xptxas", "-v"] if verbose else []
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout[-4000:], r.stderr[-8000:]))
    if verbose and r.stderr:
        sys.stderr.write(r.stderr)
    return obj


def build(verbose=False, force=False):
    """Compile every source for sm_90a and link libsnn_b200.so. Returns the library path."""
    os.makedirs(BUILD, exist_ok=True)
    nvcc = _nvcc()
    hdr = _newest_header_mtime()
    if force:
        for f in os.listdir(BUILD):
            os.remove(os.path.join(BUILD, f))
    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        objs = list(ex.map(lambda s: _compile_one(nvcc, s, hdr, verbose), SOURCES))
    if (not os.path.exists(LIB)) or any(os.path.getmtime(o) > os.path.getmtime(LIB) for o in objs):
        cmd = [nvcc, "-ccbin", _host_cxx()] + ARCH + ["-shared", "-o", LIB] + objs + ["-lcudart", "-lcuda", "-lpthread", "-ldl"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout[-4000:], r.stderr[-8000:]))
    return LIB


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv))
