"""Build libb200newton.so (hand-written sm_90a CUDA + the C ABI) in-tree with nvcc.

    python nonlinearsolve.jl_b200/build.py [--force]

The .so lands next to this file (git-ignored); object files go to build/ beside it.
"""
import concurrent.futures
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
INCLUDE = os.path.join(HERE, "..", "include")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libb200newton.so")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _deps():
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    return hdrs + [os.path.join(INCLUDE, "b200newton.h"), os.path.abspath(__file__)]


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(p) > t for p in sources() + _deps())


def _compile(src, verbose):
    obj = os.path.join(OBJ, os.path.basename(src)[:-3] + ".o")
    dep_t = max(os.path.getmtime(p) for p in [src] + _deps())
    if os.path.exists(obj) and os.path.getmtime(obj) >= dep_t:
        return obj, ""
    host_cc = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    cmd = [_nvcc(), *ARCH, "-O3", "-lineinfo", "-std=c++17", "-ccbin", host_cc, "-Xcompiler", "-fPIC,-O2,-Wall", "-Xptxas", "-v" if verbose else "-O3",
           "-I", INCLUDE, "-c", src, "-o", obj]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s" % (src, r.stdout))
    return obj, r.stdout


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    os.makedirs(OBJ, exist_ok=True)
    if force:
        for f in os.listdir(OBJ):
            os.remove(os.path.join(OBJ, f))
    with concurrent.futures.ThreadPoolExecutor(max_workers=8) as ex:
        results = list(ex.map(lambda s: _compile(s, verbose), sources()))
    objs = [o for o, _ in results]
    if verbose:
        for _, out in results:
            sys.stdout.write(out)
    host_cc = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    cmd = [_nvcc(), *ARCH, "-shared", "-ccbin", host_cc, "-cudart", "shared", "-Xlinker", "-rpath,/usr/local/cuda/lib64", "-o", LIB, *objs, "-ldl"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s" % r.stdout)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
