"""Builds libfenerf_b200.so (the C-ABI library of include/fenerf_b200.h) in-tree with nvcc for sm_90a.

One object per translation unit under build/ (so edits rebuild only what changed), linked into
fenerf_b200/libfenerf_b200.so.  No torch involvement: the library has a plain C ABI.
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OBJ_DIR = os.path.join(ROOT, "build", "obj")
LIB_PATH = os.path.join(HERE, "libfenerf_b200.so")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr",
    "-DFENERF_BUILDING_LIB",
]
# experiment builds: FENERF_NVCC_DEFINES="-DFOO=1 ..." + FENERF_B200_LIB=<output .so>
NVCC_FLAGS += os.environ.get("FENERF_NVCC_DEFINES", "").split()
if os.environ.get("FENERF_B200_LIB"):
    LIB_PATH = os.path.abspath(os.environ["FENERF_B200_LIB"])
    OBJ_DIR = os.path.join(ROOT, "build", "obj_" + os.path.basename(LIB_PATH).replace(".so", ""))


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest(paths):
    h = hashlib.sha256()
    for p in paths:
        with open(p, "rb") as f:
            h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def _headers():
    hs = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".h", ".cuh"))]
    hs.append(os.path.join(ROOT, "include", "fenerf_b200.h"))
    return hs


def _compile_one(src, verbose):
    obj = os.path.join(OBJ_DIR, src[:-3] + ".o")
    stamp = obj + ".sha"
    want = _digest([os.path.join(CSRC, src)] + _headers())
    if os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == want:
        return obj, False
    cmd = [NVCC] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(CSRC, src), "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
    if verbose:
        sys.stderr.write(r.stderr)
    with open(stamp, "w") as f:
        f.write(want)
    return obj, True


def build(force=False, verbose=False):
    """Compile every CUDA translation unit for sm_90a and link the shared library. Returns its path."""
    os.makedirs(OBJ_DIR, exist_ok=True)
    if force:
        for f in os.listdir(OBJ_DIR):
            os.remove(os.path.join(OBJ_DIR, f))
    srcs = _sources()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(lambda s: _compile_one(s, verbose), srcs))
    objs = [o for o, _ in results]
    if any(changed for _, changed in results) or not os.path.exists(LIB_PATH):
        cmd = [NVCC, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB_PATH] + objs
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
