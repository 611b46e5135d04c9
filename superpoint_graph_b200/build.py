"""In-tree build of libspg_b200.so (sm_90a only, nvcc cross-compiles without a GPU).

    python -m superpoint_graph_b200.build [--force]

Objects go to build/ (git-ignored); the shared library lands next to this file so that it
travels with the repository snapshot to the GPU box.  With SPG_REFERENCE set to a reference
checkout, the recipe oracle/build_ref.py also compiles the reference's own `prune` into
oracle/_ref/ (git-ignored) for the tests to compare against; it runs as a separate process,
so the product never imports the oracle.
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OBJ_DIR = os.path.join(ROOT, "build", "obj")
LIB_PATH = os.path.join(HERE, "libspg_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def _nvcc():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found; cannot build libspg_b200.so")
    return nvcc


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _deps_mtime():
    m = 0.0
    for f in os.listdir(CSRC):
        if f.endswith((".cuh", ".h")):
            m = max(m, os.path.getmtime(os.path.join(CSRC, f)))
    m = max(m, os.path.getmtime(os.path.join(ROOT, "include", "spg_b200.h")))
    return m


def build(force=False, verbose=True):
    nvcc = _nvcc()
    os.makedirs(OBJ_DIR, exist_ok=True)
    dep_m = _deps_mtime()
    objs, rebuilt = [], False
    for src in sources():
        obj = os.path.join(OBJ_DIR, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        if (not force and os.path.exists(obj)
                and os.path.getmtime(obj) >= max(os.path.getmtime(src), dep_m)):
            continue
        cmd = [nvcc] + NVCC_FLAGS + ["-c", src, "-o", obj]
        if verbose:
            print("[spg build]", " ".join(cmd), flush=True)
        subprocess.check_call(cmd)
        rebuilt = True
    if rebuilt or force or not os.path.exists(LIB_PATH):
        cmd = [nvcc, "-shared", "-cudart", "shared", "-o", LIB_PATH] + objs + [
            "-Xlinker", "-rpath,/usr/local/cuda/lib64"]
        if verbose:
            print("[spg build]", " ".join(cmd), flush=True)
        subprocess.check_call(cmd)
    _build_reference(force, verbose)
    return LIB_PATH


def _build_reference(force, verbose):
    if not os.environ.get("SPG_REFERENCE"):
        return
    recipe = os.path.join(ROOT, "oracle", "build_ref.py")
    out = os.path.join(ROOT, "oracle", "_ref", "libply_c_prune.so")
    if not force and os.path.exists(out) and os.path.getmtime(out) >= os.path.getmtime(recipe):
        return
    if verbose:
        print("[spg build]", sys.executable, recipe, flush=True)
    subprocess.check_call([sys.executable, recipe])


if __name__ == "__main__":
    build(force="--force" in sys.argv)
    print(LIB_PATH)
