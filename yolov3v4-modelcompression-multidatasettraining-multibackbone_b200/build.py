"""Build libb200yolo.so (sm_90a only) in-tree with nvcc.

    python build.py            # incremental: rebuilds only when a source is newer than the .so
    python build.py --force

The shared library travels to the GPU box with the repo snapshot (it is git-ignored, not gpurun-ignored).
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")
OUT = os.path.join(HERE, "libb200yolo.so")
OBJ_DIR = os.path.join(HERE, "build")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-O3", "-std=c++17", "-lineinfo",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr", "--extended-lambda",
    "-I", INCLUDE, "-I", CSRC,
]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def headers():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hs.append(os.path.join(INCLUDE, "b200yolo.h"))
    return hs


def _compile(src, verbose):
    obj = os.path.join(OBJ_DIR, os.path.basename(src)[:-3] + ".o")
    dep_m = max(os.path.getmtime(p) for p in [src] + headers())
    if os.path.exists(obj) and os.path.getmtime(obj) >= dep_m:
        return obj
    cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("nvcc failed for %s" % src)
    if verbose:
        sys.stderr.write(r.stderr)
    return obj


def build(force=False, verbose=False):
    os.makedirs(OBJ_DIR, exist_ok=True)
    srcs = sources()
    if force:
        for f in os.listdir(OBJ_DIR):
            os.remove(os.path.join(OBJ_DIR, f))
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(lambda s: _compile(s, verbose), srcs))
    if (not os.path.exists(OUT)) or any(os.path.getmtime(o) > os.path.getmtime(OUT) for o in objs):
        cmd = [NVCC, "-shared", "-o", OUT] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
