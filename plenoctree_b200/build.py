"""In-tree build of libplenoctree_b200.so (explicit nvcc, sm_90a only).

`python -m plenoctree_b200.build` compiles every .cu under csrc/ that is newer than its object
and links the shared library next to this file.  nvcc cross-compiles without a GPU.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libplenoctree_b200.so")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _deps_mtime():
    heads = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    heads.append(os.path.join(HERE, "..", "include", "plenoctree_b200.h"))
    return max(os.path.getmtime(h) for h in heads)


# per-file extra flags (none at present; octree.cu pins its rounding with __fmul_rn/__fadd_rn instead of --fmad=false)
EXTRA = {}


def _compile(src, verbose):
    obj = os.path.join(OBJ, src[:-3] + ".o")
    cmd = [NVCC] + FLAGS + EXTRA.get(src, []) + ["-c", os.path.join(CSRC, src), "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    log = r.stdout + r.stderr
    with open(obj + ".log", "w") as f:
        f.write(log)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{log}")
    if verbose:
        for line in log.splitlines():
            if "registers" in line or "spill" in line.lower() and " 0 bytes spill" not in line:
                print(f"[{src}] {line.strip()}")
    return obj


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    hdr = _deps_mtime()
    todo, objs = [], []
    for src in _sources():
        obj = os.path.join(OBJ, src[:-3] + ".o")
        objs.append(obj)
        sm = max(os.path.getmtime(os.path.join(CSRC, src)), hdr)
        if force or not os.path.exists(obj) or os.path.getmtime(obj) < sm:
            todo.append(src)
    if todo:
        with ThreadPoolExecutor(max_workers=min(8, len(todo))) as ex:
            list(ex.map(lambda s: _compile(s, verbose), todo))
    if todo or not os.path.exists(LIB):
        cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
