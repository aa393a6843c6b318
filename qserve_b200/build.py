"""Build libqserve_b200.so (sm_90a only) in-tree with nvcc.

The shared library is the product: a C-ABI (include/qserve_b200.h) with no torch or Python dependency.
`python -m qserve_b200.build` rebuilds it; `ensure_built()` is what `__graft_entry__.build()` calls.
Objects are cached per source file under qserve_b200/_build/ and rebuilt when a source or header changes.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "_build")
LIB = os.path.join(HERE, "libqserve_b200.so")
SOURCES = ["capi.cu", "gemm.cu", "attention.cu", "prefill_attention.cu", "prefix_attention.cu", "multi_token_attention.cu", "tree_verify.cu", "kv_fork.cu", "beam_search.cu", "inflight.cu", "sampling.cu", "speculative.cu", "elementwise.cu"]
HEADERS = ["common.cuh", "launch.h", "launch.cuh", "paged_attention.cuh", "prompt_attention.cuh", os.path.join("..", "..", "include", "qserve_b200.h")]

NVCC_FLAGS = [
    "-std=c++17", "-O3", "-lineinfo",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def _digest(paths) -> str:
    h = hashlib.sha256()
    for p in paths:
        with open(p, "rb") as f:
            h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()[:16]


def _compile(src: str, verbose: bool) -> str:
    path = os.path.join(CSRC, src)
    deps = [path] + [os.path.join(CSRC, h) for h in HEADERS]
    tag = _digest(deps)
    obj = os.path.join(BUILD, f"{os.path.splitext(src)[0]}.{tag}.o")
    if not os.path.exists(obj):
        for old in os.listdir(BUILD):
            if old.startswith(os.path.splitext(src)[0] + ".") and old.endswith(".o"):
                os.remove(os.path.join(BUILD, old))
        cmd = [_nvcc(), "-c", path, "-o", obj] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else [])
        res = subprocess.run(cmd, capture_output=True, text=True)
        if verbose or res.returncode != 0:
            sys.stderr.write(res.stdout + res.stderr)
        if res.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}")
    return obj


def ensure_built(verbose: bool = False, force: bool = False) -> str:
    os.makedirs(BUILD, exist_ok=True)
    if force:
        for f in os.listdir(BUILD):
            os.remove(os.path.join(BUILD, f))
    with ThreadPoolExecutor(max_workers=4) as ex:
        objs = list(ex.map(lambda s: _compile(s, verbose), SOURCES))
    stamp = os.path.join(BUILD, "link.stamp")
    want = " ".join(sorted(objs))
    have = open(stamp).read() if os.path.exists(stamp) else ""
    if want != have or not os.path.exists(LIB):
        cmd = [_nvcc(), "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static", "-Xcompiler", "-fPIC"]
        subprocess.check_call(cmd)
        with open(stamp, "w") as f:
            f.write(want)
    return LIB


if __name__ == "__main__":
    print(ensure_built(verbose="-v" in sys.argv, force="--force" in sys.argv))
