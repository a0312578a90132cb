"""Build libsorobn_b200.so (hand-written sm_90a kernels + C ABI) in-tree with nvcc.

No torch, no pybind: the library's only dependency is the CUDA runtime (linked
statically), so it loads with ctypes from any process.
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(HERE)
LIB = os.path.join(PKG, "libsorobn_b200.so")
SOURCES = [os.path.join(HERE, f) for f in ("sbn_api.cu", "sbn_tiled_u0.cu", "sbn_tiled_u1.cu", "sbn_tiled_u2.cu", "sbn_tiled_c.cu",
                                            "sbn_chain.cu", "sbn_tma.cu", "sbn_pair.cu", "sbn_triple_rows.cu", "sbn_contract.cu",
                                            "sbn_join.cu", "sbn_tally.cu", "sbn_bp.cu")]
HEADERS = [os.path.join(HERE, h) for h in ("sbn_kernels.cuh", "sbn_gibbs.cuh", "sbn_chain.h", "sbn_tma.h", "sbn_pair.h", "sbn_join.h", "sbn_internal.h", "sbn_launch.h",
                                            "sbn_launch_impl.cuh", "sbn_marginal.cuh", "sbn_count.cuh", "sbn_deriv.cuh", "sbn_sample.cuh",
                                            "sbn_mpe.cuh", "sbn_soft.cuh")] + [
    os.path.join(os.path.dirname(PKG), "include", "sorobn_b200.h")]
OBJ_DIR = os.path.join(HERE, "build")
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]  # H100 (Hopper)


def nvcc_path() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def up_to_date() -> bool:
    if not os.path.exists(LIB):
        return False
    t = os.path.getmtime(LIB)
    return all(os.path.getmtime(f) <= t for f in SOURCES + HEADERS + [os.path.abspath(__file__)])


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(f) > t for f in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile every translation unit for sm_90a (in parallel, each only when it is stale) and link
    libsorobn_b200.so in-tree."""
    if not force and up_to_date():
        return LIB
    from concurrent.futures import ThreadPoolExecutor

    os.makedirs(OBJ_DIR, exist_ok=True)
    flags = ["-Xcompiler", "-fPIC", "-O3", "-std=c++17", "-lineinfo", *GENCODE,
             "-Xptxas", "-v" if verbose else "-O3"]

    def compile_one(src):
        obj = os.path.join(OBJ_DIR, os.path.basename(src)[:-3] + ".o")
        if not force and not _stale(obj, [src, *HEADERS, os.path.abspath(__file__)]):
            return obj, None
        res = subprocess.run([nvcc_path(), "-c", *flags, "-o", obj, src], capture_output=True, text=True)
        if res.returncode != 0:
            if os.path.exists(obj):
                os.remove(obj)
            return obj, res.stdout + res.stderr
        if verbose:
            sys.stderr.write(res.stdout + res.stderr)
        return obj, None

    with ThreadPoolExecutor(len(SOURCES)) as pool:
        results = list(pool.map(compile_one, SOURCES))
    errors = [err for _, err in results if err]
    if errors:
        sys.stderr.write("\n".join(errors))
        raise RuntimeError("nvcc failed building libsorobn_b200.so")
    res = subprocess.run([nvcc_path(), "-shared", *GENCODE, "-o", LIB,
                          *[obj for obj, _ in results]], capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("linking libsorobn_b200.so failed")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
