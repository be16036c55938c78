"""Builds libb200radiomics.so in-tree with nvcc for sm_90a (no JIT cache: the .so travels with
the repository snapshot to the GPU box)."""
from __future__ import annotations

import glob
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb200radiomics.so")
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-diag-suppress", "128",
]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = glob.glob(os.path.join(CSRC, "*")) + [os.path.join(HERE, "..", "include", "b200radiomics.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def _compile_and_link(out: str, objdir: str, verbose: bool = False) -> None:
    """one nvcc per .cu in parallel (the translation units are independent: no relocatable device code), then link"""
    from concurrent.futures import ThreadPoolExecutor

    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    os.makedirs(objdir, exist_ok=True)
    jobs = []
    for src in sources():
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        jobs.append((src, obj, [nvcc, *NVCC_FLAGS, *(["-Xptxas", "-v"] if verbose else []), "-c", src, "-o", obj]))
    with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
        for rc in ex.map(lambda j: subprocess.call(j[2], cwd=CSRC), jobs):
            if rc:
                raise RuntimeError("nvcc failed")
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", out, *[j[1] for j in jobs]], cwd=CSRC)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        if os.path.exists(LIB):
            return LIB
        raise RuntimeError("nvcc not found and libb200radiomics.so is not built")
    _compile_and_link(LIB, os.path.join(HERE, "build"), verbose)
    return LIB


if __name__ == "__main__":
    import sys

    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
