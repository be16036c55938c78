"""The eigen-task kernels' ORCHESTRATION on the CPU box: tests/host_emul/solve_kernel_emul.cpp runs the text of
csrc/glcm_kernels.cuh with one std::thread per CUDA thread (barriers as barriers, shared memory as static
storage): the tile counting sort, the size groups, the block-uniform dense solves with their barriers and the register
Lanczos groups (per-thread shared vectors) must hand every queued task to exactly one solver and reproduce the direct solve."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import bench

HERE = os.path.dirname(os.path.abspath(__file__))


_LIBS = {}


def _solve_lib():
    if "solve" in _LIBS:                   # never overwrite a library this process has loaded
        return _LIBS["solve"]
    so = os.path.join(HERE, "host_emul", "libsolve_emul.so")
    src = os.path.join(HERE, "host_emul", "solve_kernel_emul.cpp")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-pthread", "-Wno-unknown-pragmas", "-shared", "-fPIC", "-o", so + ".%d" % os.getpid(), src])
    os.replace(so + ".%d" % os.getpid(), so)
    _LIBS["solve"] = C.CDLL(so)
    return _LIBS["solve"]


@pytest.mark.parametrize("kind,n", [("smooth", 12), ("uniform", 16)])
def test_emulated_solve_kernels_process_every_task_once(kind, n):
    lib = _solve_lib()
    lev = np.ascontiguousarray(bench.synth_volume(40, kind)[:n, :n, :n].astype(np.uint8))
    cap = 100000
    rk, rd, cls = np.zeros(cap), np.zeros(cap), np.zeros(cap, np.int32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    nt = lib.emul_solve_kernels(p(lev), n, n, n, 32, 3, cap, p(rk), p(rd), p(cls))
    assert 800 < nt < cap
    rk, rd, cls = rk[:nt], rd[:nt], cls[:nt]
    assert not (rk == -12345.0).any(), "a queued task was not picked up by any solve kernel"
    assert not np.isnan(rk).any()
    # bit-identical to the direct solve: both solve a task with the size template its class fixes
    assert np.array_equal(rk, rd)
    hist = np.bincount(cls, minlength=16)
    assert hist[:7].sum() and hist[7:11].sum() and hist[11:].sum()      # all three kernels had work


@pytest.mark.parametrize("kind,n", [("smooth", 12), ("uniform", 14)])
def test_emulated_glcm_pipeline_equals_per_voxel_math(kind, n):
    """phase A kernel (per-angle barriers, atomic queue reservation, non-centre voxels) -> three solve kernels -> finish
    kernel, in plane chunks like glcm_fast_run, against the single-thread composition of the same math
    (emul_fast, itself pinned on the reference's voxel-mode maps in test_host_emul.py)"""
    from pyradiomics_b200 import _lib
    pipe = _solve_lib()
    pipe.emul_glcm_pipeline.restype = C.c_longlong
    so = os.path.join(HERE, "host_emul", "libemul_pipe.so")          # own copy: test_host_emul.py rebuilds libemul.so
    if "emul" not in _LIBS:
        subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", so + ".%d" % os.getpid(), os.path.join(HERE, "host_emul", "emul.cpp")])
        os.replace(so + ".%d" % os.getpid(), so)
        _LIBS["emul"] = C.CDLL(so)
    emul = _LIBS["emul"]
    lev = np.ascontiguousarray(bench.synth_volume(40, kind)[:n, :n, :n].astype(np.uint8))
    if kind == "smooth":
        lev[3:6, 2:9, 5] = 0                      # holes: voxels that are not centres, windows with missing pairs
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    out = np.zeros((24, n, n, n))
    ntasks = pipe.emul_glcm_pipeline(p(lev), n, n, n, 32, 5, p(out))           # 3 plane chunks
    assert ntasks > 700
    ref = np.zeros((24, n, n, n))
    s = _lib.make_settings(32, 32)
    lev16 = lev.astype(np.uint16)
    assert emul.emul_fast(0, p(lev16), n, n, n, C.byref(s), None, p(ref)) == 0
    for k, name in enumerate(_lib.feature_names("glcm")):
        assert np.array_equal(out[k], ref[k], equal_nan=True), name
