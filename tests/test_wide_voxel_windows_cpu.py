"""CPU side of tests/test_wide_voxel_windows_gpu.py: the window oracle (tests/helpers.py: WindowRun, box_features,
box_mcc) equals the reference pipeline at kernelRadius 4, 5 and 7 on whole small volumes (faces, holes, a 2-D image,
force2D); the rule that sends windows to the generic or the wide kernels, at its edges; and the oracle's cost per
window at kernelRadius 7, which sizes the GPU file's corpora."""
import ctypes as C
import os
import subprocess
import time

import numpy as np
import pytest

import pipeline as PL
from helpers import FAST_NAMES, WindowRun, block_corpus, box_features, box_imc2_independent, box_mcc, box_references, window_box
from pyradiomics_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
GENERIC, WIDE, UNSUPPORTED = 0, 1, 2


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul") / "libwindowpath.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, os.path.join(HERE, "host_emul", "window_path_emul.cpp")])
    lib = C.CDLL(so)
    lib.emul_window_path.argtypes = [C.c_int, C.c_int]
    lib.emul_window_positions.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    return lib


def _volume(shape, n_levels=12, seed=0):
    """i.i.d. levels with a plateau, 10 % holes, levels 1 and n_levels present (binWidth = 1 binning is the identity)"""
    rng = np.random.default_rng(seed)
    lev = rng.integers(1, n_levels + 1, shape)
    z = min(1, shape[0] - 1)
    lev[z, :3, :4] = lev[z, 0, 0]
    lev[rng.random(shape) < 0.1] = 0
    lev.reshape(-1)[[1, -2]] = 1, n_levels
    return lev


def _compare(lev, mask, run, boxes, what, vox=None, **kw):
    indep = np.array([box_imc2_independent(b, run) for b in boxes])
    for cname, names in FAST_NAMES.items():
        if vox is None:
            ref = PL.extract(cname, lev[0] if lev.shape[0] == 1 else lev, mask[0] if lev.shape[0] == 1 else mask,
                             voxelBased=True, binWidth=1, **kw)
        else:
            ref = PL.extract(cname, lev, mask, voxelBased=True, binWidth=1, voxels=vox, **kw)
        got = [box_features(b, cname, run) for b in boxes]
        for f in names:
            if f == "MCC":
                g = np.array([box_mcc(b, run)[0] for b in boxes])
                assert np.allclose(g, ref[f], rtol=0, atol=1e-7, equal_nan=True), (what, f)
                continue
            g = np.array([x[f] for x in got])
            sel = ~indep if f == "Imc2" else np.ones(len(boxes), bool)
            assert np.allclose(g[sel], ref[f][sel], rtol=1e-12, atol=0, equal_nan=True), (what, cname, f)


SETTINGS = [
    ("r4", dict(kernelRadius=4)),
    ("r5", dict(kernelRadius=5)),
    ("r7", dict(kernelRadius=7)),
    ("r5-force2D0", dict(kernelRadius=5, force2D=True, force2Ddimension=0)),
    ("r7-force2D2", dict(kernelRadius=7, force2D=True, force2Ddimension=2, gldm_a=2)),
]


@pytest.mark.parametrize("name,kw", SETTINGS, ids=[s[0] for s in SETTINGS])
def test_box_oracle_equals_pipeline_extract(name, kw):
    """box_features / box_mcc of ROI voxels' windows (clipped by the faces of a volume smaller than the window, with
    holes) against oracle/pipeline.extract on the whole volume: 1e-12 (MCC 1e-7, Imc2 where no angle has exactly
    independent margins), as tests/test_generic_voxel_windows_cpu.py"""
    lev = _volume((7, 9, 10), seed=len(name))
    mask = lev > 0
    vox = np.array(np.where(mask)).astype(np.int32)
    vox = vox[:, np.r_[0:8, vox.shape[1] - 8:vox.shape[1], 200:208]]
    run = WindowRun(lev.shape, int(lev.max()), **kw).alive_from(lev)
    _compare(lev, mask, run, [window_box(lev, c, run.radii) for c in vox.T], name, vox=vox, **kw)


def test_box_oracle_two_d_image_equals_pipeline_extract():
    """a 2-D image at kernelRadius 5: pipeline.extract on the 2-D arrays, the box oracle on its one plane"""
    lev = _volume((1, 12, 13), seed=3)
    mask = lev > 0
    run = WindowRun(lev.shape, int(lev.max()), kernelRadius=5).alive_from(lev)
    vox = np.array(np.where(mask[0]))
    _compare(lev, mask, run, [window_box(lev, (0, y, x), run.radii) for y, x in vox.T], "2D", kernelRadius=5)


def test_window_path_rule(emul):
    """host_common.hpp window_path: generic up to 343 positions, wide from 344 to 3375, refused beyond; the forced wide
    path takes the generic windows too"""
    for cap, want in ((27, GENERIC), (343, GENERIC), (344, WIDE), (3375, WIDE), (3376, UNSUPPORTED), (4913, UNSUPPORTED)):
        assert emul.emul_window_path(cap, 0) == want, cap
    for cap, want in ((27, WIDE), (343, WIDE), (3375, WIDE), (3376, UNSUPPORTED)):
        assert emul.emul_window_path(cap, 1) == want, cap


@pytest.mark.parametrize("kw,positions,path", [
    (dict(kernelRadius=3), 343, GENERIC),
    (dict(kernelRadius=4), 729, WIDE),
    (dict(kernelRadius=7), 3375, WIDE),
    (dict(kernelRadius=8), 4913, UNSUPPORTED),
    (dict(kernelRadius=9, force2D=True, force2Ddimension=1), 361, WIDE),
    (dict(kernelRadius=12, force2D=True, force2Ddimension=0), 625, WIDE),
    (dict(kernelRadius=28, force2D=True, force2Ddimension=2), 3249, WIDE),
    (dict(kernelRadius=29, force2D=True, force2Ddimension=2), 3481, UNSUPPORTED),
], ids=["r3", "r4", "r7", "r8", "2D-r9", "2D-r12", "2D-r28", "2D-r29"])
def test_window_positions_of_each_radius(emul, kw, positions, path):
    """the positions fill_vox_params gives every class's window, and the path the rule picks for them: texture and
    first order ask the same rule about the same (2rz+1)(2ry+1)(2rx+1)"""
    s = _lib.make_settings(8, 8, **kw)
    for cls in range(5):
        assert emul.emul_window_positions(cls, 64, 64, 64, C.byref(s)) == positions
    assert emul.emul_window_path(positions, 0) == path


def test_oracle_cost_per_window_at_r7():
    """the window oracle's cost per 15^3 window (every class and MCC), measured here on the GPU file's corpus (blocks
    of more than 400 distinct levels replaced by 200 i.i.d. levels: the dense oracle of 3375 levels takes ~20 s a
    window): the GPU file checks 22 such windows at r = 7 by default and 22 more with 16-bit levels, which must stay
    well inside its run time"""
    rng = np.random.default_rng(7)
    boxes = [b if len(np.unique(b)) <= 400 else np.where(b > 0, rng.integers(1, 201, b.shape), 0)
             for b in block_corpus(11, 15, seed=7)]
    run = WindowRun((15, 15, 15), int(max(b.max() for b in boxes)), kernelRadius=7)
    box_references(boxes[:1], run)                              # warm-up
    t = time.perf_counter()
    box_references(boxes, run)
    per = (time.perf_counter() - t) / len(boxes)
    print(f"window oracle at r = 7: {per * 1e3:.1f} ms per window (all classes and MCC)")
    assert per * 44 < 120, per
