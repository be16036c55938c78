"""CPU side of tests/test_fast_voxel_windows_gpu.py: the window oracle equals the reference pipeline, the planted corpus
reaches every MCC task class of the fast path, and the fast and generic kernels' arithmetic compiled for the host
(tests/host_emul)
stays within the bounds the GPU test applies -- so those bounds are shown to hold before anything runs on a GPU."""
import ctypes as C
import os
import subprocess
from collections import Counter

import numpy as np
import pytest

import pipeline as PL
from helpers import (FAST_NAMES, GLDM_ALPHAS, compare_window_maps, imc2_angles, ng_corpus, plant, planted_corpus,
                     window_at, window_features, window_mcc, window_references)
from pyradiomics_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
NGS = (2, 3, 32, 33, 128, 254, 255)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul") / "libemul.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", so,
                           os.path.join(HERE, "host_emul", "emul.cpp")])
    return C.CDLL(so)


def _seeded_volume(Ng, holes, shape=(5, 6, 7), seed=0):
    """i.i.d. levels 1..Ng with 1 and Ng present (binWidth = 1 binning is then the identity); `holes` zeroes a tenth"""
    rng = np.random.default_rng(seed + Ng)
    lev = rng.integers(1, Ng + 1, shape)
    if Ng > 3:                                      # runs of equal levels too: long GLRLM runs, GLSZM zones, dependences
        lev[1, :3, :4] = lev[1, 0, 0]
    if holes:
        lev[rng.random(shape) < 0.1] = 0
    lev[0, 0, 1], lev[-1, -1, -2] = 1, Ng
    return lev


@pytest.mark.parametrize("holes", [False, True], ids=["full", "holes"])
@pytest.mark.parametrize("Ng", [32, 255])
def test_window_oracle_equals_pipeline_extract(Ng, holes):
    """window_features / window_mcc of every voxel's 3x3x3 window (faces and ROI holes included) against
    oracle/pipeline.extract on the whole volume: 1e-12 (MCC 1e-7: the reference's eigvals of a non-symmetric Q)"""
    lev = _seeded_volume(Ng, holes)
    mask = lev > 0
    vox = np.array(np.where(mask)).astype(np.int32)
    if Ng == 255:                                   # the oracle's Ng x Ng per voxel and angle: a subset, faces first
        vox = vox[:, np.r_[0:20, vox.shape[1] - 20:vox.shape[1], 60:80]]
    wins = [window_at(lev, c) for c in vox.T]
    indep = np.array([any(i for _, i in imc2_angles(w)) for w in wins])
    # a window with an empty angle: the reference's JointAverage is NaN when that angle is alive in the voxel batch
    # (pipeline.extract's batches here) and window_features takes all 13 alive; compared on full-angle windows only
    empty = np.array([sum(r is not None for r in window_mcc(w)[1]) < 13 for w in wins])
    assert (~indep).sum() > 0 and (~empty).sum() > 0
    for cname, names in FAST_NAMES.items():
        for a in ((0, 3) if cname == "gldm" else (0,)):
            ref = {}
            for c0 in range(0, vox.shape[1], 20):
                r = PL.extract(cname, lev, mask, voxelBased=True, binWidth=1, gldm_a=a, voxels=vox[:, c0:c0 + 20])
                for f, v in r.items():
                    ref.setdefault(f, []).append(v)
            ref = {f: np.concatenate(v) for f, v in ref.items()}
            got = [window_features(w, Ng, cname, a) for w in wins]
            for f in names:
                if f == "MCC":
                    g = np.array([window_mcc(w)[0] for w in wins])
                    assert np.allclose(g, ref[f], rtol=0, atol=1e-7, equal_nan=True), (Ng, f)
                    continue
                g = np.array([x[f] for x in got])
                sel = ~indep if f == "Imc2" else ~empty if f == "JointAverage" else np.ones(len(wins), bool)
                assert np.allclose(g[sel], ref[f][sel], rtol=1e-12, atol=0, equal_nan=True), (Ng, holes, cname, a, f)


def test_planted_corpus_reaches_every_task_class():
    """node counts 2..19 all occur; >= 100 connected non-bipartite eigen-tasks at each Lanczos size 13..18; >= 100 trees
    of 13 levels (12-pair angles) and of 19 levels (18-pair angles); bipartite and disconnected graphs occur"""
    cnt = Counter()
    for w in planted_corpus(10500, seed=0):
        for s, r in enumerate(window_mcc(w)[1]):
            if r is not None:
                npairs = 18 if s < 3 else 12 if s < 9 else 8
                cnt[(r[1], r[2], r[3], npairs)] += 1
    nodes = Counter()
    for (n, conn, bip, npairs), k in cnt.items():
        nodes[n] += k
    assert all(nodes[n] > 0 for n in range(2, 20)), nodes
    task = lambda n: sum(k for (m, conn, bip, _), k in cnt.items() if m == n and conn and not bip)
    assert all(task(n) >= 100 for n in range(13, 19)), {n: task(n) for n in range(13, 19)}
    assert cnt[(13, True, True, 12)] >= 100 and cnt[(19, True, True, 18)] >= 100
    assert sum(k for (n, conn, bip, _), k in cnt.items() if conn and bip and n < 13) >= 100
    assert sum(k for (n, conn, bip, _), k in cnt.items() if not conn) >= 100


def _emulated_kernel_math_within_gpu_bounds(emul, Ng, path):
    """the fast paths' math (emul_fast) or the generic kernels' math
    (emul_voxel_features) on a planted corpus against the window oracle, at the bounds of
    tests/test_fast_voxel_windows_gpu.py (helpers.window_bound, helpers.compare_window_maps)"""
    wins, _ = ng_corpus(planted_corpus(1500, seed=1), Ng, 400, np.random.default_rng(Ng))
    vol, cen = plant(wins)
    assert vol.max() == Ng
    refs = window_references(wins, Ng)
    lev = np.ascontiguousarray(vol, np.uint16)
    Zs, Ys, Xs = lev.shape
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    alive = np.zeros(_lib.ALIVE_WORDS, np.uint32)
    alive[0] = (1 << 13) - 1                            # every angle alive in the planted volume
    for cid, cname in enumerate(_lib.CLASSES):
        for a in (GLDM_ALPHAS if cname == "gldm" else (0,)):
            s = _lib.make_settings(Ng, len(np.unique(vol[vol > 0])), gldm_a=a)
            out = np.zeros((len(FAST_NAMES[cname]), Zs, Ys, Xs))
            if path == "generic":
                rc = emul.emul_voxel_features(cid, p(lev), None, Zs, Ys, Xs, C.byref(s), p(alive), p(out))
            else:
                rc = emul.emul_fast(cid, p(lev), Zs, Ys, Xs, C.byref(s), p(alive), p(out))
            assert rc == 0
            compare_window_maps(out[(slice(None),) + tuple(cen.T)], refs, cname, a, f"Ng={Ng}/{path}/gldm_a={a}",
                                path == "generic")


@pytest.mark.parametrize("Ng", NGS)
def test_emulated_fast_math_within_gpu_bounds(emul, Ng):
    _emulated_kernel_math_within_gpu_bounds(emul, Ng, "fast")


@pytest.mark.parametrize("Ng", NGS)
def test_emulated_generic_math_within_gpu_bounds(emul, Ng):
    """the generic kernels' MCC included: 1e-9 on windows of two and three levels too"""
    _emulated_kernel_math_within_gpu_bounds(emul, Ng, "generic")
