"""CPU side of tests/test_generic_voxel_windows_gpu.py: the general window oracle (tests/helpers.py: WindowRun,
box_features, box_mcc) equals the reference pipeline on whole small volumes for every setting the GPU file runs, the
planted corpus reaches every MCC row count and capacity condition of the generic kernel at r = 2 and r = 3, and the
generic kernel's math compiled for the host (tests/host_emul, emul_voxel_features) stays within the GPU file's bounds on
a smaller corpus of every setting -- so the bounds and the asymmetric-MCC solve are shown here before a GPU runs."""
import ctypes as C
import os
import subprocess
from collections import Counter

import numpy as np
import pytest

import pipeline as PL
from helpers import (FAST_NAMES, MCC_ATOL, WindowRun, alive_mask_bruteforce, assert_mcc_reach, block_corpus, box_features,
                     box_imc2_independent, box_mcc, box_references, compare_box_maps, mcc_matrix, mcc_over_capacity,
                     mcc_reach, plant_boxes, reach_corpus, remap_boxes, weighted_overflow, window_box)
from pyradiomics_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
SPACING_ZYX = (2.0, 0.8, 0.6)

# the settings of the GPU file, on whole small volumes
SETTINGS = [
    ("r2", dict(kernelRadius=2)),
    ("r3", dict(kernelRadius=3)),
    ("r3-d2", dict(kernelRadius=3, distances=(2,))),
    ("r3-d13", dict(kernelRadius=3, distances=(1, 3))),
    ("r2-d3", dict(kernelRadius=2, distances=(3,))),
    ("r2-d123", dict(kernelRadius=2, distances=(1, 2, 3))),
    ("asym-r1", dict(kernelRadius=1, symmetricalGLCM=False)),
    ("asym-r3", dict(kernelRadius=3, symmetricalGLCM=False)),
    ("manhattan-r2", dict(kernelRadius=2, weightingNorm="manhattan", spacing_zyx=SPACING_ZYX)),
    ("euclidean-r1", dict(kernelRadius=1, weightingNorm="euclidean", spacing_zyx=SPACING_ZYX)),
    ("infinity-r3", dict(kernelRadius=3, weightingNorm="infinity", spacing_zyx=SPACING_ZYX)),
    ("no_weighting-r2", dict(kernelRadius=2, weightingNorm="no_weighting", spacing_zyx=SPACING_ZYX)),
    ("force2D0-r2", dict(kernelRadius=2, force2D=True, force2Ddimension=0)),
    ("force2D1-r3", dict(kernelRadius=3, force2D=True, force2Ddimension=1)),
    ("force2D2-r2", dict(kernelRadius=2, force2D=True, force2Ddimension=2, gldm_a=3)),
]


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul") / "libemul.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", so,
                           os.path.join(HERE, "host_emul", "emul.cpp")])
    return C.CDLL(so)


def _volume(shape=(6, 7, 8), n_levels=12, seed=0):
    """i.i.d. levels with a plateau, 10 % holes, levels 1 and n_levels present (binWidth = 1 binning is the identity)"""
    rng = np.random.default_rng(seed)
    lev = rng.integers(1, n_levels + 1, shape)
    z = min(1, shape[0] - 1)
    lev[z, :3, :4] = lev[z, 0, 0]
    lev[rng.random(shape) < 0.1] = 0
    lev.reshape(-1)[[1, -2]] = 1, n_levels
    return lev


@pytest.mark.parametrize("name,kw", SETTINGS, ids=[s[0] for s in SETTINGS])
def test_box_oracle_equals_pipeline_extract(name, kw):
    """box_features / box_mcc of every ROI voxel's window (faces and holes included) against oracle/pipeline.extract on
    the whole volume: 1e-12 (MCC 1e-7: the reference's eigvals of a non-symmetric Q; Imc2 where no angle has exactly
    independent margins)"""
    lev = _volume(seed=len(name))
    mask = lev > 0
    vox = np.array(np.where(mask)).astype(np.int32)
    vox = vox[:, np.r_[0:12, vox.shape[1] - 12:vox.shape[1], 150:162]]
    run = WindowRun(lev.shape, int(lev.max()), **kw).alive_from(lev)
    boxes = [window_box(lev, c, run.radii) for c in vox.T]
    indep = np.array([box_imc2_independent(b, run) for b in boxes])
    for cname, names in FAST_NAMES.items():
        ref = PL.extract(cname, lev, mask, voxelBased=True, binWidth=1, voxels=vox, **kw)
        got = [box_features(b, cname, run) for b in boxes]
        for f in names:
            if f == "MCC":
                g = np.array([box_mcc(b, run)[0] for b in boxes])
                assert np.allclose(g, ref[f], rtol=0, atol=1e-7, equal_nan=True), (name, f)
                continue
            g = np.array([x[f] for x in got])
            sel = ~indep if f == "Imc2" else np.ones(len(boxes), bool)
            assert np.allclose(g[sel], ref[f][sel], rtol=1e-12, atol=0, equal_nan=True), (name, cname, f)


def test_box_oracle_two_d_image_equals_pipeline_extract():
    """a 2-D image: pipeline.extract on the 2-D arrays, the box oracle on its one plane"""
    lev = _volume((1, 9, 11), seed=3)
    mask = lev > 0
    vox = np.array(np.where(mask[0])).astype(np.int32)
    run = WindowRun(lev.shape, int(lev.max()), kernelRadius=2).alive_from(lev)
    boxes = [window_box(lev, (0, y, x), run.radii) for y, x in vox.T]
    indep = np.array([box_imc2_independent(b, run) for b in boxes])
    for cname, names in FAST_NAMES.items():
        ref = PL.extract(cname, lev[0], mask[0], voxelBased=True, binWidth=1, kernelRadius=2)
        for f in names:
            if f == "MCC":
                g = np.array([box_mcc(b, run)[0] for b in boxes])
                assert np.allclose(g, ref[f], rtol=0, atol=1e-7, equal_nan=True), f
                continue
            g = np.array([box_features(b, cname, run)[f] for b in boxes])
            sel = ~indep if f == "Imc2" else np.ones(len(boxes), bool)
            assert np.allclose(g[sel], ref[f][sel], rtol=1e-12, atol=0, equal_nan=True), (cname, f)


@pytest.mark.parametrize("r", [2, 3])
def test_corpus_reaches_every_mcc_size_and_capacity_condition(r):
    """helpers.reach_corpus(r), the corpus whose every MCC the GPU file checks (test_mcc_of_the_reach_corpus): per angle
    >= 100 MCC problems (connected, at least two rows and columns) of every row count 2..32, and >= 100 problems of more
    than 32 rows, bipartite and disconnected level graphs; pooled weighted windows over each entry-list limit"""
    run = WindowRun((40, 40, 40), 400, kernelRadius=r)
    assert_mcc_reach(mcc_reach(box_mcc(b, run)[1] for b in reach_corpus(r)), f"r{r}")
    # the weighted limits (status bit 1): 16-bit levels spread widely, r = 3, distances {1, 2, 3}
    if r == 3:
        wrun = WindowRun((7, 7, 7), 65535, kernelRadius=3, distances=(1, 2, 3), weightingNorm="euclidean")
        rng = np.random.default_rng(9)
        kinds = Counter()
        for n in (40, 45, 48):
            lv = np.sort(rng.choice(np.arange(1, 65536), n, replace=False))
            box = lv[rng.permutation(np.arange(343) % n)].reshape(7, 7, 7)
            pairs = set()
            from helpers import box_pairs
            for a in wrun.angles:
                x, y = box_pairs(box, a)
                pairs.update(zip(x.tolist(), y.tolist()))
                pairs.update(zip(y.tolist(), x.tolist()))
            sums = len({i + j for i, j in pairs})
            kinds[(len(pairs) > 2048, sums > 1024)] += 1
            assert weighted_overflow(box, wrun) == (len(pairs) > 2048 or sums > 1024)
        assert kinds[(False, True)] and kinds[(True, True)] and kinds[(False, False)], kinds


def _emul_run(emul, boxes, what, Ng=None, classes=FAST_NAMES, alphas=(0, 3, 255), **kw):
    """the GPU file's run_planted through the host-compiled generic math (emul_voxel_features with `centers`)"""
    vol, cen = plant_boxes(boxes)
    Ng = Ng or int(vol.max())
    run = WindowRun(vol.shape, Ng, **kw)
    centers = np.zeros(vol.shape, bool)
    centers[tuple(cen.T)] = True
    boxes = [window_box(vol, c, run.radii) for c in cen]
    if run.weights is not None:
        keep = np.array([not weighted_overflow(b, run) for b in boxes])
        boxes, cen = [b for b, k in zip(boxes, keep) if k], cen[keep]
        centers[:] = False
        centers[tuple(cen.T)] = True
    run.alive_from(vol, centers)
    alive = np.zeros(_lib.ALIVE_WORDS, np.uint32)
    for a in np.flatnonzero(run.alive):
        alive[a >> 5] |= np.uint32(1 << (a & 31))
    lev = np.ascontiguousarray(vol, np.uint16)
    cm = np.ascontiguousarray(centers, np.uint8)
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    worst = {}
    for cname in classes:
        for a in (alphas if cname == "gldm" else (0,)):
            run.gldm_a = a
            refs = box_references(boxes, run, classes=[cname], mcc=cname == "glcm")
            out = np.zeros((len(FAST_NAMES[cname]),) + vol.shape)
            s = run.settings(len(np.unique(vol[vol > 0])))
            st = emul.emul_voxel_features(_lib.CLASS_ID[cname], p(lev), p(cm), *vol.shape, C.byref(s), p(alive), p(out))
            assert st == (int(refs["mcc_over"].any()) if cname == "glcm" else 0), (what, cname, st)
            worst[(cname, a)] = compare_box_maps(out[(slice(None),) + tuple(cen.T)], refs, cname, a, what, run)
    return worst


EMUL_CASES = [
    ("r2", dict(kernelRadius=2), 5, None),
    ("r3", dict(kernelRadius=3), 7, None),
    ("r3-d123", dict(kernelRadius=3, distances=(1, 2, 3)), 7, None),
    ("r2-d3", dict(kernelRadius=2, distances=(3,)), 5, None),
    ("asym-r1", dict(kernelRadius=1, symmetricalGLCM=False), 3, None),
    ("asym-r2", dict(kernelRadius=2, symmetricalGLCM=False), 5, None),
    ("asym-r3", dict(kernelRadius=3, symmetricalGLCM=False), 7, None),
    ("euclidean-r2", dict(kernelRadius=2, weightingNorm="euclidean", spacing_zyx=SPACING_ZYX), 5, None),
    ("manhattan-r3", dict(kernelRadius=3, weightingNorm="manhattan", spacing_zyx=SPACING_ZYX), 7, None),
    ("force2D1-r3", dict(kernelRadius=3, force2D=True, force2Ddimension=1), 7, None),
    ("Ng65535-r2", dict(kernelRadius=2), 5, 65535),
]


@pytest.mark.parametrize("name,kw,side,Ng", EMUL_CASES, ids=[c[0] for c in EMUL_CASES])
def test_emulated_generic_math_within_gpu_bounds(emul, name, kw, side, Ng):
    n = 150 if side == 3 else 16
    boxes = block_corpus(n, side, seed=len(name), K_max=64 if kw.get("distances") else None)
    if Ng:
        boxes, _ = remap_boxes(boxes, Ng, np.random.default_rng(1))
    _emul_run(emul, boxes, name, Ng=Ng, classes=["glcm"] if "asym" in name else FAST_NAMES, **kw)


# ---------------------------------------------------------------------------------- MCC of one matrix, deterministic
def _matrix_mcc(emul, M, symmetric):
    """(MCC, status) of one GLCM through the generic kernel's per-angle math (emul_glcm_matrix_mcc)"""
    M = np.ascontiguousarray(M, np.float64)
    st = C.c_int(0)
    emul.emul_glcm_matrix_mcc.restype = C.c_double
    v = emul.emul_glcm_matrix_mcc(M.ctypes.data_as(C.c_void_p), M.shape[0], int(symmetric), C.byref(st))
    return v, st.value


def _square(T, n=None):
    """an r x c table as the top-left block of an n x n level matrix (rows and columns are levels 1..n)"""
    T = np.asarray(T, float)
    n = n or max(T.shape)
    M = np.zeros((n, n))
    M[:T.shape[0], :T.shape[1]] = T
    return M


def test_asymmetric_mcc_is_the_second_singular_value(emul):
    """the rank-1 table [[10,25,5],[4,10,2],[8,20,4]] (exact MCC 0; sqrt(lambda_2(M M^T)) gives 1.8e-8), and 3 000
    seeded asymmetric tables of two and three rows -- near rank-1 ones among them, where squaring costs most --
    against the exact second singular value at MCC_ATOL"""
    v, st = _matrix_mcc(emul, _square([[10, 25, 5], [4, 10, 2], [8, 20, 4]]), False)
    assert st == 0 and abs(v) <= MCC_ATOL, v
    rng = np.random.default_rng(4)
    worst = 0.0
    for it in range(3000):
        n = 2 + it % 2
        if it % 3 == 0:
            T = np.outer(rng.integers(1, 6, n), rng.integers(1, 6, n)).astype(float)
            T[rng.integers(n), rng.integers(n)] += rng.integers(0, 2)
        elif it % 3 == 1:
            T = rng.integers(0, 6, (n, n)).astype(float)
        else:
            T = rng.integers(0, 4, (n, n + 1 + it % 3)).astype(float)
        M = _square(T)
        ref = mcc_matrix(M)
        if ref is None:
            continue
        v, st = _matrix_mcc(emul, M, False)
        assert st == 0
        worst = max(worst, abs(v - ref[0]))
        assert abs(v - ref[0]) <= MCC_ATOL, (T, v, ref)
    print("asymmetric 2- and 3-row tables: worst |MCC error|", worst)


def test_matrix_mcc_capacity_rule(emul):
    """one row or one column level is 0 without a solve whatever the other side holds; a connected problem with more
    than 32 rows or more than 32 columns is NaN with status bit 0; 32 x 32 is solved"""
    rng = np.random.default_rng(5)
    col = rng.integers(1, 5, (34, 1))
    for T in (col, col.T):                                  # 34 x 1 and 1 x 34
        v, st = _matrix_mcc(emul, _square(T), False)
        assert (v, st) == (0.0, 0), (T.shape, v, st)
    for shape in ((33, 2), (2, 33)):                        # connected: every entry positive
        v, st = _matrix_mcc(emul, _square(rng.integers(1, 4, shape)), False)
        assert np.isnan(v) and st == 1, (shape, v, st)
    T = rng.integers(1, 4, (32, 32)).astype(float)
    for sym in (False, True):
        M = T + T.T if sym else T
        v, st = _matrix_mcc(emul, M, sym)
        ref = mcc_matrix(M)
        assert st == 0 and not ref[5] and abs(v - ref[0]) <= MCC_ATOL, (sym, v, ref)


def _single_column_volume():
    """7^3 at r = 3: the x = 0 plane holds 33 distinct levels (2..34), every other voxel level 1.  The centre's angle
    (0, 0, 1) pairs 34 row levels with the single column level 1 (MCC 0 without a solve); the angles inside the plane
    see at most 32 of its levels (a unique level in the middle of each border line) next to the isolated pair (1, 1)"""
    plane = np.zeros((7, 7), np.int64)
    mids = [(0, 3), (6, 3), (3, 0), (3, 6)]
    rest = [(z, y) for z in range(7) for y in range(7) if (z, y) not in mids]
    for k, zy in enumerate(rest):
        plane[zy] = 2 + k % 29
    for k, zy in enumerate(mids):
        plane[zy] = 31 + k
    lev = np.ones((7, 7, 7), np.int64)
    lev[:, :, 0] = plane
    return lev


@pytest.mark.parametrize("case", ["r2-L48", "r3-L64", "r3-single-column"])
def test_asymmetric_mcc_capacity_through_emulation(emul, case):
    """symmetricalGLCM=False: MCC NaN exactly on the voxels helpers.mcc_over_capacity(symmetricalGLCM=False) names,
    status bit 0 exactly when there is one, every other voxel's MCC the reference's (1e-7: its eigvals of a
    non-symmetric Q)"""
    from helpers import envelope_volume
    if case == "r3-single-column":
        lev, r = _single_column_volume(), 3
    else:
        r, n = int(case[1]), int(case.split("L")[1])
        lev = envelope_volume(n)
    mask = lev != 0
    Ng = int(lev.max())
    s = _lib.make_settings(Ng, len(np.unique(lev[mask])), kernelRadius=r, symmetricalGLCM=False)
    alive = alive_mask_bruteforce(lev, mask, __import__("cmatrices_oracle").generate_angles(lev.shape, [1], 0, False, 0),
                                  [r] * 3)
    over = mcc_over_capacity(lev, mask, r, symmetricalGLCM=False)
    if case == "r3-single-column":
        assert not over[np.ravel_multi_index((3, 3, 3), lev.shape)]
    else:
        assert over.any()
    lev16 = np.ascontiguousarray(lev, np.uint16)
    out = np.zeros((len(FAST_NAMES["glcm"]),) + lev.shape)
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    st = emul.emul_voxel_features(0, p(lev16), None, *lev.shape, C.byref(s), p(alive), p(out))
    assert st == int(over.any()), st
    got = out[FAST_NAMES["glcm"].index("MCC")][mask]
    assert np.array_equal(np.isnan(got), over)
    ref = PL.extract("glcm", lev, mask, voxelBased=True, binWidth=1, kernelRadius=r, symmetricalGLCM=False)["MCC"]
    assert np.allclose(got[~over], ref[~over], rtol=0, atol=1e-7)
