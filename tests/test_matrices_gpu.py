"""GPU parity of the cMatrices drop-in (matrix level, integer entries BIT-EXACT): against the
oracle port on random inputs (segment + voxel batches, 2-D/3-D, distances, force2D), against the
reference's own golden matrices, and against the dense per-voxel matrices of the reference."""
import json
import os

import numpy as np
import pytest

import cmatrices_oracle as O
import features_np as F
import pipeline as PL
from helpers import GOLDEN
from pyradiomics_b200 import cmatrices as B

pytestmark = pytest.mark.gpu
CASES = ["brain1", "brain2", "breast1", "lung1", "lung2"]


def _same(a, b, ngtdm=False):
    assert a.shape == b.shape, (a.shape, b.shape)
    if ngtdm:
        assert np.array_equal(a[..., [0, 2]], b[..., [0, 2]])
        assert np.allclose(a[..., 1], b[..., 1], rtol=1e-12, atol=1e-12)
    else:
        assert np.array_equal(a, b)


def test_random_inputs_match_oracle_bit_exact():
    rng = np.random.default_rng(11)
    n = 0
    for trial in range(36):
        nd = int(rng.choice([2, 3]))
        shp = tuple(int(s) for s in (rng.integers(1, 9, nd) if trial % 3 else rng.integers(3, 8, nd)))
        Ng = int(rng.integers(1, 9)) if trial % 7 else 300   # 300 -> 16-bit level path
        img = rng.integers(1, Ng + 1, shp).astype(np.int32)
        msk = rng.random(shp) > float(rng.choice([0, 0.2, 0.6]))
        if msk.sum() == 0:
            continue
        dist = np.array([[1], [1, 2], [2], [1, 3]][trial % 4])
        f2 = int(trial % 5 == 0 and nd == 3)
        f2d = int(rng.integers(0, nd))
        try:
            ref = O.calculate_glcm(img, msk, dist, Ng, f2, f2d)
            refr = O.calculate_glrlm(img, msk, Ng, max(shp), f2, f2d)
        except RuntimeError:
            with pytest.raises(RuntimeError):
                B.calculate_glcm(img, msk, dist, Ng, f2, f2d)
            continue
        got = B.calculate_glcm(img, msk, dist, Ng, f2, f2d)
        _same(got[0], ref[0]); assert np.array_equal(got[1], ref[1])
        got = B.calculate_glrlm(img, msk, Ng, max(shp), f2, f2d)
        _same(got[0], refr[0]); assert np.array_equal(got[1], refr[1])
        Ns = int(msk.sum())
        _same(B.calculate_glszm(img, msk, Ng, Ns, f2, f2d), O.calculate_glszm(img, msk, Ng, Ns, f2, f2d))
        _same(B.calculate_ngtdm(img, msk, dist, Ng, f2, f2d), O.calculate_ngtdm(img, msk, dist, Ng, f2, f2d), ngtdm=True)
        _same(B.calculate_gldm(img, msk, dist, Ng, 1, f2, f2d), O.calculate_gldm(img, msk, dist, Ng, 1, f2, f2d))
        vox = np.array(np.where(msk)).astype(np.int32)
        r = int(rng.integers(1, 3))
        _same(B.calculate_glcm(img, msk, dist, Ng, f2, f2d, r, vox)[0], O.calculate_glcm(img, msk, dist, Ng, f2, f2d, r, vox)[0])
        _same(B.calculate_glrlm(img, msk, Ng, max(shp), f2, f2d, r, vox)[0], O.calculate_glrlm(img, msk, Ng, max(shp), f2, f2d, r, vox)[0])
        _same(B.calculate_glszm(img, msk, Ng, Ns, f2, f2d, r, vox), O.calculate_glszm(img, msk, Ng, Ns, f2, f2d, r, vox))
        _same(B.calculate_ngtdm(img, msk, dist, Ng, f2, f2d, r, vox), O.calculate_ngtdm(img, msk, dist, Ng, f2, f2d, r, vox), ngtdm=True)
        _same(B.calculate_gldm(img, msk, dist, Ng, 0, f2, f2d, r, vox), O.calculate_gldm(img, msk, dist, Ng, 0, f2, f2d, r, vox))
        n += 1
    assert n > 15


@pytest.mark.parametrize("case", CASES)
def test_reference_golden_matrices(case):
    """reference tests/test_matrices.py:35-65 (data/baseline/<case>_<class>.npy), config 1 of BASELINE.json"""
    cases = np.load(os.path.join(GOLDEN, "segment_cases.npz"))
    msk = cases[f"{case}_mask"]
    img, _, levels, Ng = PL.bin_image(cases[f"{case}_image"], msk, 25)
    P, _ = B.calculate_glcm(img, msk, np.array([1]), Ng, False, 0)
    assert np.abs(F.glcm_matrix(P, levels)[0] - cases[f"{case}_glcm_P"]).max() < 1e-12
    P, _ = B.calculate_glrlm(img, msk, Ng, max(img.shape), False, 0)
    P = P[0, levels - 1]
    assert np.array_equal(P[:, P.sum((0, 2)) != 0], cases[f"{case}_glrlm_P"])
    P = B.calculate_glszm(img, msk, Ng, int(msk.sum()), False, 0)[0, levels - 1]
    assert np.array_equal(P[:, P.sum(0) != 0], cases[f"{case}_glszm_P"])
    P = B.calculate_gldm(img, msk, np.array([1]), Ng, 0, False, 0)[0, levels - 1]
    assert np.array_equal(P[:, P.sum(0) != 0], cases[f"{case}_gldm_P"])
    P = B.calculate_ngtdm(img, msk, np.array([1]), Ng, False, 0)[0]
    P = P[P[:, 0] != 0]
    ref = cases[f"{case}_ngtdm_P"]
    assert np.array_equal(P[:, [0, 2]], ref[:, [0, 2]]) and np.allclose(P[:, 1], ref[:, 1], rtol=1e-12)


def test_reference_dense_voxel_matrices():
    z = np.load(os.path.join(GOLDEN, "voxmat_small.npz"))
    img, msk, vox = z["image"], z["mask"], z["voxels"]
    got, ang = B.calculate_glcm(img, msk, np.array([1]), 6, False, 0, 1, vox)
    assert np.array_equal(got, z["glcm"]) and np.array_equal(ang, z["glcm_angles"])
    got, ang = B.calculate_glrlm(img, msk, 6, 7, False, 0, 1, vox)
    assert np.array_equal(got, z["glrlm"]) and np.array_equal(ang, z["glrlm_angles"])
    assert np.array_equal(B.calculate_glszm(img, msk, 6, int(msk.sum()), False, 0, 1, vox), z["glszm"])
    assert np.array_equal(B.calculate_gldm(img, msk, np.array([1]), 6, 0, False, 0, 1, vox), z["gldm"])
    got = B.calculate_ngtdm(img, msk, np.array([1]), 6, False, 0, 1, vox)
    assert np.array_equal(got[..., [0, 2]], z["ngtdm"][..., [0, 2]]) and np.allclose(got[..., 1], z["ngtdm"][..., 1], rtol=1e-13)


def test_error_conventions():
    img = np.ones((4, 4, 4), np.int32)
    msk = np.ones((4, 4, 4), bool)
    img[0, 0, 0] = 0
    with pytest.raises(IndexError):
        B.calculate_glcm(img, msk, [1], 3, False, 0)
    img[0, 0, 0] = 9
    with pytest.raises(IndexError):
        B.calculate_gldm(img, msk, [1], 3, 0, False, 0)
    with pytest.raises(ValueError):
        B.calculate_glcm(np.ones((4, 4)), msk, [1], 3, False, 0)
    with pytest.raises(ValueError):
        B.calculate_glcm(np.ones((4, 4, 5)), msk, [1], 3, False, 0)
    with pytest.raises(RuntimeError):
        B.calculate_glcm(np.ones((4, 4, 4)), msk, [1], 3, False, 0, 0, np.zeros((3, 2), np.int32))
    with pytest.raises(RuntimeError):
        B.calculate_glcm(np.ones((4, 4, 4)), msk, [0], 3, False, 0)


def test_segment_mode_at_scale_properties():
    """256^3 (batch-64x256^3 config shape): counts sum to the analytic number of neighbour pairs and
    the histogram is invariant under reflection of the volume."""
    rng = np.random.default_rng(5)
    N = 160
    img = rng.integers(1, 33, (N, N, N)).astype(np.int32)
    msk = np.ones(img.shape, bool)
    P, ang = B.calculate_glcm(img, msk, [1], 32, False, 0)
    for a, off in enumerate(ang):
        assert P[0, :, :, a].sum() == np.prod([N - abs(o) for o in off])
    Pf, _ = B.calculate_glcm(img[:, :, ::-1].copy(), msk, [1], 32, False, 0)
    # mirrored in x: angle (dz,dy,dx) maps to (dz,dy,-dx), i.e. the transposed matrix of that angle
    idx = {tuple(o): k for k, o in enumerate(ang)}
    for a, off in enumerate(ang):
        m = (off[0], off[1], -off[2])
        if m in idx:
            assert np.array_equal(Pf[0, :, :, idx[m]], P[0, :, :, a])
        else:
            assert np.array_equal(Pf[0, :, :, idx[tuple(-x for x in m)]], P[0, :, :, a].T)
    D = B.calculate_gldm(img, msk, [1], 32, 0, False, 0)
    assert D.sum() == N ** 3
    Z = B.calculate_glszm(img, msk, 32, N ** 3, False, 0)
    assert (Z[0] * np.arange(1, Z.shape[2] + 1)[None, :]).sum() == N ** 3


# ---- segment kernels: the tile-staged fused kernel (TMA / cooperative), the direct kernel, run-end GLRLM, device entry points
@pytest.mark.parametrize("shape,dist", [((20, 33, 64), [1]), ((9, 17, 48), [1, 2]), ((1, 40, 80), [1]), ((37, 29, 23), [1, 3])])
def test_segment_kernels_tma_equals_cooperative_equals_oracle(shape, dist, monkeypatch):
    """the fused GLCM + GLDM + NGTDM tile kernel with its box staged by TMA (row pitch a multiple of 16 bytes) or by
    cooperative loads, and the run-end GLRLM kernel: identical matrices, equal to the oracle"""
    import torch
    from pyradiomics_b200 import cmatrices, voxel
    rng = np.random.default_rng(12)
    if shape[0] == 1:
        shape = shape[1:]
    lev = rng.integers(1, 25, shape).astype(np.int32)
    msk = rng.random(shape) < 0.8
    res = {}
    for mode in ("tma", "coop"):
        monkeypatch.setenv("B200_SEG_TMA", "0" if mode == "coop" else "1")
        P, ang = cmatrices.calculate_glcm(lev, msk, dist, 24, False, -1)
        R, _ = cmatrices.calculate_glrlm(lev, msk, 24, max(shape), False, -1)
        res[mode] = (P, cmatrices.calculate_gldm(lev, msk, dist, 24, 1, False, -1), cmatrices.calculate_ngtdm(lev, msk, dist, 24, False, -1), R)
    for k in range(4):
        assert np.array_equal(res["tma"][k], res["coop"][k])
    ref = (O.calculate_glcm(lev, msk, dist, 24, False, -1)[0], O.calculate_gldm(lev, msk, dist, 24, 1, False, -1),
           O.calculate_ngtdm(lev, msk, dist, 24, False, -1), O.calculate_glrlm(lev, msk, 24, max(shape), False, -1)[0])
    for k in range(4):
        _same(res["tma"][k], ref[k], ngtdm=k == 2)
    # the same from a device-resident packed level volume, all three matrices in one pass
    monkeypatch.setenv("B200_SEG_TMA", "1")
    levd, _ = voxel.pack_levels(torch.as_tensor(lev).cuda(), torch.as_tensor(msk).cuda(), 24)
    d = cmatrices.segment_texture_device(levd, dist, 24, 1, False, -1)
    assert np.array_equal(d["glcm"][0], res["tma"][0]) and np.array_equal(d["gldm"], res["tma"][1]) and np.array_equal(d["ngtdm"], res["tma"][2])
    Rd, _ = cmatrices.calculate_glrlm_device(levd, 24, max(shape), False, -1)
    assert np.array_equal(Rd, res["tma"][3])
    Zd = cmatrices.calculate_glszm_device(levd, 24, False, -1)
    assert np.array_equal(Zd, cmatrices.calculate_glszm(lev, msk, 24, int(msk.sum()), False, -1))


def test_segment_tile_kernel_equals_direct_kernel():
    """levels 1..24 as an 8-bit volume (Ng = 24: tile kernel) and as a 16-bit one (Ng = 300: direct kernel): the leading
    24 levels of the Ng = 300 matrices are the Ng = 24 matrices bit for bit, NGTDM s_i included"""
    import torch
    from pyradiomics_b200 import cmatrices, voxel
    rng = np.random.default_rng(21)
    lev = rng.integers(1, 25, (19, 31, 48)).astype(np.int32)
    msk = rng.random(lev.shape) < 0.8
    dist = [1, 2]
    got = {}
    for Ng in (24, 300):
        levd, _ = voxel.pack_levels(torch.as_tensor(lev).cuda(), torch.as_tensor(msk).cuda(), Ng)
        assert levd.element_size() == (1 if Ng == 24 else 2)
        d = cmatrices.segment_texture_device(levd, dist, Ng, 1, False, -1)
        h = (cmatrices.calculate_glcm(lev, msk, dist, Ng, False, -1)[0], cmatrices.calculate_gldm(lev, msk, dist, Ng, 1, False, -1),
             cmatrices.calculate_ngtdm(lev, msk, dist, Ng, False, -1))
        got[Ng] = ((d["glcm"][0], d["gldm"], d["ngtdm"]), h)
    for api in range(2):
        small, big = got[24][api], got[300][api]
        assert np.array_equal(big[0][:, :24, :24], small[0]) and not big[0][:, 24:].any() and not big[0][:, :, 24:].any()
        assert np.array_equal(big[1][:, :24], small[1]) and not big[1][:, 24:].any()
        assert np.array_equal(big[2][:, :24], small[2]) and not big[2][:, 24:, :2].any()


@pytest.mark.parametrize("case", ["2d_long_offsets", "3d_glcm_193_offsets", "3d_many_levels", "16bit_one_pass"])
def test_segment_direct_kernel_triggers_match_oracle(case):
    """one input for each reason the direct kernel runs instead of the tile kernel, against the oracle"""
    import torch
    from pyradiomics_b200 import cmatrices, voxel
    from pyradiomics_b200._lib import B200Error
    rng = np.random.default_rng(33)
    shape, dist, Ng = {"2d_long_offsets": ((40, 50), [1, 4], 24),            # offsets > 3; GLCM privatised in shared memory
                       "3d_glcm_193_offsets": ((9, 11, 13), [4], 8),         # 193 unidirectional offsets: GLCM only
                       "3d_many_levels": ((10, 12, 14), [1, 2, 3], 200),     # GLDM / NGTDM histograms overflow shared memory
                       "16bit_one_pass": ((14, 17, 33), [1, 2], 300)}[case]
    lev = rng.integers(1, Ng + 1, shape).astype(np.int32)
    msk = rng.random(shape) < 0.8
    P, ang = cmatrices.calculate_glcm(lev, msk, dist, Ng, False, -1)
    Pr, ang_r = O.calculate_glcm(lev, msk, dist, Ng, False, -1)
    _same(P, Pr)
    assert np.array_equal(ang, ang_r)
    if case == "3d_glcm_193_offsets":
        assert ang.shape[0] == 193
        with pytest.raises(B200Error):
            cmatrices.calculate_gldm(lev, msk, dist, Ng, 1, False, -1)
        with pytest.raises(B200Error):
            cmatrices.calculate_ngtdm(lev, msk, dist, Ng, False, -1)
        levd, _ = voxel.pack_levels(torch.as_tensor(lev).cuda(), torch.as_tensor(msk).cuda(), Ng)
        d = cmatrices.segment_texture_device(levd, dist, Ng, 1, False, -1, glcm=True, gldm=False, ngtdm=False)
        _same(d["glcm"][0], Pr)
        assert np.array_equal(d["glcm"][1], ang_r)
        with pytest.raises(B200Error):
            cmatrices.segment_texture_device(levd, dist, Ng, 1, False, -1, glcm=True, gldm=True, ngtdm=False)
        return
    D, N = O.calculate_gldm(lev, msk, dist, Ng, 1, False, -1), O.calculate_ngtdm(lev, msk, dist, Ng, False, -1)
    _same(cmatrices.calculate_gldm(lev, msk, dist, Ng, 1, False, -1), D)
    _same(cmatrices.calculate_ngtdm(lev, msk, dist, Ng, False, -1), N, ngtdm=True)
    levd, _ = voxel.pack_levels(torch.as_tensor(lev).cuda(), torch.as_tensor(msk).cuda(), Ng)
    d = cmatrices.segment_texture_device(levd, dist, Ng, 1, False, -1)
    _same(d["glcm"][0], Pr)
    _same(d["gldm"], D)
    _same(d["ngtdm"], N, ngtdm=True)


def test_glrlm_single_voxel_lines_rule_from_pigeonhole_counts():
    """cmatrices.c:524-534: an angle none of whose lines holds two masked voxels loses its run-length-1 column"""
    import cmatrices_oracle as O
    from pyradiomics_b200 import cmatrices
    lev = np.zeros((5, 6, 7), np.int32)
    msk = np.zeros(lev.shape, bool)
    for (z, y, x, g) in [(0, 0, 0, 3), (2, 3, 4, 5), (4, 1, 6, 2), (1, 5, 2, 7)]:      # isolated voxels: most angles have no 2-voxel line
        lev[z, y, x] = g; msk[z, y, x] = True
    lev[2, 3, 5] = 5; msk[2, 3, 5] = True                                              # one x-neighbour pair
    got, ang = cmatrices.calculate_glrlm(lev, msk, 8, 7, False, -1)
    ref, ang_r = O.calculate_glrlm(lev, msk, 8, 7, False, -1)
    assert np.array_equal(ang, ang_r) and np.array_equal(got, ref)


@pytest.mark.parametrize("dist", [[1], [1, 2, 3]])
def test_segment_gldm_ngtdm_at_the_largest_ng(dist):
    """GLDM / NGTDM without GLCM at Ng = 65535 (16-bit levels, direct kernel), host and device APIs, against the oracle:
    their device buffers scale with Ng, not Ng^2"""
    import torch
    from pyradiomics_b200 import cmatrices, voxel
    rng = np.random.default_rng(44)
    Ng = 65535
    lev = rng.choice(np.array([1, 2, 3, 300, 301, 40000, 65534, 65535], np.int32), (6, 7, 8))
    msk = rng.random(lev.shape) < 0.8
    N = O.calculate_ngtdm(lev, msk, dist, Ng, False, -1)
    _same(cmatrices.calculate_ngtdm(lev, msk, dist, Ng, False, -1), N, ngtdm=True)
    levd, _ = voxel.pack_levels(torch.as_tensor(lev).cuda(), torch.as_tensor(msk).cuda(), Ng)
    d = cmatrices.segment_texture_device(levd, dist, Ng, 1, False, -1, glcm=False, gldm=dist == [1], ngtdm=True)
    _same(d["ngtdm"], N, ngtdm=True)
    if dist == [1]:          # (at [1, 2, 3] the float64 GLDM alone is 0.36 GB on the host per copy)
        D = O.calculate_gldm(lev, msk, dist, Ng, 1, False, -1)
        _same(cmatrices.calculate_gldm(lev, msk, dist, Ng, 1, False, -1), D)
        _same(d["gldm"], D)
