"""GPU checks of the voxel-based kernels on every reference voxel-mode fixture and at the generic kernel's capacity
limits:
* the tensor API (device-computed alive angles, `centers` for an unmasked kernel, a 2-D image as one plane) with the
  fast dispatch and with every class forced through the generic kernel;
* glcm_alive_kernel against a brute force;
* the r = 1 fast kernels given a `centers` mask;
* the 32-level MCC solve and the 2048-entry weighted GLCM list of the generic kernel, in uint8 and uint16 levels."""
import ctypes as C
import logging

import numpy as np
import pytest
import torch

import cmatrices_oracle as O
import pipeline as PL
from helpers import (alive_mask_bruteforce, assert_maps_close, binned, envelope_volume, mcc_over_capacity, ref_map,
                     voxel_goldens)
from pyradiomics_b200 import _lib, featureclasses as FC, image as I, voxel

pytestmark = pytest.mark.gpu
GOLDENS = voxel_goldens(extra=True)
SPACING_ZYX = (2.0, 0.7, 1.0)
CASES = [(r, n, False) for r in (2, 3) for n in (24, 36, 48, 64)] + [(2, 48, True), (3, 48, True)]


def _cuda(a, dtype=None):
    return torch.as_tensor(np.ascontiguousarray(a if dtype is None else a.astype(dtype))).cuda()


def _pack(lev):
    """binned levels (0 outside the ROI) -> the product's packed level volume: uint8, or int16 storage when Ng > 255"""
    Ng = int(lev.max())
    lev_t, _ = voxel.pack_levels(_cuda(lev, np.int32), _cuda(lev != 0), Ng)
    return lev_t, Ng


def _generic(monkeypatch, on):
    if on:
        monkeypatch.setenv("B200_RADIOMICS_FORCE_GENERIC", "1")
    else:
        monkeypatch.delenv("B200_RADIOMICS_FORCE_GENERIC", raising=False)


# ------------------------------------------------------------------------------ reference fixtures, tensor API
@pytest.mark.parametrize("generic", [False, True], ids=["dispatch", "generic"])
@pytest.mark.parametrize("name,z,kw", GOLDENS, ids=[g[0] for g in GOLDENS])
def test_tensor_api_matches_reference_maps(name, z, kw, generic, monkeypatch):
    mask = z["mask"]
    centers = None
    if kw.get("maskedKernel", True):
        lev, levels, Ng = binned(z, kw)
    else:
        # unmasked kernel (reference base.py:100-104): every voxel is binned and seen by the windows, the ROI only
        # selects the centre voxels
        lev, _, levels, Ng = PL.bin_image(z["image"], np.ones(mask.shape, bool), kw.get("binWidth", 25), kw.get("binCount"))
        centers = mask
    sp_zyx = tuple(z["spacing"][::-1])
    if lev.ndim == 2:                        # a 2-D image runs as one plane, like featureclasses._voxel_settings
        lev, mask, sp_zyx = lev[None], mask[None], (1.0,) + sp_zyx
        centers = None if centers is None else centers[None]
    lev_t, _ = _pack(lev)
    centers_t = None if centers is None else _cuda(centers, np.uint8)
    s = _lib.make_settings(Ng, len(levels), spacing_zyx=sp_zyx, **{k: v for k, v in kw.items() if k != "maskedKernel"})
    ang = O.generate_angles(lev.shape, kw.get("distances", [1]), 0, s.force2D, s.force2Ddimension)
    r3 = [0 if (s.force2D and s.force2Ddimension == k) else s.kernelRadius for k in range(3)]
    assert np.array_equal(voxel.glcm_alive_angles(lev_t, s, centers_t), alive_mask_bruteforce(lev, mask, ang, r3))
    _generic(monkeypatch, generic)
    for cname in _lib.CLASSES:
        out = voxel.voxel_features(cname, lev_t, s, centers=centers_t).cpu().numpy()
        for k, f in enumerate(_lib.feature_names(cname)):
            ref = ref_map(z, cname, f).reshape(out[k].shape)
            got = out[k] if centers is None else np.where(mask, out[k], ref)      # (outside the ROI: initValue)
            assert_maps_close(got, ref, f"{name}/{cname}/{f}")


# ------------------------------------------------------------------------------ alive angles
def _alive_case(lev, centers, r, distances, force2D=False, dim=0):
    s = _lib.make_settings(int(lev.max()), len(np.unique(lev[lev > 0])), kernelRadius=r, distances=distances,
                           force2D=force2D, force2Ddimension=dim)
    ang = O.generate_angles(lev.shape, distances, 0, force2D, dim)
    r3 = [0 if (force2D and dim == k) else r for k in range(3)]
    got = voxel.glcm_alive_angles(_cuda(lev, np.uint8), s, None if centers is None else _cuda(centers, np.uint8))
    want = alive_mask_bruteforce(lev, lev != 0 if centers is None else centers, ang, r3)
    assert np.array_equal(got, want), (got, want)
    return got


def _alive_volume(kind, seed=3, shape=(8, 9, 10)):
    """(levels, centers): 'holes' a tenth of the voxels outside the ROI; 'sparse' 3 % of the voxels in it, so that
    angles die for lack of pairs; 'roi' everything binned with an irregular centre mask that touches a corner and the
    faces, where windows are clipped"""
    rng = np.random.default_rng(seed)
    lev = rng.integers(1, 9, shape)
    if kind == "holes":
        lev[rng.random(shape) < 0.1] = 0
        return lev, None
    if kind == "sparse":
        lev[rng.random(shape) > 0.03] = 0
        return lev, None
    roi = rng.random(shape) < 0.02
    roi[0, 0, 0] = roi[-1, 4, 5] = roi[3, 0, 7] = True
    return lev, roi


@pytest.mark.parametrize("kind", ["holes", "sparse", "roi"])
@pytest.mark.parametrize("distances", [[1], [2], [1, 3]], ids=["d1", "d2", "d13"])
@pytest.mark.parametrize("r", [1, 2, 3])
def test_alive_angles_equal_bruteforce(r, distances, kind):
    lev, centers = _alive_volume(kind)
    _alive_case(lev, centers, r, distances)


@pytest.mark.parametrize("kind", ["holes", "roi"])
@pytest.mark.parametrize("dim", [0, 1, 2])
def test_alive_angles_force2d_equal_bruteforce(dim, kind):
    lev, centers = _alive_volume(kind, seed=4)
    _alive_case(lev, centers, 2, [1, 2], force2D=True, dim=dim)


def test_alive_angle_seen_from_a_single_window():
    """one co-occurrence, along (1,1,1), that only the window of centre (4,5,4) contains (r = 1 windows hold it for
    centres in {4,5}^3): the angle lives with that centre and dies without it"""
    lev = np.zeros((9, 9, 9), np.int32)
    lev[4, 4, 4], lev[5, 5, 5] = 3, 7
    centers = np.zeros(lev.shape, bool)
    for c in ((3, 3, 3), (6, 6, 6), (3, 4, 4), (4, 5, 4)):
        centers[c] = True
    got = _alive_case(lev, centers, 1, [1])
    assert sum(bin(int(w)).count("1") for w in got) == 1
    centers[4, 5, 4] = False
    assert not _alive_case(lev, centers, 1, [1]).any()


# ------------------------------------------------------------------------------ fast kernels with `centers`
@pytest.fixture(scope="module")
def binned_volume_with_roi():
    """24^3 smooth levels 1..32, every voxel binned (an unmasked kernel), and an irregular ROI of centres: a noisy ball
    cut by a face, a hole in it, and scattered voxels"""
    rng = np.random.default_rng(12)
    shape = (24, 24, 24)
    zz, yy, xx = np.meshgrid(*[np.arange(s) for s in shape], indexing="ij")
    f = np.sin(zz / 2.7) + np.cos(yy / 3.1) + np.sin(xx / 2.3 + 1) + 0.25 * rng.normal(size=shape)
    lev = (np.digitize(f, np.quantile(f, np.linspace(0, 1, 33)[1:-1])) + 1).astype(np.int32)
    d = np.sqrt((zz - 3) ** 2 + (yy - 12) ** 2 + (xx - 11) ** 2) + rng.normal(0, 1.5, shape)
    roi = (d < 9) | (rng.random(shape) < 0.02)
    roi[3:6, 10:14, 9:12] = False
    return lev, roi


@pytest.mark.parametrize("cname", _lib.CLASSES)
def test_fast_kernels_with_centers_equal_generic_kernel(binned_volume_with_roi, cname, monkeypatch):
    lev, roi = binned_volume_with_roi
    lev_t, Ng = _pack(lev)
    s = _lib.make_settings(Ng, Ng, gldm_a=1, initValue=-1)
    roi_t = _cuda(roi, np.uint8)
    fast = voxel.voxel_features(cname, lev_t, s, centers=roi_t).cpu().numpy()
    _generic(monkeypatch, True)
    gen = voxel.voxel_features(cname, lev_t, s, centers=roi_t).cpu().numpy()
    assert (fast[:, ~roi] == -1).all() and (gen[:, ~roi] == -1).all()
    for k, f in enumerate(_lib.feature_names(cname)):
        if cname == "glcm":       # tolerances of the GLCM fast-vs-generic test on 40^3 (tests/test_voxel_gpu.py)
            rtol, atol = {"MCC": (0, 1e-9), "Imc1": (2e-9, 1e-12), "Imc2": (2e-9, 1e-6)}.get(f, (1e-7, 1e-9))
            ok = np.allclose(fast[k], gen[k], rtol=rtol, atol=atol, equal_nan=True)
        else:
            ok = np.allclose(fast[k], gen[k], rtol=1e-10, atol=1e-12, equal_nan=True)
        assert ok, (cname, f, np.nanmax(np.abs(fast[k] - gen[k])))


def test_fast_kernels_with_centers_match_oracle(binned_volume_with_roi):
    lev, roi = binned_volume_with_roi
    lev, roi = lev[:8, 12:22, 12:22].copy(), roi[:8, 12:22, 12:22]
    lev[0, 0, 0] = 1                                  # binWidth=1 binning of the whole crop is the identity
    assert 30 < roi.sum() < roi.size - 30
    lev_t, Ng = _pack(lev)
    s = _lib.make_settings(Ng, len(np.unique(lev)))
    for cname in _lib.CLASSES:
        out = voxel.voxel_features(cname, lev_t, s, centers=_cuda(roi, np.uint8)).cpu().numpy()
        ref = PL.extract(cname, lev, roi, voxelBased=True, binWidth=1, maskedKernel=False)
        for k, f in enumerate(_lib.feature_names(cname)):
            assert_maps_close(out[k][roi], ref[f], f"crop/{cname}/{f}")


# ------------------------------------------------------------------------------ capacity limits of the generic kernel
def _oracle(cname, lev, mask, chunk=16, **kw):
    """PL.extract over the ROI in voxel batches (the dense per-voxel matrices are Ng^2 per angle: gigabytes when Ng > 255).
    Every alive angle has pairs in every window of these volumes, so batching deletes no angle the whole run keeps."""
    vox = np.array(np.where(mask)).astype(np.int32)
    parts = [PL.extract(cname, lev, mask, voxelBased=True, binWidth=1, voxels=vox[:, a:a + chunk], **kw)
             for a in range(0, vox.shape[1], chunk)]
    return {f: np.concatenate([p[f] for p in parts]) for f in parts[0]}


def _envelope_levels(n_levels, holes, sixteen_bit):
    lev = envelope_volume(n_levels, holes)
    if sixteen_bit:          # Ng = 256: uint16 level storage; level 1 keeps binWidth=1 binning the identity
        lev = np.where(lev > 0, lev + 256 - n_levels, 0)
        lev[0, 0, 0] = 1
    return lev


def _check_mcc(got, ref, over, what):
    finite_wrong = int(np.sum(over & np.isfinite(got)))
    assert finite_wrong == 0, f"{what}: {finite_wrong} over-capacity voxels hold a finite MCC"
    assert not np.isnan(got[~over]).any(), f"{what}: NaN MCC outside the over-capacity voxels"
    assert_maps_close(got, np.where(over, np.nan, ref), what)


# uint16 levels on the over-capacity cases only: the oracle's dense Ng^2 matrices make each one several seconds
DEVICE_CASES = [c + (False,) for c in CASES] + [c + (True,) for c in CASES if c[1] in (36, 64) or c[2]]


@pytest.mark.parametrize("r,n_levels,holes,sixteen_bit", DEVICE_CASES,
                         ids=[f"r{r}-L{n}" + ("-holes" if h else "") + ("-u16" if u else "-u8") for r, n, h, u in DEVICE_CASES])
def test_generic_kernel_beyond_the_mcc_capacity(r, n_levels, holes, sixteen_bit):
    lev = _envelope_levels(n_levels, holes, sixteen_bit)
    mask = lev != 0
    lev_t, Ng = _pack(lev)
    assert lev_t.dtype == (torch.int16 if sixteen_bit else torch.uint8)
    s = _lib.make_settings(Ng, len(np.unique(lev[mask])), kernelRadius=r)
    over = mcc_over_capacity(lev, mask, r)
    assert over.any() == (n_levels > 32)
    for cname in _lib.CLASSES:
        status = torch.zeros(1, dtype=torch.int32, device="cuda")
        out = voxel.voxel_features(cname, lev_t, s, status=status).cpu().numpy()
        assert int(status.item()) == (int(over.any()) if cname == "glcm" else 0)
        ref = _oracle(cname, lev, mask, kernelRadius=r)
        for k, f in enumerate(_lib.feature_names(cname)):
            what = f"r{r}/L{n_levels}/{cname}/{f}"
            if f == "MCC":
                _check_mcc(out[k][mask], ref[f], over, what)
            else:
                assert_maps_close(out[k][mask], ref[f], what)


@pytest.mark.parametrize("n_levels", [24, 48])
def test_plugin_warns_and_stores_nan_when_mcc_is_over_capacity(n_levels, caplog):
    lev = envelope_volume(n_levels)
    mask = lev != 0
    over = mcc_over_capacity(lev, mask, 2)
    with caplog.at_level(logging.WARNING, logger="radiomics.glcm"):
        got = FC.RadiomicsGLCM(I.ArrayImage(lev), I.ArrayImage(mask.astype(np.uint8)), voxelBased=True, kernelRadius=2,
                               binWidth=1).execute()
    warned = [rec for rec in caplog.records if rec.name == "radiomics.glcm" and "MCC" in rec.getMessage()]
    assert bool(warned) == over.any()
    assert np.array_equal(np.isnan(I.as_array(got["MCC"])[mask]), over)


def _host_api_glcm(lev, **kw):
    img = np.ascontiguousarray(lev, dtype=np.int32)
    msk = np.ascontiguousarray(lev != 0, dtype=np.uint8)
    s = _lib.make_settings(int(lev.max()), len(np.unique(lev[lev > 0])), **kw)
    out = np.empty((24,) + img.shape)
    _lib.check(_lib.lib().rb_voxel_features_host(_lib.CLASS_ID["glcm"], img.ctypes.data_as(C.c_void_p),
                                                  msk.ctypes.data_as(C.c_void_p), *img.shape, C.byref(s),
                                                  out.ctypes.data_as(C.c_void_p)), "glcm")
    return out


@pytest.mark.parametrize("r,n_levels", [(3, 32), (2, 64)])
def test_weighted_glcm_pooled_matrix_on_device(r, n_levels):
    """euclidean weights on anisotropic spacing: r = 3 with 32 levels fits; r = 2 with 64 levels fits the entry list
    but not the MCC solve (NaN exactly where the pooled matrix is over capacity)"""
    lev = envelope_volume(n_levels)
    mask = lev != 0
    kw = dict(kernelRadius=r, weightingNorm="euclidean")
    lev_t, Ng = _pack(lev)
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    out = voxel.voxel_features("glcm", lev_t, _lib.make_settings(Ng, Ng, spacing_zyx=SPACING_ZYX, **kw), status=status)
    out = out.cpu().numpy()
    over = mcc_over_capacity(lev, mask, r, spacing_zyx=SPACING_ZYX, weightingNorm="euclidean")
    assert over.any() == (n_levels > 32)
    assert int(status.item()) == int(over.any())
    ref = PL.extract("glcm", lev, mask, voxelBased=True, binWidth=1, spacing_zyx=SPACING_ZYX, **kw)
    for k, f in enumerate(_lib.feature_names("glcm")):
        what = f"weighted/r{r}/L{n_levels}/{f}"
        if f == "MCC":
            _check_mcc(out[k][mask], ref[f], over, what)
        else:
            assert_maps_close(out[k][mask], ref[f], what)


def test_weighted_glcm_entry_list_overflow_is_loud():
    """r = 3 with 64 i.i.d. levels: windows with more than 2048 distinct (level, level) pairs"""
    lev = envelope_volume(64)
    kw = dict(kernelRadius=3, weightingNorm="euclidean")
    with pytest.raises(_lib.B200Error, match="entry list overflow"):
        FC.RadiomicsGLCM(I.ArrayImage(lev, SPACING_ZYX[::-1]), I.ArrayImage((lev != 0).astype(np.uint8), SPACING_ZYX[::-1]),
                         voxelBased=True, binWidth=1, **kw).execute()
    with pytest.raises(_lib.B200Error, match="entry list overflow"):
        _host_api_glcm(lev, spacing_zyx=SPACING_ZYX, **kw)
