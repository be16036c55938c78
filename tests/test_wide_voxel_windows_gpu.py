"""The wide voxel kernels (csrc/voxel_wide.cu, firstorder_wide_kernel in csrc/firstorder.cu): windows of 344 to 3375
positions, one thread block per centre.

* Bit identity where both run: with B200_RADIOMICS_FORCE_WIDE=1 every window goes to the wide kernels, and every map of
  the five texture classes and first order, NaN positions and status word included, equals the generic kernel's at
  kernelRadius 1, 2 and 3 on the settings the generic kernel serves (distances, asymmetric and weighted GLCM / GLRLM,
  force2D, a 2-D image, 8- and 16-bit levels, ROI holes and faces, an unmasked kernel, a non-zero initValue, float64
  and float32 maps).
* The window oracle at kernelRadius 4, 5 and 7 (tests/helpers.py: box_references), on planted 9^3, 11^3 and 15^3 blocks
  (helpers.block_corpus), at the bounds of tests/test_generic_voxel_windows_gpu.py with the entropy floor scaled to the
  window's positions; one force2D case at kernelRadius 12 (25 x 25 = 625 positions).
* Every loop runs: a volume on which every resident block handles at least three centres.
* End to end: the plugin classes at kernelRadius 5 against oracle/pipeline.extract, and extract_to_nrrd against them."""
import os
from contextlib import contextmanager

import numpy as np
import pytest
import torch

import pipeline as PL
from helpers import (FAST_NAMES, RTOL, WindowRun, assert_maps_close, block_corpus, box_references, compare_box_maps,
                     plant_boxes, remap_boxes, weighted_overflow, window_box)
from pyradiomics_b200 import _lib, featureclasses as FC, image as I, voxel

pytestmark = pytest.mark.gpu

SPACING_ZYX = (2.0, 0.8, 0.6)
CLASSES = tuple(FAST_NAMES)


class WideRun(WindowRun):
    """WindowRun whose window capacity is the window's own size above 343 positions: the entropy floor of
    helpers.entropy_atol then counts the wide kernel's 2 * positions entries per angle"""

    @property
    def window_cap(self):
        n = int(np.prod([2 * r + 1 for r in self.radii]))
        return n if n > 343 else WindowRun.window_cap.fget(self)


@contextmanager
def wide(on=True):
    """B200_RADIOMICS_FORCE_WIDE=1 (every window to the wide kernels) or B200_RADIOMICS_FORCE_GENERIC=1 (every window
    of <= 343 positions to the generic kernels, the r = 1 fast paths' included)"""
    keys = ("B200_RADIOMICS_FORCE_WIDE", "B200_RADIOMICS_FORCE_GENERIC")
    old = {k: os.environ.pop(k, None) for k in keys}
    os.environ[keys[0] if on else keys[1]] = "1"
    try:
        yield
    finally:
        for k in keys:
            os.environ.pop(k, None)
            if old[k] is not None:
                os.environ[k] = old[k]


def _cuda(a, dtype=None):
    return torch.as_tensor(np.ascontiguousarray(a if dtype is None else a.astype(dtype))).cuda()


def _pack(vol):
    lev, _ = voxel.pack_levels(_cuda(vol, np.int32), _cuda(vol != 0), int(vol.max()))
    return lev


def _at(out, cen):
    idx = tuple(torch.as_tensor(cen[:, d], device=out.device) for d in range(3))
    return out[(slice(None),) + idx].cpu().numpy()


def assert_bits_equal(a, b, what):
    """the same bits everywhere, NaN at the same positions"""
    na, nb = torch.isnan(a), torch.isnan(b)
    assert torch.equal(na, nb), (what, int((na != nb).sum()))
    iv = torch.int64 if a.dtype == torch.float64 else torch.int32
    a0, b0 = torch.where(na, torch.zeros_like(a), a), torch.where(nb, torch.zeros_like(b), b)
    diff = a0.view(iv) != b0.view(iv)
    assert not bool(diff.any()), (what, int(diff.sum()), a0[diff][:3].tolist(), b0[diff][:3].tolist())


def texture_both(cname, lev, s, centers=None, dtype=torch.float64):
    """(generic maps, wide maps, generic status, wide status) of one class"""
    res = []
    for on in (False, True):
        st = torch.zeros(1, dtype=torch.int32, device="cuda")
        with wide(on):
            out = voxel.voxel_features(cname, lev, s, centers=centers, status=st, dtype=dtype)
        res.append((out, int(st.item())))
    return res[0][0], res[1][0], res[0][1], res[1][1]


def firstorder_both(image, lev, roi, dtype=torch.float64, **kw):
    outs = []
    for on in (False, True):
        with wide(on):
            outs.append(voxel.firstorder_features(image, lev, roi, dtype=dtype, **kw))
    return outs


def check_identity(vol, what, centers=None, classes=CLASSES, alphas=(0, 3), dtypes=(torch.float64,), image=None,
                   roi="levels", **kw):
    """every class's maps on `vol` (and first order's on `image`, default: a float image of the levels with signed
    zeros) through the generic and the wide kernels: the same bits and status words"""
    lev = _pack(vol)
    Ng = int(vol.max())
    n_roi = len(np.unique(vol[vol > 0]))
    cen = None if centers is None else _cuda(centers, np.uint8)
    for dtype in dtypes:
        for cname in classes:
            for a in (alphas if cname == "gldm" else (0,)):
                s = _lib.make_settings(Ng, n_roi, gldm_a=a, **kw)
                g, w, sg, sw = texture_both(cname, lev, s, cen, dtype)
                assert sg == sw, (what, cname, sg, sw)
                assert_bits_equal(g, w, f"{what}/{cname}/a{a}/{dtype}")
        if image is None:
            rng = np.random.default_rng(Ng)
            image = (vol - 0.5 * Ng) * 0.37 + rng.normal(size=vol.shape).round(1)
            image[rng.random(vol.shape) < 0.05] = -0.0
        r3 = dict(kernelRadius=kw.get("kernelRadius", 1), force2D=kw.get("force2D", False),
                  force2Ddimension=kw.get("force2Ddimension", 0), initValue=kw.get("initValue", 0))
        roi_t = None if roi is None else _cuda(vol != 0, np.uint8)
        g, w = firstorder_both(_cuda(image), lev, roi_t, dtype=dtype, centers=cen, voxelArrayShift=7, **r3)
        assert_bits_equal(g, w, f"{what}/firstorder/{dtype}")


def _planted(side, n, seed, Ng=None, K_max=None, shape=None):
    boxes = block_corpus(n, side, seed=seed, K_max=K_max)
    if Ng is not None:
        boxes, _ = remap_boxes(boxes, Ng, np.random.default_rng(seed + Ng))
    if shape is not None:
        c = side // 2
        boxes = [b[tuple(slice(c - s // 2, c + s // 2 + 1) for s in shape)] for b in boxes]
        boxes = [b for b in boxes if b[tuple(s // 2 for s in shape)] > 0]
    vol, cen = plant_boxes(boxes)
    centers = np.zeros(vol.shape, bool)
    centers[tuple(cen.T)] = True
    return vol, centers


# --------------------------------------------------------------------------------------- bit identity, r = 1 to 3
IDENTITY = [
    ("r1", 1, {}, {}),
    ("r2", 2, {}, {}),
    ("r3", 3, {}, {}),
    ("r2-d2", 2, {}, dict(distances=(2,))),
    ("r3-d13", 3, {}, dict(distances=(1, 3))),
    ("r2-asym", 2, dict(Ng=255), dict(symmetricalGLCM=False)),
    ("r3-asym", 3, {}, dict(symmetricalGLCM=False)),
    ("r2-manhattan", 2, dict(K_max=40), dict(weightingNorm="manhattan", spacing_zyx=SPACING_ZYX)),
    ("r3-euclidean", 3, dict(K_max=40), dict(weightingNorm="euclidean", spacing_zyx=SPACING_ZYX)),
    ("r1-infinity", 1, {}, dict(weightingNorm="infinity", spacing_zyx=SPACING_ZYX)),
    ("r3-force2D0", 3, {}, dict(force2D=True, force2Ddimension=0)),
    ("r2-force2D1", 2, {}, dict(force2D=True, force2Ddimension=1)),
    ("r3-force2D2", 3, {}, dict(force2D=True, force2Ddimension=2)),
    ("r3-2D", 3, dict(shape=(1, 7, 7)), {}),
    ("r2-Ng32", 2, dict(Ng=32), {}),
    ("r2-Ng255", 2, dict(Ng=255), {}),
    ("r2-Ng256", 2, dict(Ng=256), {}),
    ("r1-Ng4096", 1, dict(Ng=4096), {}),
    ("r3-Ng4096", 3, dict(Ng=4096), {}),
]


@pytest.mark.parametrize("name,r,corpus,kw", IDENTITY, ids=[c[0] for c in IDENTITY])
def test_wide_equals_generic_on_planted_windows(name, r, corpus, kw):
    side = 2 * r + 1
    vol, centers = _planted(side, 60 if r > 1 else 200, seed=[c[0] for c in IDENTITY].index(name), **corpus)
    check_identity(vol, name, centers=centers, dtypes=(torch.float64, torch.float32), kernelRadius=r, **kw)


@pytest.mark.parametrize("r", [2, 3])
def test_wide_equals_generic_with_faces_holes_and_every_roi_voxel(r):
    """a random volume with 15 % ROI holes, every ROI voxel a centre (windows clipped by every face), initValue -3; first
    order with an unmasked kernel too"""
    rng = np.random.default_rng(40 + r)
    vol = rng.integers(1, 25, (9, 30, 31))
    vol[rng.random(vol.shape) < 0.15] = 0
    vol[4, 10:20, 5:25] = 7                                   # a plateau: long runs, a big zone
    vol[0, 0, 0], vol[-1, -1, -1] = 1, 24
    check_identity(vol, f"faces/r{r}", dtypes=(torch.float64, torch.float32), kernelRadius=r, initValue=-3.0)
    check_identity(vol, f"unmasked/r{r}", classes=(), roi=None, kernelRadius=r, initValue=-3.0)


def test_wide_equals_generic_with_nan_intensities():
    """a window holding NaN intensities takes the insertion sort on one thread: the same bits as the generic kernel"""
    rng = np.random.default_rng(5)
    vol = rng.integers(1, 9, (7, 12, 13))
    img = rng.normal(size=vol.shape)
    img[rng.random(vol.shape) < 0.02] = np.nan
    lev = _pack(vol)
    g, w = firstorder_both(_cuda(img), lev, _cuda(vol != 0, np.uint8), kernelRadius=2)
    assert torch.isnan(g).any()
    assert_bits_equal(g, w, "nan")


# ------------------------------------------------------------------------------------- the window oracle, r = 4 to 7
def run_oracle(vol, centers, what, Ng=None, classes=CLASSES, alphas=(0, 3), **kw):
    cen = np.argwhere(centers)
    Ng = Ng or int(vol.max())
    run = WideRun(vol.shape, Ng, **kw)
    run.alive_from(vol, centers)
    boxes = [window_box(vol, c, run.radii) for c in cen]
    if run.weights is not None:
        keep = np.array([not weighted_overflow(b, run) for b in boxes])
        boxes, cen = [b for b, k in zip(boxes, keep) if k], cen[keep]
        centers = np.zeros(vol.shape, bool)
        centers[tuple(cen.T)] = True
        run.alive_from(vol, centers)
    lev = _pack(vol)
    cen_t = _cuda(centers, np.uint8)
    for cname in classes:
        for a in (alphas if cname == "gldm" else (0,)):
            run.gldm_a = a
            refs = box_references(boxes, run, classes=[cname], mcc=cname == "glcm")
            st = torch.zeros(1, dtype=torch.int32, device="cuda")
            out = voxel.voxel_features(cname, lev, run.settings(len(np.unique(vol[vol > 0]))), centers=cen_t, status=st)
            want = int(refs["mcc_over"].any()) if cname == "glcm" else 0
            assert int(st.item()) == want, (what, cname, int(st.item()), want)
            w = compare_box_maps(_at(out, cen), refs, cname, a, f"{what}/gldm_a={a}", run)
            print(what, cname, a, "worst |error| / bound:", {f: f"{v:.2g}" for f, v in w.items() if v > 1e-3})


def _oracle_corpus(r, n, seed, **kw):
    """planted (2r+1)^3 blocks of helpers.block_corpus; above r = 4 the blocks with every voxel its own level (the
    dense oracle would hold a 3375^2 matrix per angle) are replaced by 200 i.i.d. levels"""
    side = 2 * r + 1
    boxes = block_corpus(n, side, seed=seed, **kw)
    rng = np.random.default_rng(seed)
    if r > 4:
        boxes = [b if len(np.unique(b)) <= 400 else np.where(b > 0, rng.integers(1, 201, b.shape), 0) for b in boxes]
    return boxes


@pytest.mark.parametrize("r,n", [(4, 44), (5, 33), (7, 22)])
def test_oracle_default_settings(r, n):
    vol, cen = plant_boxes(_oracle_corpus(r, n, seed=100 + r))
    centers = np.zeros(vol.shape, bool)
    centers[tuple(cen.T)] = True
    run_oracle(vol, centers, f"r{r}", kernelRadius=r)


@pytest.mark.parametrize("r", [4, 7])
def test_oracle_sixteen_bit_levels(r):
    boxes, _ = remap_boxes(_oracle_corpus(r, 22, seed=110 + r, K_max=60), 4096, np.random.default_rng(r))
    vol, cen = plant_boxes(boxes)
    centers = np.zeros(vol.shape, bool)
    centers[tuple(cen.T)] = True
    run_oracle(vol, centers, f"Ng4096/r{r}", Ng=4096, kernelRadius=r)


def test_oracle_weighted_and_asymmetric_r5():
    vol, cen = plant_boxes(_oracle_corpus(5, 22, seed=120, K_max=30))
    centers = np.zeros(vol.shape, bool)
    centers[tuple(cen.T)] = True
    run_oracle(vol, centers, "r5-euclidean", classes=("glcm", "glrlm"), kernelRadius=5, weightingNorm="euclidean",
               spacing_zyx=SPACING_ZYX)
    run_oracle(vol, centers, "r5-asym", classes=("glcm",), kernelRadius=5, symmetricalGLCM=False)


def test_oracle_force2d_r12():
    """force2D at kernelRadius 12: a 25 x 25 window of 625 positions, planted as one-plane blocks"""
    boxes = [b[12:13] for b in block_corpus(22, 25, seed=130, K_max=50)]
    vol, cen = plant_boxes(boxes)
    centers = np.zeros(vol.shape, bool)
    centers[tuple(cen.T)] = True
    run_oracle(vol, centers, "force2D-r12", kernelRadius=12, force2D=True, force2Ddimension=0)


def test_window_over_3375_positions_is_refused():
    vol = np.ones((18, 18, 18), np.int64)                        # first order clips r to the ROI's extent - 1 = 17
    s = _lib.make_settings(1, 1, kernelRadius=8)                    # 17^3 = 4913 positions
    with pytest.raises(_lib.B200Error, match="3375"):
        voxel.voxel_features("glcm", _pack(vol), s)
    with pytest.raises(_lib.B200Error, match="3375"):
        voxel.firstorder_features(_cuda(vol, np.float64), _pack(vol), _cuda(vol, np.uint8), kernelRadius=8)


# ------------------------------------------------------------------------------------------------ every loop runs
def test_every_resident_block_loops():
    """voxel_wide.cu wide_grid / firstorder_wide_launch: at most one resident wave, sms * (blocks per SM) blocks, and
    an SM holds at most 32 blocks on sm_90.  With >= 3 * sms * 32 centres every block handles >= 3.  Sampled centres
    against the oracle; the whole volume bit for bit against a second run, z-slab calls cut at and inside a chunk
    boundary, and float32 maps equal to the float64 maps rounded."""
    r = 4
    shape = (20, 28, 28)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    total = int(np.prod(shape))
    assert total >= 3 * sms * 32, (total, sms)
    rng = np.random.default_rng(150)
    zz, yy, xx = np.meshgrid(*[np.arange(s, dtype=np.float64) for s in shape], indexing="ij", sparse=True)
    f = np.sin(zz / 2.1) + np.cos(yy / 3.3) + np.sin(xx / 2.7 + 1) + 0.4 * rng.normal(size=shape)
    vol = np.digitize(f, np.quantile(f, np.linspace(0, 1, 16)[1:-1])) + 1
    vol[rng.random(shape) < 0.05] = 0
    vol[0, 0, 0] = 1
    run = WideRun(shape, int(vol.max()), kernelRadius=r)
    c = np.stack([rng.integers(0, s, 40) for s in shape], 1)
    c = c[vol[tuple(c.T)] > 0]
    run.alive_from(vol)
    boxes = [window_box(vol, x, run.radii) for x in c]
    refs = box_references(boxes, run)
    lev = _pack(vol)
    s = run.settings(len(np.unique(vol[vol > 0])))
    for cname in CLASSES:
        st = torch.zeros(1, dtype=torch.int32, device="cuda")
        out = voxel.voxel_features(cname, lev, s, status=st)
        compare_box_maps(_at(out, c), refs, cname, 0, "loops/r4", run)
        assert_bits_equal(voxel.voxel_features(cname, lev, s), out, f"{cname} again")
        parts = [voxel.voxel_features(cname, lev, s, z0=a, z1=b) for a, b in ((0, 5), (5, 13), (13, 20))]
        assert_bits_equal(torch.cat(parts, 1), out, f"{cname} slabs")
        f32 = voxel.voxel_features(cname, lev, s, dtype=torch.float32)
        assert_bits_equal(f32, out.to(torch.float32), f"{cname} float32")
    img = _cuda(f)
    roi = _cuda(vol != 0, np.uint8)
    fo = voxel.firstorder_features(img, lev, roi, kernelRadius=r)
    assert_bits_equal(voxel.firstorder_features(img, lev, roi, kernelRadius=r), fo, "firstorder again")
    parts = [voxel.firstorder_features(img, lev, roi, kernelRadius=r, z0=a, z1=b) for a, b in ((0, 5), (5, 13), (13, 20))]
    assert_bits_equal(torch.cat(parts, 1), fo, "firstorder slabs")
    assert_bits_equal(voxel.firstorder_features(img, lev, roi, kernelRadius=r, dtype=torch.float32, zchunk=7),
                      fo.to(torch.float32), "firstorder float32")


# ------------------------------------------------------------------------------------------------------ end to end
def _e2e_volume():
    rng = np.random.default_rng(160)
    shape = (9, 11, 12)
    raw = ((rng.integers(1, 14, shape) - 1) * 25 + 3).astype(np.int16)
    raw[3:6, 2:9, 3:10] = 128
    msk = (rng.random(shape) < 0.85).astype(np.uint8)
    msk[0] = 0
    return raw, msk


def test_plugins_at_kernel_radius_5_match_the_pipeline():
    import firstorder_np as FO
    raw, msk = _e2e_volume()
    img, m = I.ArrayImage(raw), I.ArrayImage(msk)
    for cname, cls in FC.FEATURE_CLASSES.items():
        got = cls(img, m, voxelBased=True, kernelRadius=5, binWidth=25).execute()
        ref = PL.extract(cname, raw, msk.astype(bool), voxelBased=True, kernelRadius=5, binWidth=25)
        for f, im in got.items():
            a = I.as_array(im)
            assert_maps_close(a[msk.astype(bool)], ref[f], f"r5/{cname}/{f}", rtol=RTOL)
    got = FC.RadiomicsFirstOrder(img, m, voxelBased=True, kernelRadius=5, binWidth=25, voxelArrayShift=100).execute()
    ref = FO.extract(raw, msk.astype(bool), voxelBased=True, kernelRadius=5, binWidth=25, voxelArrayShift=100)
    for f in FO.NAMES:
        assert np.allclose(I.as_array(got[f])[msk.astype(bool)], ref[f], rtol=1e-9, atol=1e-9), f


def _read_nrrd(path, shape):
    raw = open(path, "rb").read()
    head, data = raw.split(b"\n\n", 1)
    return np.frombuffer(data, "<f4" if b"\ntype: float\n" in head else "<f8").reshape(shape).copy()


def test_extract_to_nrrd_at_kernel_radius_5_equals_the_plugins(tmp_path):
    raw, msk = _e2e_volume()
    img, m = I.ArrayImage(raw), I.ArrayImage(msk)
    plug = {c: cls(img, m, voxelBased=True, kernelRadius=5, binWidth=25).execute()
            for c, cls in FC.FEATURE_CLASSES.items()}
    plug["firstorder"] = FC.RadiomicsFirstOrder(img, m, voxelBased=True, kernelRadius=5, binWidth=25).execute()
    d_img, d_msk = torch.from_numpy(raw).cuda(), torch.from_numpy(msk).cuda()
    _, _, lev, levels, Ng = voxel.discretize(d_img, d_msk, binWidth=25)
    s = _lib.make_settings(Ng, len(levels), kernelRadius=5)
    paths = voxel.extract_to_nrrd(lev, s, tmp_path, classes=tuple(plug), compress=False, image=d_img)
    for c, maps in plug.items():
        for f, im in maps.items():
            a = _read_nrrd(paths[f"original_{c}_{f}"], raw.shape)
            b = np.ascontiguousarray(I.as_array(im))
            assert a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8)), (c, f)
