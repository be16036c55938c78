"""Voxel-based first-order maps (csrc/firstorder.cu, firstorder.cuh) against a float64 / long-double restatement of each
kernel window: Minimum / Maximum / Range bit-equal, the percentiles within a few ulps, the moments within a rounding
bound derived from the window size, Entropy / Uniformity against exact level counts, constant windows exactly 0.

Covered: r = 1, 2, 3 (window capacities 27 / 125 / 343), radii clipped per axis by the ROI's extent, 2-D images,
force2D on each axis, unmasked kernels (centers), every device pixel type, initValue, z-slab calls (z0 / z1 / out_z0) and
a volume larger than the kernel's grid (32 blocks of 128 threads per SM), so the grid-stride loop runs."""
import numpy as np
import pytest
import torch

import firstorder_np as FO
import pipeline as PL
from pyradiomics_b200 import featureclasses as FC, image as I
from pyradiomics_b200._lib import DTYPE_CODE, check, lib, ptr, stream

pytestmark = pytest.mark.gpu
U = np.finfo(np.float64).eps / 2                          # unit roundoff of float64
F = {n: k for k, n in enumerate(FO.NAMES)}                 # the kernel's feature order is the oracle's
FLAT_ZERO = ("Variance", "Skewness", "Kurtosis", "MeanAbsoluteDeviation", "RobustMeanAbsoluteDeviation",
             "InterquartileRange")


def _upload(a):
    return torch.from_numpy(np.ascontiguousarray(a).reshape(-1).view(np.uint8)).cuda()


def _fo_device(img, kmask, centers, lev, radii, shift=0.0, vv=1.0, init=0.0, z0=0, z1=None, out=None, out_z0=None):
    """rb_firstorder_voxel_dev on planes [z0, z1): img any device pixel type (Z, Y, X); kmask = voxels that belong to
    kernels (None = all); centers (None = kmask); lev = levels (0 outside), packed to 1 or 2 bytes.  -> (18, nz, Y, X)"""
    Z, Y, X = img.shape
    z1 = Z if z1 is None else z1
    lb = 1 if lev.max() <= 255 else 2
    d_lev = _upload(lev.astype(np.uint8 if lb == 1 else np.uint16))
    d_img = _upload(img)
    d_m = None if kmask is None else _upload(kmask.astype(np.uint8))
    d_c = None if centers is None else _upload(centers.astype(np.uint8))
    if out is None:
        out = torch.full((len(FO.NAMES), z1 - z0, Y, X), -1234.5, dtype=torch.float64, device="cuda")
        out_z0 = z0
    check(lib().rb_firstorder_voxel_dev(ptr(d_img), DTYPE_CODE[img.dtype], ptr(d_m), ptr(d_c), ptr(d_lev), lb, Z, Y, X,
                                        *radii, float(shift), float(vv), float(init), ptr(out), out.stride(0), z0, z1,
                                        out_z0, stream()), "firstorder")
    torch.cuda.synchronize()
    return out


def _windows(vals, kmask, lev, coords, radii):
    """(V, K) window intensities (NaN = outside the volume or the kernel mask) and levels (0 = none) of the centres
    `coords` (3, V)"""
    rz, ry, rx = radii
    pad = ((rz, rz), (ry, ry), (rx, rx))
    P = np.pad(np.where(kmask, vals.astype(np.float64), np.nan), pad, constant_values=np.nan)
    Lp = np.pad(np.where(kmask, lev, 0), pad, constant_values=0)
    off = np.array([(a, b, c) for a in range(-rz, rz + 1) for b in range(-ry, ry + 1) for c in range(-rx, rx + 1)])
    idx = np.asarray(coords).T[:, None, :] + off[None] + np.array(radii)
    return P[idx[..., 0], idx[..., 1], idx[..., 2]], Lp[idx[..., 0], idx[..., 1], idx[..., 2]]


def _check(got, T, L, shift=0.0, vv=1.0, what=""):
    """got: (18, V) maps at the centres; T, L: their windows"""
    g = {n: got[k] for n, k in F.items()}
    ok = ~np.isnan(T)
    n = ok.sum(1)
    xs = np.sort(T, 1)                                     # NaN last
    mn, mx = xs[:, 0], xs[np.arange(len(n)), n - 1]
    # exact
    assert np.array_equal(g["Minimum"], mn), what
    assert np.array_equal(g["Maximum"], mx), what
    assert np.array_equal(g["Range"], mx - mn), what
    # percentiles: the kernel forms pos = (n-1)*q/100, NumPy (n-1)*(q/100): |d pos| <= 3u(n-1), times the range, plus
    # one rounding of the lerp's result
    A = np.maximum(np.abs(mn), np.abs(mx))
    pb = 4 * U * n * (mx - mn) + 2 * np.spacing(A)
    for name, q in (("10Percentile", 10), ("90Percentile", 90)):
        assert (np.abs(g[name] - np.nanpercentile(T, q, axis=1)) <= pb).all(), (what, name)
    assert (np.abs(g["Median"] - np.nanmedian(T, 1)) <= pb).all(), what
    iqr = np.nanpercentile(T, 75, axis=1) - np.nanpercentile(T, 25, axis=1)
    assert (np.abs(g["InterquartileRange"] - iqr) <= 2 * pb + np.spacing(np.abs(iqr))).all(), what
    # moments: long-double two-pass restatement; float64 naive sums of n terms err by <= ~n u of their magnitudes
    x = np.where(ok, T, 0).astype(np.longdouble)
    nl = n.astype(np.longdouble)
    mean = x.sum(1) / nl
    d = np.where(ok, x - mean[:, None], 0)
    M = np.abs(d).max(1)
    m2, m3, m4 = ((d ** k).sum(1) / nl for k in (2, 3, 4))
    dm = 2 * (n + 1) * U * A                               # error of the kernel's mean
    b2 = 2 * dm * M + 2 * (n + 3) * U * M ** 2
    b3 = 3 * dm * M ** 2 + 2 * (n + 4) * U * M ** 3
    b4 = 4 * dm * M ** 3 + 2 * (n + 5) * U * M ** 4
    ref = {"Mean": (mean, dm), "MeanAbsoluteDeviation": (np.abs(d).sum(1) / nl, dm + 2 * (n + 2) * U * M),
           "Variance": (m2, b2)}
    en = (np.where(ok, x + shift, 0) ** 2).sum(1)
    ref["Energy"] = (en, 2 * (n + 2) * U * en)
    ref["TotalEnergy"] = (en * vv, 2 * (n + 3) * U * en * vv)
    ref["RootMeanSquared"] = (np.sqrt(en / nl), (n + 4) * U * np.sqrt(en / nl))
    pos = m2 > 0
    m2s = np.where(pos, m2, 1)
    sk, ku = m3 / m2s ** 1.5, m4 / m2s ** 2
    ref["Skewness"] = (sk, np.where(pos, b3 / m2s ** 1.5 + 1.5 * np.abs(m3) * b2 / m2s ** 2.5 + 4 * U * np.abs(sk), 0))
    ref["Kurtosis"] = (ku, np.where(pos, b4 / m2s ** 2 + 2 * m4 * b2 / m2s ** 3 + 4 * U * ku, 0))
    sel = ok & (T >= g["10Percentile"][:, None]) & (T <= g["90Percentile"][:, None])     # the kernel's own p10 / p90
    kn = sel.sum(1)
    xk = np.where(sel, x, 0)
    km = xk.sum(1) / np.maximum(kn, 1)
    ref["RobustMeanAbsoluteDeviation"] = (np.where(sel, np.abs(xk - km[:, None]), 0).sum(1) / np.maximum(kn, 1),
                                          2 * (2 * kn + 3) * U * np.maximum(A, mx - mn))
    # (no value between p10 and p90, e.g. n = 2: RMAD is 0 / 0, NaN, as the reference's nanmean of nothing)
    assert np.isnan(g["RobustMeanAbsoluteDeviation"][kn == 0]).all(), what
    for name, (r, b) in ref.items():
        err = np.abs(g[name].astype(np.longdouble) - r)[kn > 0]
        assert (err <= np.asarray(b, np.longdouble)[kn > 0] * 1.0001).all(), (what, name, float(err.max()))
    # Entropy / Uniformity from exact level counts: c(i) = how often voxel i's level occurs in its window
    has = L != 0
    c = ((L[:, :, None] == L[:, None, :]) & has[:, None, :]).sum(2)
    N = has.sum(1)
    sq = np.where(has, c, 0).sum(1)                        # sum over levels of count^2
    assert (np.abs(g["Uniformity"] - sq.astype(np.float64) / (N.astype(np.float64) ** 2)) <= 1e-14).all(), what
    p = np.where(has, c, 1).astype(np.longdouble) / N[:, None]
    ent = -np.where(has, np.log2(p + np.longdouble(FO.EPS)) / N[:, None], 0).sum(1)
    assert (np.abs(g["Entropy"] - ent) <= 1e-14).all(), what


def _levels(img, mask, binWidth=25, binCount=None):
    """the product's levels: the reference's binning, integer images in int64 (its edges cannot wrap, DESIGN.md 5)"""
    return PL.bin_image(img.astype(np.int64) if img.dtype.kind in "iu" else img, mask, binWidth, binCount)[0]


def _radii(mask3, r, force2D=False, dim=0, masked=True):
    if masked:
        idx = np.array(np.where(mask3))
        size = idx.max(1) - idx.min(1) + 1
    else:
        size = np.array(mask3.shape)
    rad = [int(min(r, s - 1)) for s in size]
    if force2D:
        rad[dim] = 0
    return rad


def _plugin_case(img, msk, **kw):
    """RadiomicsFirstOrder maps (3-D view) at the centres, checked against the windows and the oracle"""
    sp = (1.0, 1.0, 1.0)[:img.ndim]
    got = FC.RadiomicsFirstOrder(I.ArrayImage(img, sp), I.ArrayImage(msk.astype(np.uint8), sp), voxelBased=True,
                                 **kw).execute()
    maps = np.stack([I.as_array(got[f]) for f in FO.NAMES])
    m = msk.astype(bool)
    masked = kw.get("maskedKernel", True)
    binmask = m if masked else np.ones_like(m)
    lev = _levels(img, binmask, kw.get("binWidth", 25), kw.get("binCount"))
    rad = _radii(m, kw.get("kernelRadius", 1), kw.get("force2D", False), kw.get("force2Ddimension", 0), masked)
    if img.ndim == 2:                                                        # one plane, no window along z
        img3, m3, b3, lev3, maps3, rad = img[None], m[None], binmask[None], lev[None], maps[:, None], [0] + rad
    else:
        img3, m3, b3, lev3, maps3 = img, m, binmask, lev, maps
    T, L = _windows(img3, b3, lev3, np.where(m3), rad)
    at = maps3[:, m3]
    _check(at, T, L, kw.get("voxelArrayShift", 0), 1.0, str(kw))
    assert (maps3[:, ~m3] == kw.get("initValue", 0)).all()
    # and the oracle's float64 restatement agrees
    ref = FO.extract(img.astype(np.int64) if img.dtype.kind in "iu" else img, m, voxelBased=True, **kw)
    for f in FO.NAMES:
        assert np.allclose(at[F[f]], ref[f], rtol=1e-9, atol=1e-9, equal_nan=True), (kw, f)
    return rad


@pytest.mark.parametrize("r", [1, 2, 3])
def test_plugin_maps_at_every_radius(r):
    rng = np.random.default_rng(r)
    img = rng.normal(300, 120, (14, 15, 16)).astype(np.float64)
    msk = rng.random(img.shape) < 0.7
    assert _plugin_case(img, msk, kernelRadius=r, binWidth=25, voxelArrayShift=50) == [r, r, r]


@pytest.mark.parametrize("r", [2, 3])
def test_plugin_radii_clipped_per_axis_by_the_roi_extent(r):
    rng = np.random.default_rng(10 + r)
    img = rng.integers(-200, 900, (12, 13, 14)).astype(np.int16)
    msk = np.zeros(img.shape, bool)
    msk[5:7, 3:6, 1:13] = rng.random((2, 3, 12)) < 0.8                  # bounding box 2 x 3 x 12 (if filled)
    msk[5, 3, 1] = msk[6, 5, 12] = True
    rad = _plugin_case(img, msk, kernelRadius=r, binWidth=25)
    assert rad == [1, 2, r]


@pytest.mark.parametrize("dim", [0, 1, 2])
def test_plugin_force2d_on_each_axis(dim):
    rng = np.random.default_rng(20 + dim)
    img = rng.normal(0, 40, (9, 10, 11)).astype(np.float32)
    msk = rng.random(img.shape) < 0.8
    rad = _plugin_case(img, msk, kernelRadius=2, binWidth=3.5, force2D=True, force2Ddimension=dim)
    assert rad[dim] == 0 and sum(rad) == 4


@pytest.mark.parametrize("r", [1, 3])
def test_plugin_2d_images(r):
    rng = np.random.default_rng(30 + r)
    img = rng.integers(0, 255, (23, 29)).astype(np.uint8)
    msk = rng.random(img.shape) < 0.75
    _plugin_case(img, msk, kernelRadius=r, binWidth=10)


def test_plugin_unmasked_kernel_and_init_value():
    rng = np.random.default_rng(40)
    img = rng.normal(100, 30, (10, 11, 12))
    msk = np.zeros(img.shape, bool)
    msk[2:8, 3:9, 1:10] = rng.random((6, 6, 9)) < 0.6
    _plugin_case(img, msk, kernelRadius=2, binWidth=25, maskedKernel=False, initValue=-7.5)


DEVICE_TYPES = ["int16", "int32", "float32", "float64", "uint8", "uint16", "int64"]


def _typed_image(dtype, shape, rng):
    dt = np.dtype(dtype)
    if np.issubdtype(dt, np.integer):
        lo = 0 if dt.kind == "u" else -3000
        hi = 255 if dt == np.uint8 else 60000 if dt == np.uint16 else 3000
        return rng.integers(lo, hi, shape).astype(dt)
    return (rng.standard_normal(shape) * 700 + 20).astype(dt)


@pytest.mark.parametrize("dtype", DEVICE_TYPES)
def test_every_device_pixel_type_masked_and_unmasked(dtype):
    rng = np.random.default_rng(DEVICE_TYPES.index(dtype) + 50)
    img = _typed_image(dtype, (11, 12, 13), rng)
    m = rng.random(img.shape) < 0.65
    for masked in (True, False):
        kmask = m if masked else np.ones_like(m)
        lev = _levels(img, kmask, binCount=300 if dtype == "uint16" else 40)     # uint16: 2-byte levels
        out = _fo_device(img, kmask if masked else None, None if masked else m, lev, (1, 2, 1), shift=11.0, vv=0.5,
                         init=3.25).cpu().numpy()
        T, L = _windows(img, kmask, lev, np.where(m), (1, 2, 1))
        _check(out[:, m], T, L, 11.0, 0.5, f"{dtype} masked={masked}")
        assert (out[:, ~m] == 3.25).all()


@pytest.mark.parametrize("r", [1, 2, 3])
@pytest.mark.parametrize("dtype", ["int16", "int32", "float32", "uint8"])
def test_constant_windows_have_exactly_zero_spread(dtype, r):
    """piecewise-constant blocks: a window inside one block holds n copies of one integer or float32 value, whose sums
    are exact in double, so Variance, Skewness, Kurtosis, MAD, RMAD and IQR are exactly 0 and Mean / Median the value,
    for every window size n (a random mask varies n; sum * (1/n) misses the value by an ulp for some n > 27)"""
    rng = np.random.default_rng(7 + r)
    b = 2 * r + 3
    blocks = _typed_image(dtype, (4, 4, 5), rng)
    img = np.kron(blocks, np.ones((b, b, b), blocks.dtype))
    msk = rng.random(img.shape) < rng.uniform(0.3, 1.0, img.shape)
    lev = _levels(img, msk)
    out = _fo_device(img, msk, None, lev, (r, r, r)).cpu().numpy()
    z, y, x = np.meshgrid(*(np.arange(s) % b for s in img.shape), indexing="ij")
    inner = msk & (z >= r) & (z < b - r) & (y >= r) & (y < b - r) & (x >= r) & (x < b - r)   # window in one block
    assert inner.sum() > 1000
    for f in FLAT_ZERO:
        v = out[F[f]][inner]
        assert (v == 0).all(), (dtype, f, v[v != 0][:5])
    assert np.array_equal(out[F["Mean"]][inner], img[inner].astype(np.float64))
    assert np.array_equal(out[F["Median"]][inner], img[inner].astype(np.float64))


def test_z_slabs_equal_one_call():
    rng = np.random.default_rng(60)
    img = rng.normal(50, 20, (17, 12, 14)).astype(np.float32)
    m = rng.random(img.shape) < 0.7
    lev = _levels(img, m, 2.5)
    full = _fo_device(img, m, None, lev, (2, 1, 2), shift=3.0, init=-1.0)
    cuts = [0, 5, 11, 17]
    parts = [_fo_device(img, m, None, lev, (2, 1, 2), shift=3.0, init=-1.0, z0=a, z1=b) for a, b in zip(cuts, cuts[1:])]
    assert torch.equal(torch.cat(parts, 1), full)
    into = torch.full_like(full, np.nan)
    for a, b in zip(cuts, cuts[1:]):                                         # slabs written into one buffer
        _fo_device(img, m, None, lev, (2, 1, 2), shift=3.0, init=-1.0, z0=a, z1=b, out=into, out_z0=0)
    assert torch.equal(into, full)
    # a buffer that starts at plane 4 (out_z0 = 4) holds planes 4..16
    tail = torch.full((len(FO.NAMES), 13) + img.shape[1:], np.nan, dtype=torch.float64, device="cuda")
    _fo_device(img, m, None, lev, (2, 1, 2), shift=3.0, init=-1.0, z0=4, z1=17, out=tail, out_z0=4)
    assert torch.equal(tail, full[:, 4:])


def test_grid_stride_loop_on_a_large_volume():
    """128 x 128 x 100 = 1.6 M centres > 32 blocks x 128 threads x 132 SMs: Minimum / Maximum / Range of every voxel
    exactly, all features on a sample of 20 000 centres spread over the whole volume"""
    rng = np.random.default_rng(70)
    img = (rng.standard_normal((100, 128, 128)) * 300).astype(np.float32)
    m = rng.random(img.shape) < 0.9
    lev = _levels(img, m)
    out = _fo_device(img, m, None, lev, (1, 1, 1), shift=7.0)
    got = {f: out[F[f]].cpu().numpy() for f in ("Minimum", "Maximum", "Range")}
    P = np.pad(np.where(m, img.astype(np.float64), np.nan), 1, constant_values=np.nan)
    lo = np.full(img.shape, np.inf)
    hi = np.full(img.shape, -np.inf)
    Z, Y, X = img.shape
    for a in range(3):
        for b in range(3):
            for c in range(3):
                v = P[a:a + Z, b:b + Y, c:c + X]
                lo, hi = np.fmin(lo, v), np.fmax(hi, v)
    assert np.array_equal(got["Minimum"][m], lo[m]) and np.array_equal(got["Maximum"][m], hi[m])
    assert np.array_equal(got["Range"][m], (hi - lo)[m])
    assert (got["Minimum"][~m] == 0).all()
    coords = np.array(np.where(m))
    pick = np.sort(rng.choice(coords.shape[1], 20000, replace=False))
    pick[-1] = coords.shape[1] - 1                                           # the last centre is in the last pass
    sub = coords[:, pick]
    T, L = _windows(img, m, lev, sub, (1, 1, 1))
    at = out[:, torch.as_tensor(sub[0]).cuda(), torch.as_tensor(sub[1]).cuda(), torch.as_tensor(sub[2]).cuda()]
    _check(at.cpu().numpy(), T, L, 7.0, 1.0, "large")
