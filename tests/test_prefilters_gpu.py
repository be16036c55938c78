"""The kernels in front of the texture engine on every launch path: the fused 3-D stationary wavelet kernel at all four
tap counts, slabs and ragged tiles, the axis-by-axis wavelet kernel up to 24 taps, the recursive-Gaussian LoG passes on
anisotropic spacing, float64 input and grid-stride shapes, and the B-spline resampler (prefilter, evaluation, cast) for
every pixel type.  Each is compared with a float64 restatement of the same operation (oracle/filters_np.py,
oracle/resample_np.py) at a tolerance set by its rounding, not by the feature tolerances."""
import numpy as np
import pytest
import scipy.ndimage as ndi
import torch

import filters_np as FN
import resample_np as RS
from helpers import (RESAMPLE_DTYPES, RESAMPLE_NEAR_TIE_SHARE, RESAMPLE_NEW_SPACING_XYZ, RESAMPLE_SPACING_XYZ, log_bound,
                     near_integer, resample_case)
from pyradiomics_b200 import distributed as D, image as I, imageoperations as IO
from pyradiomics_b200._lib import DTYPE_CODE, B200Error, check, lib, ptr, stream

pytestmark = pytest.mark.gpu

# PyWavelets' db4 decomposition low-pass filter (published to ~1e-12)
DB4 = [-0.010597401784997278, 0.032883011666982945, 0.030841381835986965, -0.18703481171888114, -0.02798376941698385,
       0.6308807679295904, 0.7148465705525415, 0.23037781330885523]


class Taps:
    """a pywt.Wavelet-like object: what getWaveletImage accepts for wavelets outside the built-in table"""

    def __init__(self, lo, hi=None):
        self.dec_lo = list(lo)
        F = len(lo)
        self.dec_hi = list(hi) if hi is not None else [(-1) ** (k + 1) * lo[F - 1 - k] for k in range(F)]


def _random_taps(F, seed=0):
    rng = np.random.default_rng(100 + F + seed)
    return Taps(rng.normal(size=F) / np.sqrt(F), rng.normal(size=F) / np.sqrt(F))


def _builtin_or_random(F):
    return {2: "haar", 4: "db2", 6: "coif1"}.get(F) or _random_taps(F)


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _names(levels, nd):
    out = {}
    for idx, dec in enumerate(levels, start=1):
        for key, arr in dec.items():
            band = key.replace("a", "L").replace("d", "H")
            out[f"wavelet-{band}" if idx == 1 else f"wavelet{idx}-{band}"] = arr
    return out


def _check_wavelet_image(x, wavelet, level, start_level):
    lo, hi = IO.wavelet_filters(wavelet)
    nd = x.ndim
    approx, levels = FN.swt3_levels(x, lo, hi, tuple(range(nd - 1, -1, -1)), level, start_level)
    ref = _names(levels, nd)
    ref[f"wavelet-{'L' * nd}" if level == 1 else f"wavelet{level}-{'L' * nd}"] = approx
    got = {n: I.as_array(im) for im, n, _ in IO.getWaveletImage(I.ArrayImage(x), None, wavelet=wavelet, level=level,
                                                                  start_level=start_level)}
    assert set(got) == set(ref)
    scale = max(np.abs(v).max() for v in ref.values())
    for n, v in ref.items():
        assert got[n].shape == v.shape
        assert np.abs(got[n] - v).max() <= 1e-12 * scale, n


# ------------------------------------------------------------------------------------------------------------ wavelet
@pytest.mark.parametrize("F", [2, 4, 6, 8])
@pytest.mark.parametrize("shape", [(10, 22, 70), (6, 2, 2), (2, 14, 40)], ids=["ragged-tiles", "short-axes", "z2"])
def test_fused_kernel_matches_restatement(F, shape):
    """even sizes (the fused kernel is purely periodic): 22 rows = 3 tiles of 8 with a ragged one, 70 columns = 3 tiles
    of 32 with a ragged one; Y = X = 2 shorter than every filter but haar; Z = 2"""
    x = np.random.default_rng(F).normal(size=shape)
    lo, hi = IO.wavelet_filters(_builtin_or_random(F))
    assert lo.size == F
    got = IO.swt_level1_device(torch.as_tensor(x, device="cuda"), (2, 1, 0), lo, hi)
    ref = FN.swtn_level1(x, lo, hi, (2, 1, 0))
    assert set(got) == set(ref)
    for k, v in ref.items():
        assert np.abs(got[k].cpu().numpy() - v).max() <= 1e-12 * np.abs(x).max(), k


def test_fused_db4_is_an_isometry():
    lo = np.array(DB4)
    assert abs(lo.sum() - np.sqrt(2)) < 1e-11 and abs((lo ** 2).sum() - 1) < 1e-11
    for m in (1, 2, 3):                                   # double-shift orthogonality
        assert abs(np.dot(lo[2 * m:], lo[:8 - 2 * m])) < 1e-11
    lo, hi = IO.wavelet_filters(Taps(DB4))
    x = np.random.default_rng(4).normal(size=(12, 18, 40))
    got = IO.swt_level1_device(torch.as_tensor(x, device="cuda"), (2, 1, 0), lo, hi)
    e = sum(float((t.double() ** 2).sum()) for t in got.values())
    assert abs(e - 8 * (x ** 2).sum()) <= 1e-10 * e
    const = IO.swt_level1_device(torch.full((6, 10, 34), 3.0, dtype=torch.float64, device="cuda"), (2, 1, 0), lo, hi)
    for k, t in const.items():
        assert np.allclose(t.cpu().numpy(), 3.0 * 2 ** 1.5 if k == "aaa" else 0.0, atol=1e-10), k


@pytest.mark.parametrize("F", [10, 12, 20, 24])
@pytest.mark.parametrize("shape", [(8, 10, 12), (7, 9, 11), (10, 12), (9, 11)])
def test_axis_kernel_long_filters_through_getWaveletImage(F, shape):
    """more than 8 taps (coif2 has 12, db5 / sym5 10, db10 20): one axis per pass, the odd sizes wrap-padded by index"""
    x = np.random.default_rng(F + len(shape)).normal(size=shape)
    _check_wavelet_image(x, _random_taps(F), level=2, start_level=1)


def test_filter_length_limits():
    x = torch.randn((4, 6, 8), dtype=torch.float64, device="cuda")
    for F in (1, 25):
        with pytest.raises(B200Error):
            list(IO.getWaveletImage(I.ArrayImage(x.cpu().numpy()), None, wavelet=_random_taps(F)))
    lo, hi = IO.wavelet_filters(_random_taps(10))
    with pytest.raises(ValueError):
        IO.swt_level1_device(x, (2, 1, 0), lo, hi, z_range=(1, 3))


@pytest.mark.parametrize("F", [6, 8])
@pytest.mark.parametrize("Z,world", [(13, 3), (13, 4), (4, 3), (4, 4)])
def test_fused_kernel_slabs_are_bit_identical(F, Z, world):
    """each slab's buffer holds F-1-F/2 planes below and F/2 above, wrapped around the volume like
    SlabHalo(periodic=True); z_range asks for the slab's own planes (Z = 4 splits into one-plane slabs)"""
    lo, hi = IO.wavelet_filters(_builtin_or_random(F))
    x = torch.randn((Z, 19, 40), dtype=torch.float64, device="cuda", generator=torch.Generator(device="cuda").manual_seed(Z + F))
    whole = IO.swt_level1_device(x, (2, 1, 0), lo, hi)
    below, above = F - 1 - F // 2, F // 2
    sizes = []
    for rank in range(world):
        z0, z1 = D.slab_range(Z, rank, world)
        sizes.append(z1 - z0)
        buf = x[torch.arange(z0 - below, z1 + above, device="cuda") % Z].contiguous()
        part = IO.swt_level1_device(buf, (2, 1, 0), lo, hi, z_range=(below, below + z1 - z0))
        for k, t in whole.items():
            assert torch.equal(part[k], t[z0:z1]), (rank, k)
    assert sum(sizes) == Z and (Z != 4 or min(sizes) == 1)


@pytest.mark.parametrize("F", [2, 4, 6, 8])
@pytest.mark.parametrize("level", [1, 2])
@pytest.mark.parametrize("shape", [(9, 11, 13), (7, 10, 33)])
def test_fused_kernel_odd_sizes_through_getWaveletImage(F, level, shape):
    """getWaveletImage wrap-pads the odd axes once and then runs the periodic fused kernel on the even volume"""
    x = np.random.default_rng(F * 10 + level).normal(size=shape)
    _check_wavelet_image(x, _builtin_or_random(F), level=level, start_level=0)


# ------------------------------------------------------------------------------------------------------------ LoG
SPACING_XYZ = (0.6, 0.8, 2.0)


def _check_log(got, x, sigma, spacing_zyx, in_dtype):
    ref, terms = FN.log_restatement(x, sigma, spacing_zyx, in_dtype=in_dtype, return_terms=True)
    assert got.dtype == np.float32 and got.shape == ref.shape
    d = np.abs(got.astype(np.float64) - ref.astype(np.float64))
    bound = log_bound(terms, x)
    worst = float((d / bound).max())
    same = int((got == ref).sum())
    print(f"LoG {np.dtype(in_dtype).name} sigma {sigma} shape {x.shape}: {same} of {got.size} voxels bit-identical, "
          f"worst |diff| / bound {worst:.3g}")
    assert (d <= bound).all(), worst
    return same


@pytest.mark.parametrize("dtype", ["float32", "int16", "float64"])
@pytest.mark.parametrize("sigma", [2.0, 3.0])
def test_log_anisotropic_matches_restatement_and_analytic_laplacian(dtype, sigma):
    x = ndi.gaussian_filter(np.random.default_rng(7).normal(size=(30, 56, 72)), 2.0) * 1000
    arr = x.astype(dtype)
    spacing_zyx = SPACING_XYZ[::-1]
    out = [I.as_array(im) for im, n, _ in IO.getLoGImage(I.ArrayImage(arr, SPACING_XYZ), None, sigma=[sigma])]
    assert len(out) == 1
    _check_log(out[0], arr, sigma, spacing_zyx, arr.dtype)
    # analytic sigma^2-normalised Laplacian with sigma_d = sigma / spacing_d voxels (SciPy FIR, no shared coefficients)
    s = [sigma / v for v in spacing_zyx]
    xf = arr.astype(np.float64)
    ana = sum(s[d] ** 2 * ndi.gaussian_filter(xf, s, order=[2 if e == d else 0 for e in range(3)], mode="nearest",
                                              truncate=6.0) for d in range(3))
    c = tuple(slice(int(np.ceil(4 * v)) + 2, -int(np.ceil(4 * v)) - 2) for v in s)
    err = np.abs(out[0][c] - ana[c]).max() / np.abs(ana[c]).max()
    assert err < 0.03, err


@pytest.mark.parametrize("shape,axis", [((300, 1000, 4), 2), ((400, 4, 400), 1), ((4, 400, 400), 0), ((6, 7, 33), None),
                                        ((5, 9, 65), None), ((7, 6, 4), None)],
                         ids=["x-lines", "y-lines", "z-lines", "X33", "X65", "X4"])
def test_log_grid_stride_and_partial_tiles(shape, axis):
    """the first three shapes give the launches along `axis` more lines than their grid holds (x: grid_for(lines / 32, 4,
    16) blocks of 4 warps x 32 lines; y / z: grid_for(lines, 128, 8) blocks of 128 lines), so the grid-stride loop sweeps
    twice; the last three end in a partial 32-column x tile"""
    Z, Y, X = shape
    lines = {0: Y * X, 1: Z * X, 2: Z * Y}
    if axis is not None:
        assert lines[axis] > _sms() * (16 * 4 * 32 if axis == 2 else 8 * 128)
    x = np.random.default_rng(sum(shape)).normal(size=shape).astype(np.float32) * 100
    spacing_zyx = SPACING_XYZ[::-1]
    got = IO.log_filter_device(torch.as_tensor(x, device="cuda"), 1.5, spacing_zyx).cpu().numpy()
    _check_log(got, x, 1.5, spacing_zyx, np.float32)


@pytest.mark.parametrize("in_dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_log_single_pass_both_input_types(in_dtype, axis):
    """one pass of each kernel (x: recursive_gauss_x_kernel, y / z: recursive_gauss_axis_kernel) with float32 and float64
    input, plain and accumulating: float32((causal + anti-causal) * scale) of the float64 recursion"""
    x = torch.randn((9, 21, 70), dtype=in_dtype, device="cuda", generator=torch.Generator(device="cuda").manual_seed(axis)) * 50
    xn = x.cpu().numpy().astype(np.float64)
    for order, sigma, scale in ((0, 1.7, 1.0), (2, 2.3, 2.3 ** 2)):
        ref = (FN.recursive_gaussian_axis(xn, IO.recursive_gaussian_coefficients(sigma, order), axis) * scale).astype(np.float32)
        got = IO._rg_pass(x, axis, sigma, order, scale=scale).cpu().numpy()
        assert (np.abs(got - ref) <= np.spacing(np.abs(ref))).all()
        acc = torch.full(x.shape, 0.25, dtype=torch.float32, device="cuda")
        IO._rg_pass(x, axis, sigma, order, out=acc, scale=scale, accumulate=True)
        assert (np.abs(acc.cpu().numpy() - (np.float32(0.25) + ref)) <= 2 * np.spacing(np.abs(ref) + 0.25)).all()


@pytest.mark.parametrize("parts", [2, 3])
def test_log_z_pass_hook_on_y_ranges_is_bit_identical(parts):
    """the single-GPU form of pipeline.derived_images_slab: the z pass run on separate y-ranges of the volume"""
    x = torch.randn((23, 17, 40), dtype=torch.float32, device="cuda", generator=torch.Generator(device="cuda").manual_seed(parts))
    Y = x.shape[1]

    def z_pass(t, sigma_vox, order, scale):
        out = torch.empty(t.shape, dtype=torch.float32, device=t.device)
        for k in range(parts):
            y0, y1 = D.slab_range(Y, k, parts)
            out[:, y0:y1] = IO._rg_pass(t[:, y0:y1].contiguous(), 0, sigma_vox, order, scale=scale)
        return out

    spacing_zyx = SPACING_XYZ[::-1]
    assert torch.equal(IO.log_filter_device(x, 2.0, spacing_zyx, z_pass=z_pass), IO.log_filter_device(x, 2.0, spacing_zyx))


# ------------------------------------------------------------------------------------------------------------ resampling
def _prefilter(x):
    t = torch.as_tensor(np.ascontiguousarray(x, dtype=np.float64), device="cuda").clone()
    check(lib().rb_bspline_prefilter_dev(ptr(t), *t.shape, stream()), "bspline prefilter")
    return t


@pytest.mark.parametrize("n", [1, 2, 3, 18, 19, 64, 199, 200, 300])
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_bspline_prefilter_matches_itk_restatement(n, axis):
    """X = 199 is the longest line of the shared-memory x tile, X >= 200 takes the strided kernel; N = 18 is the last
    length with the closed-form causal start"""
    shape = [3, 5, 7]
    shape[axis] = n
    x = np.random.default_rng(n + axis).normal(size=shape) * 1000
    ref = RS.bspline_coefficients(x, exact=False)
    got = _prefilter(x).cpu().numpy()
    assert np.abs(got - ref).max() <= 1e-13 * np.abs(ref).max()


@pytest.mark.parametrize("shape", [(300, 240, 4), (400, 4, 400), (4, 400, 400)], ids=["x", "y", "z"])
def test_bspline_prefilter_grid_stride(shape):
    Z, Y, X = shape
    x_cap, axis_cap = _sms() * 4 * 4 * 32, _sms() * 8 * 128          # lines per sweep of the x-tile / strided launches
    assert Z * Y > x_cap if X == 4 else (Z * X > axis_cap if Y == 4 else Y * X > axis_cap)
    x = np.random.default_rng(Z + X).normal(size=shape) * 1000
    ref = RS.bspline_coefficients(x, exact=False)
    assert np.abs(_prefilter(x).cpu().numpy() - ref).max() <= 1e-13 * np.abs(ref).max()


def _resample_f64(src, interp, osz, start, step, default):
    src_t = torch.as_tensor(np.ascontiguousarray(src, dtype=np.float64), device="cuda")
    dst = torch.empty(osz, dtype=torch.float64, device="cuda")
    import ctypes as C
    code = DTYPE_CODE[np.dtype(np.float64)]
    check(lib().rb_resample_dev(ptr(src_t), code, (C.c_int * 3)(*src.shape), ptr(dst), code, (C.c_int * 3)(*osz),
                                (C.c_double * 3)(*start), (C.c_double * 3)(*step), interp, default, stream()), "resample")
    return dst.cpu().numpy()


RESAMPLE_GEOMETRIES = {          # no coordinate lies on a half sample (nearest neighbour and the inside test have no ties)
    "down": ((12, 20, 17), (9, 9, 7), (0.1234, -0.2113, 0.3071), (1.3137, 1.7071, 2.2361)),
    "up": ((8, 11, 13), (17, 23, 30), (-0.3071, 0.0512, -0.4123), (0.4513, 0.4671, 0.4319)),
    "past-every-face": ((7, 9, 11), (14, 17, 20), (-2.3117, -1.7213, -3.1071), (0.7071, 0.8123, 0.9137)),
    "size-1-axis": ((1, 12, 15), (3, 20, 22), (-0.3117, 0.2071, -0.1213), (0.2513, 0.5471, 0.6519)),
    "two-sweeps": ((20, 24, 28), (70, 70, 70), (-0.2071, 0.1123, 0.1517), (0.2813, 0.3319, 0.3807)),
}


@pytest.mark.parametrize("interp", [0, 1, 3])
@pytest.mark.parametrize("geom", list(RESAMPLE_GEOMETRIES))
def test_resample_kernel_matches_oracle_evaluation(interp, geom):
    """float64 output (no cast) against the oracle's evaluation of the same coefficients; outside the input buffer the
    default value exactly"""
    shape, osz, start, step = RESAMPLE_GEOMETRIES[geom]
    if geom == "two-sweeps":
        assert np.prod(osz) > _sms() * 8 * 256
    x = np.random.default_rng(interp).normal(size=shape) * 1000
    src = _prefilter(x).cpu().numpy() if interp == 3 else x
    default = -123.25
    got = _resample_f64(src, interp, osz, start, step, default)
    ref = RS.evaluate(src, osz, start, step, interp, default_value=np.nan)
    outside = np.isnan(ref)
    assert (got[outside] == default).all()
    assert np.abs(got[~outside] - ref[~outside]).max() <= 1e-12 * np.abs(src).max()
    if geom == "past-every-face":
        for ax in range(3):
            assert outside.take(0, axis=ax).all() and outside.take(-1, axis=ax).all()
    else:
        assert not outside.any()


@pytest.mark.parametrize("dtype", RESAMPLE_DTYPES)
def test_resampleImage_casts_every_pixel_type_like_itk(dtype):
    """B-spline resampling of i.i.d. full-range values overshoots both ends of the type: every integer voxel equals the
    oracle's clamp + truncation except the counted near-ties; float32 within 1 ulp; masks bit-identical"""
    img, msk = resample_case(dtype)
    sp = RESAMPLE_SPACING_XYZ
    ri, rm = IO.resampleImage(I.ArrayImage(img, sp), I.ArrayImage(msk, sp), resampledPixelSpacing=list(RESAMPLE_NEW_SPACING_XYZ),
                              interpolator="sitkBSpline", padDistance=20)
    val, out, m, _ = RS.resample_itk(img, msk, sp, RESAMPLE_NEW_SPACING_XYZ, padDistance=20)
    got = ri.array
    assert got.dtype == img.dtype and got.shape == out.shape
    assert rm.array.dtype == msk.dtype and np.array_equal(rm.array, m)
    tau = 1e-12 * np.abs(RS.bspline_coefficients(img)).max()
    if np.issubdtype(img.dtype, np.integer):
        info = np.iinfo(img.dtype)
        if img.dtype.itemsize < 8:
            assert (got == info.min).any() and (got == info.max).any()           # both clamps hit
        ties = near_integer(val, tau) & (val != 0)                               # (outside the buffer: exactly 0)
        diff = got != out
        print(f"resampleImage {dtype}: {int(ties.sum())} of {val.size} voxels within tau = {tau:.3g} of an integer "
              f"excluded, {int((diff & ties).sum())} of them differ")
        assert not (diff & ~ties).any(), np.argwhere(diff & ~ties)[:5]
        assert ties.mean() <= RESAMPLE_NEAR_TIE_SHARE
        if diff.any():
            assert np.abs(got[diff].astype(np.float64) - out[diff].astype(np.float64)).max() <= 1
    elif img.dtype == np.float32:
        assert (np.abs(got.astype(np.float64) - out.astype(np.float64)) <= np.spacing(np.abs(out))).all()
    else:
        assert np.abs(got - val).max() <= tau
