"""The kernelRadius-1 first-order tile kernel (csrc/firstorder.cu firstorder_tiles_kernel: full-window body + deferred
generic body) against the generic kernel (B200_RADIOMICS_FORCE_GENERIC=1) through rb_firstorder_voxel_dev, bit for bit,
NaN positions included; the first-order maps of the device-resident filter suite (pipeline.voxel_suite_with_filters)
against the oracle; and extract_to_nrrd's first-order files against the plugin class."""
import os

import numpy as np
import pytest
import torch

import firstorder_np as FO
from pyradiomics_b200 import _lib, featureclasses as FC, image as I, imageoperations as IO, pipeline, voxel
from pyradiomics_b200._lib import TORCH_DTYPE_CODE, check, lib, ptr, stream
from test_firstorder_full_window_emul import INT_RANGES, level_windows, special_windows

pytestmark = pytest.mark.gpu
NF = 18
FO_NT = 128                      # firstorder.cu FO_NT: one tile = 128 consecutive voxels of the chunk
MAX_BLOCKS_PER_SM = 32           # sm_90's limit: the resident grid (resident_grid) never exceeds SMs x 32 blocks


def _fo(img, kmask, centers, lev, radii=(1, 1, 1), shift=0.0, vv=1.0, init=0.0, z0=0, z1=None, out_z0=None, out=None,
        generic=False):
    """rb_firstorder_voxel_dev on CUDA tensors; generic=True forces the generic kernel"""
    Z, Y, X = lev.shape
    z1 = Z if z1 is None else z1
    if out is None:
        out = torch.full((NF, z1 - z0, Y, X), -1234.5, dtype=torch.float64, device="cuda")
        out_z0 = z0
    old = os.environ.get("B200_RADIOMICS_FORCE_GENERIC")
    os.environ["B200_RADIOMICS_FORCE_GENERIC"] = "1" if generic else "0"
    try:
        check(lib().rb_firstorder_voxel_dev(ptr(img), TORCH_DTYPE_CODE[img.dtype], ptr(kmask), ptr(centers), ptr(lev),
                                            voxel.level_bytes(lev), Z, Y, X, *radii, float(shift), float(vv), float(init),
                                            ptr(out), out.stride(0), z0, z1, out_z0, stream()), "firstorder")
        torch.cuda.synchronize()
    finally:
        if old is None:
            del os.environ["B200_RADIOMICS_FORCE_GENERIC"]
        else:
            os.environ["B200_RADIOMICS_FORCE_GENERIC"] = old
    return out


def _same_bits(a, b, what=""):
    assert a.shape == b.shape and a.dtype == b.dtype == torch.float64, what
    eq = a.view(torch.int64) == b.view(torch.int64)
    assert bool(eq.all()), (what, int((~eq).sum()), torch.nonzero(~eq)[:5].tolist())


def _fast_equals_generic(img, kmask, centers, lev, what, **kw):
    fast = _fo(img, kmask, centers, lev, **kw)
    gen = _fo(img, kmask, centers, lev, generic=True, **kw)
    _same_bits(fast, gen, what)
    return fast


# the device pixel types: (torch type, NumPy range type); uint16 travels as int32
DTYPES = [(torch.int16, "int16"), (torch.int32, "int32"), (torch.float32, None), (torch.float64, None),
          (torch.uint8, "uint8"), (torch.int64, "int64"), (torch.int32, "uint16")]


def _cast_window(w, tdt, rng_name):
    """the window in the pixel type, or None when it does not fit (NaN, or a float window for an integer type)"""
    if rng_name is None:
        with np.errstate(over="ignore"):                                   # float32: 1e300 becomes inf
            return w.astype(np.float32 if tdt == torch.float32 else np.float64)
    if not np.isfinite(w).all():
        return None
    lo, hi = INT_RANGES[rng_name]
    return np.clip(np.round(w), lo, min(hi, 2 ** 63 - 1024)).astype(np.float64)    # int64: the largest double below 2^63


def _planted(tdt, rng_name, seed):
    """a volume tiled with 3x3x3 blocks that each hold one adversarial window (the window of the block's centre) and
    its levels (1 to 27 classes)"""
    rng = np.random.default_rng(seed)
    wins = [w for w in (_cast_window(x, tdt, rng_name) for x in special_windows(rng)) if w is not None]
    nb = (4, 8, 8)
    shape = tuple(3 * n for n in nb)
    img = np.zeros(shape)
    lev = np.zeros(shape, np.int64)
    k = 0
    for a in range(nb[0]):
        for b in range(nb[1]):
            for c in range(nb[2]):
                x = wins[k % len(wins)]
                levs = [w for w in level_windows(rng, x) if w.max() <= 255]      # 8-bit levels
                img[3 * a:3 * a + 3, 3 * b:3 * b + 3, 3 * c:3 * c + 3] = x.reshape(3, 3, 3)
                lev[3 * a:3 * a + 3, 3 * b:3 * b + 3, 3 * c:3 * c + 3] = levs[k % len(levs)].reshape(3, 3, 3)
                k += 1
    return img, lev


def _to_dev(a, tdt, rng_name):
    if rng_name is None:
        return torch.from_numpy(np.ascontiguousarray(a)).to(tdt).cuda()
    if a.dtype != np.int64:
        a = a.astype(np.int64)
    return torch.from_numpy(np.ascontiguousarray(a.astype(rng_name))).to(tdt).cuda()


def _random_case(tdt, rng_name, shape, seed):
    """random intensities of the pixel type, a ROI with holes that touches all six faces, levels 0 outside it"""
    rng = np.random.default_rng(seed)
    if rng_name is None:
        img = np.round(rng.normal(0, 30, shape), 1)
        img[rng.random(shape) < 0.05] = -0.0
        img[rng.random(shape) < 0.05] = 0.0
    else:
        lo, hi = INT_RANGES[rng_name]
        vals = rng.integers(max(lo, -1000), min(hi, 1000), shape, endpoint=True, dtype=np.int64)
        img = np.where(rng.random(shape) < 0.2, rng.choice(np.array([lo, hi], np.int64), shape), vals)
    roi = rng.random(shape) > 0.1
    lev = np.where(roi, rng.integers(1, 9, shape), 0)
    return img, roi, lev


@pytest.mark.parametrize("tdt,rng_name", DTYPES, ids=[f"{t}".split(".")[1] + (f"-{n}" if n else "") for t, n in DTYPES])
def test_tile_kernel_equals_generic_kernel_on_adversarial_windows(tdt, rng_name):
    img, lev = _planted(tdt, rng_name, 11)
    d_img = _to_dev(img, tdt, rng_name)
    d_lev = torch.from_numpy(lev.astype(np.uint8)).cuda()
    ones = torch.ones(lev.shape, dtype=torch.uint8, device="cuda")
    for kmask in (ones, None):
        for shift, init in ((0.0, 0.0), (1000.0, -7.5)):
            out = _fast_equals_generic(d_img, kmask, None, d_lev, f"planted {tdt} {rng_name}", shift=shift, vv=0.42, init=init)
    # the block centres hold the planted windows: their Minimum is the window's
    mins = out[FO.NAMES.index("Minimum"), 1::3, 1::3, 1::3].cpu().numpy()
    blocks = img.reshape(4, 3, 8, 3, 8, 3).transpose(0, 2, 4, 1, 3, 5).reshape(4, 8, 8, 27)
    assert np.array_equal(mins, blocks.min(-1).astype(mins.dtype))


@pytest.mark.parametrize("tdt,rng_name", DTYPES, ids=[f"{t}".split(".")[1] + (f"-{n}" if n else "") for t, n in DTYPES])
def test_tile_kernel_equals_generic_kernel_with_roi_holes_faces_and_slabs(tdt, rng_name):
    img, roi, lev = _random_case(tdt, rng_name, (9, 13, 150), 5)
    d_img = _to_dev(img, tdt, rng_name)
    d_roi = torch.from_numpy(roi.astype(np.uint8)).cuda()
    d_lev = torch.from_numpy(lev.astype(np.uint8)).cuda()
    whole = _fast_equals_generic(d_img, d_roi, None, d_lev, "holes", shift=3.0, vv=2.0, init=0.5)
    assert (whole[:, ~torch.from_numpy(roi).cuda()] == 0.5).all()
    # z-slabs into a shared buffer, and a slab with its own out_z0, equal the whole-volume call
    for generic in (False, True):
        buf = torch.full_like(whole, -1.0)
        for za, zb in ((0, 4), (4, 5), (5, 9)):
            _fo(d_img, d_roi, None, d_lev, shift=3.0, vv=2.0, init=0.5, z0=za, z1=zb, out_z0=0, out=buf, generic=generic)
        _same_bits(buf, whole, f"slabs generic={generic}")
    part = _fo(d_img, d_roi, None, d_lev, shift=3.0, vv=2.0, init=0.5, z0=2, z1=7)
    _same_bits(part, whole[:, 2:7], "out_z0")


@pytest.mark.parametrize("tdt", [torch.float32, torch.float64])
def test_tile_kernel_equals_generic_kernel_unmasked_with_nan_and_inf_outside_the_roi(tdt):
    rng = np.random.default_rng(7)
    shape = (8, 12, 40)
    img = rng.normal(0, 5, shape)
    roi = np.zeros(shape, bool)
    roi[1:7, 2:10, 3:37] = True
    roi &= rng.random(shape) > 0.05
    out_roi = ~roi
    img[out_roi & (rng.random(shape) < 0.3)] = np.nan
    img[out_roi & (rng.random(shape) < 0.2)] = np.inf
    img[out_roi & (rng.random(shape) < 0.2)] = -np.inf
    lev = rng.integers(1, 12, shape)                         # an unmasked kernel: levels everywhere
    d_img = torch.from_numpy(img).to(tdt).cuda()
    d_lev = torch.from_numpy(lev.astype(np.uint8)).cuda()
    d_c = torch.from_numpy(roi.astype(np.uint8)).cuda()
    out = _fast_equals_generic(d_img, None, d_c, d_lev, "unmasked", shift=-2.0, init=1.0)
    assert torch.isnan(out).any() and torch.isinf(out).any()


def test_tile_kernel_equals_generic_kernel_when_every_block_runs_three_tiles():
    shape = (7, 1024, 1024)
    total = shape[0] * shape[1] * shape[2]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = -(-total // FO_NT)
    assert tiles >= 3 * sms * MAX_BLOCKS_PER_SM               # every block of the resident grid walks >= 3 tiles
    g = torch.Generator(device="cuda").manual_seed(3)
    lev = torch.randint(1, 33, shape, device="cuda", generator=g, dtype=torch.int32)
    roi = (torch.rand(shape, device="cuda", generator=g) > 0.02).to(torch.uint8)
    lev = (lev * roi).to(torch.uint8)
    img = ((lev.to(torch.int32) - 1) * 25 + 3).to(torch.int16)
    _fast_equals_generic(img, roi, None, lev, "large", shift=0.0)


# ---------------------------------------------------------------------------------------------- pipeline and NRRD
def _suite_case(shape=(14, 18, 20), seed=21):
    rng = np.random.default_rng(seed)
    z, y, x = np.meshgrid(*(np.linspace(-1, 1, n) for n in shape), indexing="ij")
    img = 400 * np.exp(-(x ** 2 + y ** 2 + z ** 2)) + rng.normal(0, 20, shape)
    msk = np.zeros(shape, np.uint8)
    msk[1:-2, 2:-2, 2:-1] = 1
    msk[tuple(n // 2 for n in shape)] = 0                                  # a hole
    return torch.from_numpy(img.astype(np.float32)).cuda(), torch.from_numpy(msk).cuda()


SUITE = dict(sigmas=(1.0,), image_types=("square",), normalize={}, resegment={"resegmentRange": [-2.5, 2.5],
             "resegmentMode": "sigma"}, binWidth=0.2, voxelArrayShift=300, spacing_zyx=(1.5, 0.9, 0.8))


def _run_suite(img, msk, classes, map_dtype=torch.float64, **kw):
    maps = {}
    info = pipeline.voxel_suite_with_filters(img, msk, classes=classes, map_dtype=map_dtype,
                                             consume=lambda name, c, m: maps.__setitem__((name, c), m.clone()), **kw)
    return maps, info


def test_suite_firstorder_maps_match_the_oracle_on_every_derived_image():
    img, msk = _suite_case()
    kw = dict(SUITE)
    classes = ("firstorder", "glrlm", "ngtdm")
    got, info = _run_suite(img, msk, classes, **kw)
    plain, _ = _run_suite(img, msk, ("glrlm", "ngtdm"), **kw)
    names = [n for n, _, _ in info]
    assert len(names) == 1 + 8 + 1 + 1
    for key, m in plain.items():                              # texture maps do not change with first order beside them
        _same_bits(got[key], m, str(key))
    # the derived images the suite saw: normalised image, resegmented ROI
    x = IO.normalize_image_device(img, 1, None)
    roi, _, _ = IO.resegment_mask_device(x, (msk != 0).to(torch.uint8).contiguous(), kw["resegment"]["resegmentRange"],
                                         "sigma")
    roi_np = roi.cpu().numpy() != 0
    derived = dict(pipeline.derived_images(x, kw["spacing_zyx"], sigmas=kw["sigmas"], image_types=kw["image_types"]))
    assert list(derived) == names
    for name in names:
        ref = FO.extract(derived[name].cpu().numpy(), roi_np, voxelBased=True, spacing_xyz=kw["spacing_zyx"][::-1],
                         kernelRadius=1, binWidth=kw["binWidth"], voxelArrayShift=kw["voxelArrayShift"])
        m = got[(name, "firstorder")].cpu().numpy()
        for k, f in enumerate(FO.NAMES):
            a, r = m[k][roi_np], ref[f]
            scale = max(1.0, float(np.nanmax(np.abs(r))))
            assert np.allclose(a, r, rtol=1e-9, atol=1e-9 * scale, equal_nan=True), (name, f)
            assert (m[k][~roi_np] == 0).all(), (name, f)
    # float32 maps are the float64 maps rounded once
    got32, _ = _run_suite(img, msk, ("firstorder",), map_dtype=torch.float32, **kw)
    for name in names:
        a64 = got[(name, "firstorder")]
        a32 = got32[(name, "firstorder")]
        ref = a64.to(torch.float32)
        assert torch.equal(torch.isnan(a32), torch.isnan(ref))
        assert torch.equal(a32.nan_to_num(0).view(torch.int32), ref.nan_to_num(0).view(torch.int32)), name


def test_suite_one_plane_roi_has_no_z_window_like_the_plugin():
    img, _ = _suite_case()
    img = img.to(torch.float64)
    msk = torch.zeros(img.shape, dtype=torch.uint8, device="cuda")
    msk[5, 3:15, 4:17] = 1
    got, _ = _run_suite(img, msk, ("firstorder",), wavelet=None, sigmas=(), binWidth=25, voxelArrayShift=10)
    plug = FC.RadiomicsFirstOrder(I.ArrayImage(img.cpu().numpy()), I.ArrayImage(msk.cpu().numpy()), voxelBased=True,
                                  kernelRadius=1, binWidth=25, voxelArrayShift=10)
    assert plug._window_radii() == [0, 1, 1]
    res = plug.execute()
    m = got[("original", "firstorder")]
    for k, f in enumerate(FO.NAMES):
        _same_bits(m[k].cpu(), torch.from_numpy(np.ascontiguousarray(I.as_array(res[f]), dtype=np.float64)), f)


def test_suite_rejects_unknown_classes():
    img, msk = _suite_case((5, 6, 7))
    with pytest.raises(ValueError):
        pipeline.voxel_suite_with_filters(img, msk, classes=("firstorder", "shape"), wavelet=None, sigmas=())


def _read_nrrd(path, shape):
    raw = open(path, "rb").read()
    head, data = raw.split(b"\n\n", 1)
    dt = "<f4" if b"\ntype: float\n" in head else "<f8"
    return np.frombuffer(data, dt).reshape(shape).copy()


@pytest.mark.parametrize("out_dtype", [torch.float64, torch.float32])
def test_extract_to_nrrd_writes_the_plugins_firstorder_maps(tmp_path, out_dtype):
    rng = np.random.default_rng(4)
    shape = (10, 12, 14)
    raw = ((rng.integers(1, 20, shape) - 1) * 25 + 3).astype(np.int16)
    msk = (rng.random(shape) < 0.85).astype(np.uint8)
    msk[0] = 0
    spacing_xyz = (0.8, 0.9, 1.5)
    plug = FC.RadiomicsFirstOrder(I.ArrayImage(raw, spacing_xyz), I.ArrayImage(msk, spacing_xyz), voxelBased=True,
                                  kernelRadius=1, binWidth=25, voxelArrayShift=50,
                                  b200_map_dtype="float64" if out_dtype == torch.float64 else "float32").execute()
    d_img = torch.from_numpy(raw).cuda()
    d_msk = torch.from_numpy(msk).cuda()
    _, _, lev, levels, Ng = voxel.discretize(d_img, d_msk, binWidth=25)
    s = _lib.make_settings(Ng, len(levels), kernelRadius=1, spacing_zyx=spacing_xyz[::-1])
    paths = voxel.extract_to_nrrd(lev, s, tmp_path, classes=("firstorder", "ngtdm"), out_dtype=out_dtype, compress=False,
                                  spacing_xyz=spacing_xyz, image=d_img, voxelArrayShift=50)
    assert len(paths) == 18 + 5
    for f in FO.NAMES:
        a = _read_nrrd(paths[f"original_firstorder_{f}"], shape)
        b = np.asarray(I.as_array(plug[f]))
        assert a.dtype == b.dtype and np.array_equal(a.view(np.uint8), np.ascontiguousarray(b).view(np.uint8)), f
    with pytest.raises(ValueError):
        voxel.extract_to_nrrd(lev, s, tmp_path, classes=("firstorder",))
