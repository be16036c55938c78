"""Gray-level discretisation on the GPU against NumPy on the host: the ROI min / max reduction (rb_minmax_dev), the
np.digitize-exact binning (rb_digitize_dev), binImage / getBinEdges / bin_image_device for every NumPy pixel type, the
non-finite and empty-slab ROIs, and the level packing every texture kernel reads (rb_pack_levels_dev).

Volumes of >= 1 M voxels make every thread of the reductions' grids (<= 8 blocks of 256 per SM, ~270 k threads on an
H100) loop at least three times; the special values sit both in the first and in the last grid-stride pass."""
import math

import numpy as np
import pytest
import torch

import pipeline as PL
from pyradiomics_b200 import imageoperations as IO, voxel
from pyradiomics_b200._lib import B200Error, DTYPE_CODE, check, lib, ptr, stream

pytestmark = pytest.mark.gpu
N_BIG = 3 * (1 << 20) + 4099
DEVICE_TYPES = ["int16", "int32", "float32", "float64", "uint8", "uint16", "int64"]


def _upload(a):
    """any rb_dtype array -> its bytes on the device (torch has no full uint16 support; the kernels read the bytes)"""
    return torch.from_numpy(np.ascontiguousarray(a).reshape(-1).view(np.uint8)).cuda()


def _special(dt):
    """the values where min / max / digitize go wrong: type extremes, +-0.0, subnormals, +-inf"""
    if np.issubdtype(dt, np.integer):
        i = np.iinfo(dt)
        return np.array([i.min, i.min + 1, -1 if i.min else 0, 0, 1, i.max - 1, i.max], dt)
    f = np.finfo(dt)
    return np.array([-f.max, -f.tiny, -f.smallest_subnormal, -0.0, 0.0, f.smallest_subnormal, f.tiny, f.max, -np.inf,
                     np.inf], dt)


def _volume(dt, rng, n=N_BIG):
    dt = np.dtype(dt)
    if np.issubdtype(dt, np.integer):
        i = np.iinfo(dt)
        a = rng.integers(max(i.min, -(1 << 40)), min(i.max, 1 << 40), n, endpoint=True).astype(dt)
    else:
        a = (rng.standard_normal(n) * 1e3).astype(dt)
    return a


def _minmax(a, mask):
    keys = torch.tensor([2 ** 63 - 1, -(2 ** 63), 0, 0], dtype=torch.int64, device="cuda")
    m = None if mask is None else _upload(mask.astype(np.uint8))
    d = _upload(a)
    check(lib().rb_minmax_dev(ptr(d), DTYPE_CODE[a.dtype], ptr(m), a.size, ptr(keys), stream()), "minmax")
    k = keys.cpu().tolist()
    return IO._decode_key(k[0]), IO._decode_key(k[1]), k[2], k[3]


def _digitize(a, mask, edges):
    out = torch.full((a.size,), -7, dtype=torch.int32, device="cuda")
    e = torch.from_numpy(np.ascontiguousarray(edges, np.float64)).cuda()
    m = None if mask is None else _upload(mask.astype(np.uint8))
    d = _upload(a)
    check(lib().rb_digitize_dev(ptr(d), DTYPE_CODE[a.dtype], ptr(m), a.size, ptr(e), int(edges.size), ptr(out), stream()),
          "digitize")
    return out.cpu().numpy()


# ------------------------------------------------------------------------------ rb_minmax_dev
@pytest.mark.parametrize("masked", [False, True], ids=["nomask", "mask"])
@pytest.mark.parametrize("dtype", DEVICE_TYPES)
def test_minmax_is_exact_for_every_device_type(dtype, masked):
    rng = np.random.default_rng(DEVICE_TYPES.index(dtype) + 10 * masked)
    dt = np.dtype(dtype)
    a = _volume(dt, rng)
    sp = _special(dt)
    for pos in (0, a.size - 3 * sp.size):                  # first and last grid-stride pass
        a[pos:pos + sp.size] = sp
    mask = rng.random(a.size) < 0.6 if masked else None
    if masked:
        mask[-sp.size:] = False                            # extremes outside the ROI must not count
        a[-sp.size:] = sp[::-1]
        mask[a.size - 3 * sp.size:a.size - 2 * sp.size] = True
    roi = a if mask is None else a[mask]
    mn, mx, cnt, nans = _minmax(a, mask)
    assert cnt == roi.size and nans == 0
    assert mn == roi.min() and mx == roi.max()
    # the ROI without the extremes: every thread's own min / max matter
    if masked:
        mask[:] = False
        mask[1000:a.size - 7:3] = True
        mask[a.size - 8] = True
        a[a.size - 8] = sp[-1] if np.issubdtype(dt, np.integer) else sp[-3]       # the maximum, in the very last pass
        roi = a[mask]
        mn, mx, cnt, _ = _minmax(a, mask)
        assert (mn, mx, cnt) == (roi.min(), roi.max(), roi.size)


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_minmax_counts_nan_and_leaves_it_out_of_min_max(dtype):
    rng = np.random.default_rng(3)
    a = _volume(dtype, rng)
    where = np.array([5, 777, a.size // 2, a.size - 1])
    a[where] = np.nan
    mask = np.ones(a.size, bool)
    mask[where[0]] = False
    mn, mx, cnt, nans = _minmax(a, mask)
    assert (cnt, nans) == (a.size - 1, 3)
    assert mn == np.nanmin(a) and mx == np.nanmax(a)
    mn, mx, cnt, nans = _minmax(a, None)
    assert (cnt, nans) == (a.size, 4)
    z = np.zeros(1000, dtype)
    z[::2] = -0.0
    mn, mx, _, _ = _minmax(z, None)
    assert mn == 0.0 and mx == 0.0                         # -0.0 == 0.0 (which zero is kept is not specified)


def test_minmax_of_an_empty_roi_keeps_the_initial_keys():
    a = np.arange(5000, dtype=np.int16)
    keys = torch.tensor([2 ** 63 - 1, -(2 ** 63), 0, 0], dtype=torch.int64, device="cuda")
    d, m = _upload(a), _upload(np.zeros(a.size, np.uint8))
    check(lib().rb_minmax_dev(ptr(d), DTYPE_CODE[a.dtype], ptr(m), a.size, ptr(keys), stream()), "minmax")
    assert keys.cpu().tolist() == [2 ** 63 - 1, -(2 ** 63), 0, 0]


# ------------------------------------------------------------------------------ rb_digitize_dev
def _edges_and_probes(dt, ne, rng):
    """`ne` increasing float64 edges exactly representable in `dt`, and probe values: every edge, its neighbours one ulp
    (floats) or one unit (integers) to either side, values below the first and above the last edge"""
    dt = np.dtype(dt)
    if np.issubdtype(dt, np.integer):
        i = np.iinfo(dt)
        lo, hi = max(int(i.min) + 2, -(1 << 40)), min(int(i.max) - 2, 1 << 40)
        if ne > hi - lo:
            raise ValueError
        e = np.sort(rng.choice(np.arange(lo, hi + 1) if hi - lo < 1 << 20 else rng.integers(lo, hi, 4 * ne), ne,
                               replace=False)).astype(np.int64)
        probes = np.concatenate([e, e - 1, e + 1, [i.min, i.max]]).astype(dt)
        return e.astype(np.float64), probes
    cand = np.unique((rng.standard_normal(ne * 2 + 16) * 500).astype(dt))
    cand = cand[cand != 0]
    e = np.sort(np.concatenate([[dt.type(0.0)], rng.choice(cand, ne - 1, replace=False)]).astype(dt))   # 0.0: +-0.0 on an edge
    f = np.finfo(dt)
    probes = np.concatenate([e, np.nextafter(e, dt.type(-np.inf)), np.nextafter(e, dt.type(np.inf)),
                             [-f.max, f.max, -np.inf, np.inf, 0.0, -0.0, f.smallest_subnormal, -f.smallest_subnormal]])
    return e.astype(np.float64), probes.astype(dt)


@pytest.mark.parametrize("ne", [1, 2, 4096, 4097])
@pytest.mark.parametrize("dtype", DEVICE_TYPES)
def test_digitize_is_bit_equal_to_numpy_on_and_next_to_every_edge(dtype, ne):
    """ne <= 4096 edges are staged in shared memory, more are searched in global memory"""
    dt = np.dtype(dtype)
    rng = np.random.default_rng(ne + 7 * DEVICE_TYPES.index(dtype))
    if dt == np.uint8 and ne > 250:
        ne = 250                                            # (uint8 has 256 values; 250 distinct edges)
    e, probes = _edges_and_probes(dt, ne, rng)
    a = np.resize(probes, N_BIG)
    a[probes.size:] = rng.permutation(a[probes.size:])
    a[-probes.size:] = probes                               # every probe in the first and in the last pass
    mask = rng.random(a.size) < 0.7
    mask[:probes.size] = True
    mask[-probes.size:] = True
    ref = np.digitize(a.astype(np.float64), e)
    assert np.array_equal(_digitize(a, None, e), ref)
    assert np.array_equal(_digitize(a, mask, e), np.where(mask, ref, 0))


# ------------------------------------------------------------------------------ binImage / getBinEdges / bin_image_device
ALL_TYPES = ["int8", "uint8", "int16", "uint16", "int32", "uint32", "int64", "uint64", "float32", "float64"]
BINNINGS = [dict(binWidth=25), dict(binWidth=3.5), dict(binWidth=0.1), dict(binCount=1), dict(binCount=64)]


def _reference(img, msk, kw):
    """the reference's binImage; integer images in int64 (NumPy 1's promotion: the edges here cannot wrap, DESIGN.md 5)"""
    if np.issubdtype(img.dtype, np.integer):
        img = img.astype(np.int64)
    return PL.bin_image(img, msk, kw.get("binWidth", 25), kw.get("binCount"))[:2]


def _image(dtype, rng, shape=(23, 41, 37), at_limit=False):
    dt = np.dtype(dtype)
    if np.issubdtype(dt, np.integer):
        i = np.iinfo(dt)
        top = min(int(i.max), 1 << 40) if at_limit else min(int(i.max), 900)
        base = max(int(i.min), top - 250)
        img = rng.integers(base, top + 1, shape).astype(dt)
        if at_limit:
            img.flat[:3] = [top, top - 1, base]
    else:
        img = (rng.standard_normal(shape) * 120 + (3.0e4 if at_limit else 300)).astype(dt)
    return img


@pytest.mark.parametrize("at_limit", [False, True], ids=["mid", "limit"])
@pytest.mark.parametrize("kw", BINNINGS, ids=lambda k: "-".join(f"{a}{b}" for a, b in k.items()))
@pytest.mark.parametrize("dtype", ALL_TYPES)
def test_bin_image_matches_numpy_for_every_pixel_type(dtype, kw, at_limit):
    """`limit`: the ROI's maximum within 2 binWidth of the type's largest value (64-bit integers: 2^40, float64's exact
    range for these edges), where the reference's NumPy 2 arithmetic wraps for uint8 / int16"""
    rng = np.random.default_rng(ALL_TYPES.index(dtype) * 31 + at_limit)
    img = _image(dtype, rng, at_limit=at_limit)
    msk = rng.random(img.shape) < 0.55
    msk.flat[:3] = True
    got, edges = IO.binImage(img, msk, **kw)
    ref, redges = _reference(img, msk, kw)
    assert np.array_equal(np.asarray(edges, np.float64), np.asarray(redges, np.float64))
    assert np.array_equal(got, ref)
    assert got[msk].min() >= 1 and (got[~msk] == 0).all()
    assert np.array_equal(np.asarray(IO.getBinEdges(img[msk], **kw), np.float64), np.asarray(redges, np.float64))
    # the device-tensor entry, no mask: the whole volume is the ROI
    t = IO._to_device(img)
    lev, e2 = IO.bin_image_device(t, None, **kw)
    ref2, redges2 = _reference(img, np.ones(img.shape, bool), kw)
    assert np.array_equal(np.asarray(e2, np.float64), np.asarray(redges2, np.float64))
    assert np.array_equal(lev.cpu().numpy(), ref2)


@pytest.mark.parametrize("kw", [dict(binWidth=25), dict(binCount=64)], ids=["binWidth", "binCount"])
def test_bin_image_on_a_volume_where_every_thread_loops(kw):
    rng = np.random.default_rng(5)
    img = (rng.standard_normal((96, 128, 112)) * 300).astype(np.float32)
    msk = rng.random(img.shape) < 0.8
    img.flat[-1] = 5000.0                                   # the maximum in the last grid-stride pass
    msk.flat[-1] = True
    got, edges = IO.binImage(img, msk, **kw)
    ref, redges = _reference(img, msk, kw)
    assert np.array_equal(np.asarray(edges, np.float64), np.asarray(redges, np.float64))
    assert np.array_equal(got, ref)


# ------------------------------------------------------------------------------ non-finite ROIs, empty slabs
@pytest.mark.parametrize("kw", [dict(binWidth=25), dict(binWidth=0.1), dict(binCount=1), dict(binCount=64)],
                         ids=["bw25", "bw0.1", "bc1", "bc64"])
@pytest.mark.parametrize("bad", ["nan", "inf", "-inf"])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_non_finite_roi_raises_value_error_like_the_reference(dtype, bad, kw):
    rng = np.random.default_rng(8)
    img = (rng.standard_normal((10, 12, 14)) * 100).astype(dtype)
    msk = np.ones(img.shape, bool)
    msk[0] = False
    img[4, 5, 6] = float(bad)
    with pytest.raises(ValueError), np.errstate(invalid="ignore", over="ignore"):
        PL.bin_image(img, msk, kw.get("binWidth", 25), kw.get("binCount"))
    with pytest.raises(ValueError):
        IO.binImage(img, msk, **kw)
    with pytest.raises(ValueError):
        IO.getBinEdges(img[msk], **kw)
    # outside the ROI it is just another voxel
    img[0, 1, 2] = img[4, 5, 6]
    img[4, 5, 6] = 0
    got, edges = IO.binImage(img, msk, **kw)
    ref, redges = _reference(img, msk, kw)
    assert np.array_equal(np.asarray(edges, np.float64), redges) and np.array_equal(got, ref)


def test_first_order_class_refuses_a_nan_roi():
    from pyradiomics_b200 import featureclasses as FC
    img = np.random.default_rng(1).normal(100, 20, (6, 7, 8))
    img[3, 3, 3] = np.nan
    msk = np.ones(img.shape, np.uint8)
    with pytest.raises(ValueError):
        FC.RadiomicsFirstOrder(img, msk, voxelBased=True, binWidth=25).execute()


def test_slab_binning_with_a_reducer_on_one_gpu():
    """the multi-GPU slab path calls bin_image_device per z-slab with an all-reduce of (min, max): here two slabs of one
    volume on one GPU, the reducer a callable that combines them.  A slab without ROI voxels bins to zeros with the whole
    ROI's edges; together the slabs equal binning the whole volume"""
    rng = np.random.default_rng(6)
    img = (rng.standard_normal((20, 16, 18)) * 200).astype(np.float32)
    msk = np.zeros(img.shape, np.uint8)
    msk[11:18, 3:12, 2:15] = rng.random((7, 9, 13)) < 0.8            # the ROI lies in the second slab only
    t, m = torch.as_tensor(img).cuda(), torch.as_tensor(msk).cuda()
    slabs = [(t[:10].contiguous(), m[:10].contiguous()), (t[10:].contiguous(), m[10:].contiguous())]
    ext = [IO.roi_extent(a, b) for a, b in slabs]
    assert ext[0][:3] == (math.inf, -math.inf, 0)
    seen = []

    def reduce_minmax(mn, mx):
        seen.append((mn, mx))
        return min(mn, *(e[0] for e in ext)), max(mx, *(e[1] for e in ext))

    outs = [IO.bin_image_device(a, b, minmax_reduce=reduce_minmax, binWidth=25) for a, b in slabs]
    assert seen[0] == (math.inf, -math.inf)
    ref, redges = PL.bin_image(img, msk.astype(bool), 25)[:2]
    for lev, edges in outs:
        assert np.array_equal(np.asarray(edges, np.float64), redges)
    assert (outs[0][0].cpu().numpy() == 0).all()
    assert np.array_equal(np.concatenate([o[0].cpu().numpy() for o in outs]), ref)
    with pytest.raises(ValueError, match="empty ROI"):               # empty after the reduction too
        IO.bin_image_device(*slabs[0], minmax_reduce=lambda mn, mx: (mn, mx), binWidth=25)
    # a NaN in one slab: that slab hands (-inf, +inf) to the reduction, so every slab refuses the range
    bad = slabs[1][0].clone()
    bad[3, 5, 5] = float("nan")
    m1 = slabs[1][1].clone()
    m1[3, 5, 5] = 1
    seen.clear()
    with pytest.raises(ValueError):
        IO.bin_image_device(bad, m1, minmax_reduce=reduce_minmax, binWidth=25)
    assert seen == [(-math.inf, math.inf)]
    with pytest.raises(ValueError):
        IO.bin_image_device(*slabs[0], minmax_reduce=lambda mn, mx: (-math.inf, math.inf), binWidth=25)


# ------------------------------------------------------------------------------ rb_pack_levels_dev
@pytest.mark.parametrize("Ng", [1, 255, 256, 65535])
def test_pack_levels_keeps_the_levels_and_counts_them(Ng):
    rng = np.random.default_rng(Ng)
    shape = (33, 160, 200)                                  # 1.06 M voxels: grid_for(n, 256, 16) threads loop
    lev = rng.integers(1, Ng + 1, shape).astype(np.int32)
    lev.flat[-1] = Ng
    lev.flat[0] = 1
    msk = rng.random(shape) < 0.75
    msk.flat[0] = msk.flat[-1] = True
    junk = rng.integers(-5, Ng + 7, shape).astype(np.int32)
    img = np.where(msk, lev, junk)                          # anything outside the mask is ignored
    packed, presence = voxel.pack_levels(torch.as_tensor(img).cuda(), torch.as_tensor(msk.astype(np.uint8)).cuda(), Ng)
    assert packed.dtype == (torch.uint8 if Ng <= 255 else torch.int16)
    got = packed.cpu().numpy()
    got = got.view(np.uint16) if Ng > 255 else got
    assert np.array_equal(got, np.where(msk, lev, 0))
    assert np.array_equal(presence.cpu().numpy(), np.bincount(lev[msk], minlength=Ng + 1)[1:])


@pytest.mark.parametrize("Ng", [1, 255, 256, 65535])
def test_pack_levels_status_bit_marks_a_masked_level_outside_1_to_Ng(Ng):
    rng = np.random.default_rng(Ng + 1)
    n = (1 << 20) + 301
    msk = (rng.random(n) < 0.5).astype(np.uint8)
    lev = rng.integers(1, Ng + 1, n).astype(np.int32)
    where = np.flatnonzero(msk == 0)
    lev[where[:3]] = [0, Ng + 1, -1]                        # out of range but outside the mask: fine

    def status(levels):
        out = torch.empty(n, dtype=torch.uint8 if Ng <= 255 else torch.int16, device="cuda")
        st = torch.zeros(1, dtype=torch.int32, device="cuda")
        d_lev, d_msk = torch.as_tensor(levels).cuda(), torch.as_tensor(msk).cuda()     # alive until the kernel has run
        check(lib().rb_pack_levels_dev(ptr(d_lev), ptr(d_msk), n, Ng, ptr(out), None, ptr(st), stream()), "pack_levels")
        return int(st.item())

    assert status(lev) == 0
    for bad in (0, Ng + 1, -1, 1 << 20):
        for pos in (np.flatnonzero(msk)[0], np.flatnonzero(msk)[-1]):    # first and last grid-stride pass
            b = lev.copy()
            b[pos] = bad
            assert status(b) == 1, (bad, pos)
            with pytest.raises(IndexError):
                voxel.pack_levels(torch.as_tensor(b).cuda(), torch.as_tensor(msk).cuda(), Ng)


@pytest.mark.parametrize("Ng", [0, -1, 65536])
def test_pack_levels_refuses_ng_outside_1_to_65535(Ng):
    img = torch.ones(64, dtype=torch.int32, device="cuda")
    msk = torch.ones(64, dtype=torch.uint8, device="cuda")
    out = torch.empty(64, dtype=torch.int16, device="cuda")
    with pytest.raises(B200Error, match="outside 1..65535"):
        check(lib().rb_pack_levels_dev(ptr(img), ptr(msk), 64, Ng, ptr(out), None, None, stream()), "pack_levels")
