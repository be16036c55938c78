"""GPU versions of the pyradiomics image operations that sit on the texture hot path
(reference radiomics/imageoperations.py): gray-level discretisation (getBinEdges / binImage,
:67-174), the level-1 stationary wavelet decomposition (getWaveletImage / _swt3, :839-970) and the
Laplacian-of-Gaussian filter (getLoGImage, :756-836).  Same function names, arguments and yielded
tuples as the reference so they can be dropped into ``radiomics.imageoperations``.

Parity status (DESIGN.md): binning is bit-identical to NumPy; wavelet and LoG restate PyWavelets'
and ITK's published algorithms -- neither library is available offline and the reference's own
tests do not pin them (SURVEY.md section 8c) -> "parity unpinned" for those two.
"""
from __future__ import annotations

import ctypes as C
import logging
import math

import numpy as np
import torch

from . import image as I
from ._lib import check, lib

logger = logging.getLogger("radiomics.imageoperations")

_DT = {np.dtype("int16"): 0, np.dtype("int32"): 1, np.dtype("float32"): 2, np.dtype("float64"): 3,
       np.dtype("uint8"): 4, np.dtype("uint16"): 5, np.dtype("int64"): 6}
_TORCH_DT = {torch.int16: 0, torch.int32: 1, torch.float32: 2, torch.float64: 3, torch.uint8: 4, torch.int64: 6}


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dev():
    return torch.device("cuda", torch.cuda.current_device())


_TORCH_OF_NP = {np.int16: torch.int16, np.int32: torch.int32, np.float32: torch.float32, np.float64: torch.float64,
                np.uint8: torch.uint8, np.int64: torch.int64}
_STAGE = {"bufs": None, "pool": None}
_STAGE_CHUNK = 32 << 20
_STAGE_MIN = 64 << 20


def _upload_staged(a):
    """pageable NumPy array -> CUDA tensor through two page-locked 32 MB staging blocks: a few threads copy chunk k+1 into
    one block (NumPy releases the GIL) while the DMA engine drains chunk k from the other.  A plain ``tensor.to(device)`` of
    pageable memory lets the driver stage it single-threaded, at a fraction of the link's rate."""
    import concurrent.futures as cf
    flat = a.reshape(-1).view(np.uint8)
    n = flat.size
    dev = _dev()
    out = torch.empty(n, dtype=torch.uint8, device=dev)
    if _STAGE["bufs"] is None:
        _STAGE["bufs"] = [torch.empty(_STAGE_CHUNK, dtype=torch.uint8, pin_memory=True) for _ in range(2)]
        _STAGE["pool"] = cf.ThreadPoolExecutor(max_workers=4)
    bufs, pool = _STAGE["bufs"], _STAGE["pool"]
    views = [b.numpy() for b in bufs]
    done = [None, None]
    stream = torch.cuda.current_stream()
    for k, off in enumerate(range(0, n, _STAGE_CHUNK)):
        m = min(_STAGE_CHUNK, n - off)
        j = k & 1
        if done[j] is not None:
            done[j].synchronize()                   # the DMA out of this block has finished
        q = (m + 3) // 4
        list(pool.map(lambda s: np.copyto(views[j][s:min(s + q, m)], flat[off + s:off + min(s + q, m)]), range(0, m, q)))
        out[off:off + m].copy_(bufs[j][:m], non_blocking=True)
        done[j] = torch.cuda.Event()
        done[j].record(stream)
    for e in done:
        if e is not None:
            e.synchronize()                         # the staging blocks are reused by the next upload
    return out.view(_TORCH_OF_NP[a.dtype.type]).reshape(a.shape)


def _to_device(arr):
    """NumPy / torch -> contiguous CUDA tensor of a supported dtype (uint16 travels as int32)."""
    if isinstance(arr, torch.Tensor):
        t = arr
        if t.dtype == torch.bool:
            t = t.to(torch.uint8)
        if t.dtype not in _TORCH_DT:
            t = t.to(torch.float64)
        return t.to(_dev()).contiguous()
    a = np.asarray(arr)
    if a.dtype == np.bool_:
        a = a.view(np.uint8)
    elif a.dtype == np.uint16:
        a = a.astype(np.int32)
    elif a.dtype not in _DT:
        a = a.astype(np.float64)
    a = np.ascontiguousarray(a)
    if a.nbytes >= _STAGE_MIN and a.dtype.type in _TORCH_OF_NP:
        return _upload_staged(a)
    return torch.from_numpy(a).to(_dev())


def _decode_key(k: int) -> float:
    bits = k if k >= 0 else k ^ 0x7FFFFFFFFFFFFFFF
    return float(np.array([bits], dtype=np.int64).view(np.float64)[0])


def roi_minmax(img_t: torch.Tensor, mask_t: torch.Tensor | None):
    """(min, max, count) of the ROI, one streaming kernel (replaces builtin min()/max())."""
    keys = torch.tensor([2 ** 63 - 1, -(2 ** 63), 0], dtype=torch.int64, device=img_t.device)
    check(lib().rb_minmax_dev(_ptr(img_t), _TORCH_DT[img_t.dtype], _ptr(mask_t), C.c_longlong(img_t.numel()), _ptr(keys),
                              _stream()), "minmax")
    k = keys.cpu().tolist()
    if k[2] == 0:
        raise ValueError("empty ROI")
    return _decode_key(k[0]), _decode_key(k[1]), k[2]


_NP_OF_TORCH = {torch.int16: np.int16, torch.int32: np.int32, torch.float32: np.float32, torch.float64: np.float64,
                torch.uint8: np.uint8, torch.int64: np.int64}


def _edges_from_minmax(minimum, maximum, np_type, **kwargs):
    """reference getBinEdges arithmetic (imageoperations.py:119-149) on the scalars min / max, carried
    out in the image's own NumPy scalar type so that float32 / integer inputs round exactly as
    `min(values) - (min(values) % binWidth)`, np.arange and np.histogram do in the reference."""
    binWidth = kwargs.get("binWidth", 25)
    binCount = kwargs.get("binCount")
    minimum, maximum = np_type(minimum), np_type(maximum)
    if binCount is not None:
        # np.histogram(values, binCount)[1]: linspace(min, max, binCount + 1) in the result type of
        # the data (float64 for integers), degenerate range widened by +-0.5; then last edge + 1
        et = np.dtype(np.float64) if np.issubdtype(np_type, np.integer) else np.dtype(np_type)
        lo, hi = et.type(minimum), et.type(maximum)
        if lo == hi:
            lo, hi = lo - et.type(0.5), hi + et.type(0.5)
        e = np.linspace(lo, hi, int(binCount) + 1, endpoint=True, dtype=et)
        e[-1] += 1
        return e
    lowBound = minimum - (minimum % binWidth)
    highBound = maximum + 2 * binWidth
    e = np.arange(lowBound, highBound, binWidth)
    if len(e) == 1:
        e = np.array([e[0] - 0.5, e[0] + 0.5])
    return e


def getBinEdges(parameterValues, **kwargs):
    """reference signature: 1-D array of the segmented voxel values -> bin edges."""
    t = _to_device(parameterValues).reshape(-1)
    mn, mx, _ = roi_minmax(t, None)
    return _edges_from_minmax(mn, mx, _NP_OF_TORCH[t.dtype], **kwargs)


def bin_image_device(img_t: torch.Tensor, mask_t: torch.Tensor | None, minmax_reduce=None, **kwargs):
    """device tensors in -> (int32 levels tensor (0 outside the mask), edges ndarray).  `minmax_reduce(mn, mx)` turns a
    slab's ROI minimum / maximum into the whole ROI's (multi-GPU: all-reduce MIN / MAX), so every rank bins with the
    same edges."""
    mn, mx, _ = roi_minmax(img_t, mask_t)
    if minmax_reduce is not None:
        mn, mx = minmax_reduce(mn, mx)
    edges_native = _edges_from_minmax(mn, mx, _NP_OF_TORCH[img_t.dtype], **kwargs)
    edges = np.ascontiguousarray(edges_native, dtype=np.float64)
    e_t = torch.from_numpy(edges).to(img_t.device)
    out = torch.empty(img_t.shape, dtype=torch.int32, device=img_t.device)
    check(lib().rb_digitize_dev(_ptr(img_t), _TORCH_DT[img_t.dtype], _ptr(mask_t), C.c_longlong(img_t.numel()), _ptr(e_t),
                                int(edges.size), _ptr(out), _stream()), "digitize")
    return out, edges_native


def binImage(parameterMatrix, parameterMatrixCoordinates=None, **kwargs):
    """reference signature (imageoperations.py:156): returns (discretised int array, binEdges).
    `parameterMatrixCoordinates` is the boolean ROI mask the feature classes pass."""
    img_t = _to_device(parameterMatrix)
    mask_t = None
    if parameterMatrixCoordinates is not None:
        m = np.asarray(parameterMatrixCoordinates)
        if m.dtype != np.bool_ or m.shape != tuple(img_t.shape):
            mm = np.zeros(tuple(img_t.shape), dtype=bool)
            mm[parameterMatrixCoordinates] = True
            m = mm
        mask_t = _to_device(m)
    out, edges = bin_image_device(img_t, mask_t, **kwargs)
    return out.cpu().numpy().astype(np.int64), edges


# ------------------------------------------------------------------------------------ cropping
def cropToTumorMask(imageNode, maskNode, boundingBox, **kwargs):
    """reference signature (imageoperations.py:407-445): crop image and mask to the ROI's bounding box
    `boundingBox` = (x_lo, x_hi, y_lo, y_hi, z_lo, z_hi) (inclusive, SimpleITK x,y,z order, as checkMask returns it),
    grown by kwargs['padDistance'] voxels on every side and clipped to the image (the orchestrator passes
    padDistance = kernelRadius in voxel-based mode, 0 otherwise: featureextractor.py:304-307,385-387).  Host-side
    slicing (views, no copy): the crop decides which voxels ever reach the GPU."""
    padDistance = int(kwargs.get("padDistance", 0))
    bb = np.asarray(boundingBox, dtype=np.int64)
    size = np.array(I.size_xyz(maskNode), dtype=np.int64)
    nd = size.size
    lo = np.maximum(bb[0::2][:nd] - padDistance, 0)
    hi = np.minimum(bb[1::2][:nd] + padDistance, size - 1)
    logger.debug("Cropping to size %s", (bb[1::2][:nd] - bb[0::2][:nd]) + 1)
    sl = tuple(slice(int(lo[d]), int(hi[d]) + 1) for d in range(nd))[::-1]          # arrays are (z,y,x)
    return I.like(imageNode, I.as_array(imageNode)[sl]), I.like(maskNode, I.as_array(maskNode)[sl])


# ------------------------------------------------------------------------------------ resampling
_INTERPOLATORS = {"sitkNearestNeighbor": 0, "sitkLinear": 1, "sitkBSpline": 3, 1: 0, 2: 1, 3: 3}      # (sitk enum values 1, 2, 3)
_NP_DT = {np.dtype("int16"): 0, np.dtype("int32"): 1, np.dtype("float32"): 2, np.dtype("float64"): 3, np.dtype("uint8"): 4,
          np.dtype("int64"): 6}


def resample_device(arr_t: torch.Tensor, out_size_zyx, start_zyx, step_zyx, interpolator=3, default_value=0.0, out_dtype=None):
    """CUDA tensor (Z,Y,X) -> CUDA tensor of `out_size_zyx` sampled at input continuous indices start + k * step
    (rb_bspline_prefilter_dev + rb_resample_dev); cubic B-spline (3), linear (1) or nearest neighbour (0); the result is
    clamped and truncated to `out_dtype` (default: the input's) like ITK's ResampleImageFilter"""
    src = arr_t.contiguous()
    out_dtype = out_dtype or src.dtype
    if out_dtype not in _TORCH_DT:
        raise ValueError(f"unsupported pixel type {out_dtype}")
    Z, Y, X = src.shape
    dst = torch.empty(tuple(int(v) for v in out_size_zyx), dtype=out_dtype, device=src.device)
    if interpolator == 3:
        src = src.to(torch.float64).clone()
        check(lib().rb_bspline_prefilter_dev(_ptr(src), Z, Y, X, _stream()), "bspline prefilter")
    elif src.dtype not in _TORCH_DT:
        src = src.to(torch.float64)
    isz = (C.c_int * 3)(Z, Y, X)
    osz = (C.c_int * 3)(*[int(v) for v in out_size_zyx])
    st = (C.c_double * 3)(*[float(v) for v in start_zyx])
    sp = (C.c_double * 3)(*[float(v) for v in step_zyx])
    check(lib().rb_resample_dev(_ptr(src), _TORCH_DT[src.dtype], isz, _ptr(dst), _TORCH_DT[out_dtype], osz, st, sp, int(interpolator),
                                C.c_double(float(default_value)), _stream()), "resample")
    return dst


def resampleImage(imageNode, maskNode, **kwargs):
    """reference signature (radiomics/imageoperations.py:448-612): resample image (B-spline by default) and mask (nearest
    neighbour) to `resampledPixelSpacing`, cropped to the ROI's bounding box grown by `padDistance` new-grid voxels; the
    grid is aligned to the input origin.  The geometry arithmetic is the reference's (:509-566); image and mask are taken
    to share one axis-aligned grid (the array stand-in of SimpleITK images carries spacing and origin, no direction
    cosines).  Interpolation and cast happen on the GPU (resample_device)."""
    resampledPixelSpacing = kwargs["resampledPixelSpacing"]
    interpolator = kwargs.get("interpolator", "sitkBSpline")
    padDistance = kwargs.get("padDistance", 5)
    label = int(kwargs.get("label", 1))
    if imageNode is None or maskNode is None:
        raise ValueError("Requires both image and mask to resample")
    img, msk = I.as_array(imageNode), I.as_array(maskNode)
    if img.shape != msk.shape:
        raise ValueError("image and mask must share one grid")
    nd = msk.ndim
    maskSpacing = np.array(I.spacing_xyz(maskNode), dtype=np.float64)
    assert len(resampledPixelSpacing) == nd, f"Wrong dimensionality ({len(resampledPixelSpacing)}-D) of resampledPixelSpacing!, {nd}-D required"
    newSp = np.array(resampledPixelSpacing, dtype=np.float64)
    newSp = np.where(newSp == 0, maskSpacing, newSp)
    # bounding box (lower bounds then sizes, x,y,z) of the label: what LabelShapeStatisticsImageFilter gives _checkROI (:346-404)
    idx = np.array(np.where(msk == label))
    if idx.shape[1] == 0:
        raise ValueError(f"Label ({label}) not present in mask")
    lo, hi = idx.min(1)[::-1], idx.max(1)[::-1]
    bb = np.concatenate([lo, hi - lo + 1]).astype(np.float64)
    maskSize = np.array(msk.shape[::-1], dtype=np.float64)
    newSp = np.where(bb[nd:] != 1, newSp, maskSpacing)                  # no resampling across a single-slice ROI (:509-511)
    if np.allclose(maskSpacing, newSp):                                  # nothing to interpolate: crop only (:517-537)
        low_up = np.empty(nd * 2, dtype=int)
        low_up[::2], low_up[1::2] = lo, hi
        return cropToTumorMask(imageNode, maskNode, low_up, **kwargs)
    ratio = maskSpacing / newSp
    L = np.floor((bb[:nd] - 0.5) * ratio - padDistance)
    U = np.ceil((bb[:nd] + bb[nd:] - 0.5) * ratio + padDistance)
    maxU = np.ceil(maskSize * ratio) - 1
    L = np.where(L < 0, 0, L)
    U = np.where(U > maxU, maxU, U)
    newSize = np.array(U - L + 1, dtype=int)
    start = 0.5 * (newSp - maskSpacing) / maskSpacing + L / ratio       # continuous index of output voxel 0 (:549-556)
    step = newSp / maskSpacing
    if isinstance(interpolator, str) and interpolator not in _INTERPOLATORS:
        logger.warning('interpolator "%s" not recognized, using sitkBSpline', interpolator)
        interpolator = "sitkBSpline"
    if interpolator not in _INTERPOLATORS:
        raise ValueError(f"interpolator {interpolator!r} is not implemented (sitkBSpline, sitkLinear, sitkNearestNeighbor)")
    logger.info("Applying resampling from spacing %s and size %s to spacing %s and size %s", maskSpacing, maskSize, newSp, newSize)
    pad3 = (1,) * (3 - nd)
    img_t = _to_device(img).reshape(pad3 + img.shape)
    msk_t = _to_device(msk).reshape(pad3 + msk.shape)
    osz = pad3 + tuple(int(v) for v in newSize[::-1])
    st3 = (0.0,) * (3 - nd) + tuple(start[::-1])
    sp3 = (1.0,) * (3 - nd) + tuple(step[::-1])
    out_img = resample_device(img_t, osz, st3, sp3, _INTERPOLATORS[interpolator])
    out_msk = resample_device(msk_t, osz, st3, sp3, 0)
    origin = np.array(I.origin_xyz(maskNode), dtype=np.float64) + start * maskSpacing      # TransformContinuousIndexToPhysicalPoint (:557)
    a_img = out_img.cpu().numpy().reshape(osz[3 - nd:]).astype(img.dtype, copy=False)
    a_msk = out_msk.cpu().numpy().reshape(osz[3 - nd:]).astype(msk.dtype if msk.dtype != np.bool_ else np.uint8, copy=False)
    return I.ArrayImage(a_img, tuple(newSp), tuple(origin)), I.ArrayImage(a_msk, tuple(newSp), tuple(origin))


# ------------------------------------------------------------------------------------ wavelet
# decomposition low-pass filters (PyWavelets conventions); dec_hi[k] = (-1)^(k+1) dec_lo[F-1-k]
_DEC_LO = {
    "haar": [0.7071067811865476, 0.7071067811865476],
    "db1": [0.7071067811865476, 0.7071067811865476],
    "db2": [-0.12940952255126037, 0.2241438680420134, 0.8365163037378079, 0.48296291314453416],
    "sym2": [-0.12940952255126037, 0.2241438680420134, 0.8365163037378079, 0.48296291314453416],
    "coif1": [-0.01565572813546454, -0.0727326195128539, 0.38486484686420286, 0.8525720202122554,
              0.3378976624578092, -0.0727326195128539],
}


def wavelet_filters(name):
    if not isinstance(name, str):          # a pywt.Wavelet-like object
        return np.asarray(name.dec_lo, float), np.asarray(name.dec_hi, float)
    if name not in _DEC_LO:
        raise ValueError(f"wavelet '{name}' is not in the built-in table {sorted(_DEC_LO)}; pass an object with dec_lo/dec_hi")
    lo = np.asarray(_DEC_LO[name], float)
    F = lo.size
    hi = np.array([(-1) ** (k + 1) * lo[F - 1 - k] for k in range(F)])
    return lo, hi


def swt_level1_device(x: torch.Tensor, axes, lo, hi, z_range=None):
    """one undecimated level over `axes` (in that order) of a float64 CUDA volume (Z,Y,X), periodic extension:
    {'aad': tensor, ...} with one letter per axis in `axes` order, like pywt.swtn.  Three axes with a 2/4/6/8-tap
    filter take the fused single-pass kernel (rb_swt3d_dev); anything else runs one axis per pass."""
    Z, Y, X = x.shape
    lo = np.ascontiguousarray(lo, dtype=np.float64)
    hi = np.ascontiguousarray(hi, dtype=np.float64)
    axes = [int(a) for a in axes]
    if sorted(axes) == [0, 1, 2] and lo.size in (2, 4, 6, 8):
        x = x.contiguous()
        zb, ze = (0, Z) if z_range is None else (int(z_range[0]), int(z_range[1]))      # slab + halo in, interior planes out
        out = torch.empty((8, ze - zb, Y, X), dtype=torch.float64, device=x.device)
        check(lib().rb_swt3d_dev(_ptr(x), Z, Y, X, lo.ctypes.data_as(C.c_void_p), hi.ctypes.data_as(C.c_void_p), int(lo.size),
                                 _ptr(out), C.c_longlong(out.stride(0)), zb, ze, _stream()), "swt3d")
        res = {}
        for b in range(8):
            band = {2: b & 1, 1: b >> 1 & 1, 0: b >> 2 & 1}          # axis (0 = z, 1 = y, 2 = x) -> high-pass?
            res["".join("d" if band[a] else "a" for a in axes)] = out[b]
        return res
    if z_range is not None:
        raise ValueError("z_range needs the fused 3-D kernel (three axes, 2/4/6/8 taps)")
    cur = {"": x}
    for ax in axes:
        nxt = {}
        for key, t in cur.items():
            a = torch.empty_like(t)
            d = torch.empty_like(t)
            check(lib().rb_swt_axis_dev(_ptr(t), Z, Y, X, int(ax), lo.ctypes.data_as(C.c_void_p), hi.ctypes.data_as(C.c_void_p),
                                        int(lo.size), _ptr(a), _ptr(d), _stream()), "swt")
            nxt[key + "a"], nxt[key + "d"] = a, d
        cur = nxt
    return cur


def _wrap_pad_even(data: torch.Tensor, axes3):
    """reference imageoperations.py:914-919: every transformed axis of odd length gets ONE wrap-around sample appended;
    returns the padded tensor and the crop slices that undo it (:947-951, :961-963)"""
    crop = [slice(None)] * 3
    for ax in axes3:
        if data.shape[ax] % 2:
            crop[ax] = slice(0, data.shape[ax])
            data = torch.cat([data, data.narrow(ax, 0, 1)], dim=ax)
    return data.contiguous(), tuple(crop)


def _swt3(inputImage, axes, **kwargs):
    """reference _swt3 (imageoperations.py:899-970): pad ONCE, keep the padded approximation between the levels (each
    level is a level-1 transform of the previous approximation), crop only what is handed out"""
    wavelet = kwargs.get("wavelet", "coif1")
    level = kwargs.get("level", 1)
    start_level = kwargs.get("start_level", 0)
    lo, hi = wavelet_filters(wavelet)
    arr = I.as_array(inputImage)
    nd = arr.ndim
    data = _to_device(arr).to(torch.float64)
    if nd == 2:
        data = data[None]
    ax3 = [a + (3 - nd) for a in axes]
    data, crop = _wrap_pad_even(data, ax3)
    key_a = "a" * len(axes)
    for _ in range(start_level):
        data = swt_level1_device(data, ax3, lo, hi)[key_a]
    ret = []
    for _ in range(start_level, start_level + level):
        dec = swt_level1_device(data, ax3, lo, hi)
        data = dec[key_a]
        dec_im = {}
        for name, t in dec.items():
            if name == key_a:
                continue
            a = t[crop].cpu().numpy()
            dec_im[name.replace("a", "L").replace("d", "H")] = I.like(inputImage, a[0] if nd == 2 else a)
        ret.append(dec_im)
    a = data[crop].cpu().numpy()
    return I.like(inputImage, a[0] if nd == 2 else a), ret


def getWaveletImage(inputImage, _inputMask, **kwargs):
    """reference generator (imageoperations.py:839-896): yields (image, name, kwargs)."""
    Nd = I.as_array(inputImage).ndim
    axes = list(range(Nd - 1, -1, -1))
    if kwargs.get("force2D", False):
        axes.remove(kwargs.get("force2Ddimension", 0))
    approx, ret = _swt3(inputImage, tuple(axes), **kwargs)
    for idx, wl in enumerate(ret, start=1):
        for decompositionName, decompositionImage in wl.items():
            name = f"wavelet-{decompositionName}" if idx == 1 else f"wavelet{idx}-{decompositionName}"
            yield decompositionImage, name, kwargs
    name = f"wavelet-{'L' * len(axes)}" if len(ret) == 1 else f"wavelet{len(ret)}-{'L' * len(axes)}"
    yield approx, name, kwargs


# ------------------------------------------------------------------------------------ LoG
def recursive_gaussian_coefficients(sigmad: float, order: int, scale_norm: float = 1.0):
    """Deriche-type 4th-order recursive Gaussian (Farneback-Westin parameterisation) as used by ITK's
    RecursiveGaussianImageFilter: returns the 20 coefficients N0..3, D1..4, M1..4, BN1..4, BM1..4 for
    smoothing (order 0) or the second derivative (order 2), sigma in voxels."""
    A1 = (1.3530, -0.6724, -1.3563); B1 = (1.8151, -3.4327, 5.2318); W1 = 0.6681; L1 = -1.3932
    A2 = (-0.3531, 0.6724, 0.3446); B2 = (0.0902, 0.6100, -2.2355); W2 = 2.0787; L2 = -1.3732
    s1, s2 = math.sin(W1 / sigmad), math.sin(W2 / sigmad)
    c1, c2 = math.cos(W1 / sigmad), math.cos(W2 / sigmad)
    e1, e2 = math.exp(L1 / sigmad), math.exp(L2 / sigmad)
    D4 = e1 * e1 * e2 * e2
    D3 = -2 * c1 * e1 * e2 * e2 - 2 * c2 * e2 * e1 * e1
    D2 = 4 * c2 * c1 * e1 * e2 + e1 * e1 + e2 * e2
    D1 = -2 * (e2 * c2 + e1 * c1)
    SD = 1 + D1 + D2 + D3 + D4
    DD = D1 + 2 * D2 + 3 * D3 + 4 * D4
    ED = D1 + 4 * D2 + 9 * D3 + 16 * D4

    def ncoef(a1, b1, a2, b2):
        N0 = a1 + a2
        N1 = e2 * (b2 * s2 - (a2 + 2 * a1) * c2) + e1 * (b1 * s1 - (a1 + 2 * a2) * c1)
        N2 = 2 * e1 * e2 * ((a1 + a2) * c2 * c1 - b1 * c2 * s1 - b2 * c1 * s2) + a2 * e1 * e1 + a1 * e2 * e2
        N3 = e2 * e1 * e1 * (b2 * s2 - a2 * c2) + e1 * e2 * e2 * (b1 * s1 - a1 * c1)
        N = np.array([N0, N1, N2, N3])
        return N, N.sum(), N1 + 2 * N2 + 3 * N3, N1 + 4 * N2 + 9 * N3

    if order == 0:
        N, SN, _, _ = ncoef(A1[0], B1[0], A2[0], B2[0])
        alpha0 = 2 * SN / SD - N[0]
        N = N * (scale_norm / alpha0)
    elif order == 2:
        N0s, SN0, DN0, EN0 = ncoef(A1[0], B1[0], A2[0], B2[0])
        N2s, SN2, DN2, EN2 = ncoef(A1[2], B1[2], A2[2], B2[2])
        beta = -(2 * SN2 - SD * N2s[0]) / (2 * SN0 - SD * N0s[0])
        N = N2s + beta * N0s
        SN, DN, EN = SN2 + beta * SN0, DN2 + beta * DN0, EN2 + beta * EN0
        alpha2 = (EN * SD * SD - ED * SN * SD - 2 * DN * DD * SD + 2 * DD * DD * SN) / (SD * SD * SD)
        N = N * (scale_norm / alpha2)
    else:
        raise ValueError("order must be 0 or 2")
    D = np.array([D1, D2, D3, D4])
    M = np.array([N[1] - D1 * N[0], N[2] - D2 * N[0], N[3] - D3 * N[0], -D4 * N[0]])   # symmetric kernel
    SNn, SM = N.sum(), M.sum()
    BN = D * SNn / SD
    BM = D * SM / SD
    return np.concatenate([N, D, M, BN, BM]).astype(np.float64)


def _rg_pass(src: torch.Tensor, axis: int, sigma_vox: float, order: int, out: torch.Tensor | None = None, scale: float = 1.0,
             accumulate: bool = False):
    """one recursive-Gaussian axis pass (order 0 = smoothing, 2 = second derivative) of a float32 / float64 CUDA volume
    into a float32 volume"""
    Z, Y, X = src.shape
    if out is None:
        out = torch.empty((Z, Y, X), dtype=torch.float32, device=src.device)
    scratch = torch.empty((Z, Y, X), dtype=torch.float64, device=src.device)
    coef = recursive_gaussian_coefficients(sigma_vox, order)
    check(lib().rb_recursive_gaussian_axis_dev(_ptr(src), int(src.dtype == torch.float32), Z, Y, X, int(axis),
                                               coef.ctypes.data_as(C.c_void_p), _ptr(out), _ptr(scratch), C.c_double(scale),
                                               int(accumulate), _stream()), "LoG")
    return out


def log_filter_device(x: torch.Tensor, sigma_mm: float, spacing_zyx, z_pass=None):
    """sigma^2-normalised Laplacian of Gaussian of a CUDA volume (Z,Y,X) -> float32 tensor: for each direction d,
    Gaussian smoothing along the other two axes (z first) then the second derivative along d, summed over d (ITK's
    LaplacianRecursiveGaussianImageFilter, reference radiomics/imageoperations.py:824-830).
    `z_pass(src, sigma_vox, order, scale)` replaces the pass along z: a multi-GPU caller holding a z-slab transposes to
    y-slabs, runs the scan over the whole lines there and transposes back (pipeline.derived_images_slab); every other
    pass is local to the slab, so the distributed result is bit-identical to the single-GPU one."""
    src = x.to(torch.float32).contiguous() if x.dtype != torch.float64 else x.contiguous()
    sz, sy, sx = (sigma_mm / spacing_zyx[0], sigma_mm / spacing_zyx[1], sigma_mm / spacing_zyx[2])
    if z_pass is None:
        z_pass = lambda t, sv, order, scale: _rg_pass(t, 0, sv, order, scale=scale)
    # d = z: smooth y, x; derivative z
    cur = _rg_pass(_rg_pass(src, 1, sy, 0), 2, sx, 0)
    out = z_pass(cur, sz, 2, sz * sz)
    # d = y and d = x both start with the smoothing along z of the input
    gz = z_pass(src, sz, 0, 1.0)
    _rg_pass(_rg_pass(gz, 2, sx, 0), 1, sy, 2, out=out, scale=sy * sy, accumulate=True)      # + sigma^2 d2/dy2
    _rg_pass(_rg_pass(gz, 1, sy, 0), 2, sx, 2, out=out, scale=sx * sx, accumulate=True)      # + sigma^2 d2/dx2
    return out


def getLoGImage(inputImage, _inputMask, **kwargs):
    """reference generator (imageoperations.py:756-836)."""
    arr = I.as_array(inputImage)
    size = np.array(arr.shape[::-1])
    spacing = np.array(I.spacing_xyz(inputImage), dtype=float)
    if arr.ndim != 3 or np.min(size) < 4:
        logger.warning("Image too small to apply LoG filter, size: %s", size)
        return
    x = _to_device(arr)
    for sigma in kwargs.get("sigma", []):
        if sigma > 0.0:
            if np.all(size >= np.ceil(sigma / spacing) + 1):
                out = log_filter_device(x, float(sigma), tuple(spacing[::-1]))
                name = f"log-sigma-{str(sigma).replace('.', '-')}-mm-3D"
                yield I.like(inputImage, out.cpu().numpy()), name, kwargs
            else:
                logger.warning("applyLoG: sigma(%s)/spacing(%s) + 1 must be greater than the size(%s) of the inputImage",
                               sigma, spacing, size)
        else:
            logger.warning("applyLoG: sigma must be greater than 0.0: %s", sigma)
