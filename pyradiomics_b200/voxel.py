"""Voxel-based (feature-map) extraction on device-resident volumes: the headline path.

Mirrors what the reference does per feature class in voxel-based mode (reference
radiomics/base.py:98-111,200-245 + the per-class _calculateMatrix/_calculateCoefficients/get*
methods) but as one fused CUDA kernel per class that never materialises per-voxel matrices.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib, imageoperations
from ._lib import CLASS_ID, CLASSES, check, lib, ptr, stream


def pack_levels(image: torch.Tensor, mask: torch.Tensor, Ng: int):
    """int32 gray-level volume + mask (both CUDA) -> compact level volume (uint8 when Ng <= 255,
    else int16 storage of uint16), 0 outside the mask; returns (levels, presence[Ng] int32 counts).
    Raises IndexError when a masked voxel is outside 1..Ng (reference _cmatrices.c:219)."""
    assert image.is_cuda and mask.is_cuda and image.shape == mask.shape
    image = image.to(torch.int32).contiguous()
    mask = (mask != 0).to(torch.uint8).contiguous()
    lb = lib().rb_level_bytes(int(Ng))
    lev = torch.empty(image.shape, dtype=torch.uint8 if lb == 1 else torch.int16, device=image.device)
    presence = torch.zeros(int(Ng), dtype=torch.int32, device=image.device)
    status = torch.zeros(1, dtype=torch.int32, device=image.device)
    check(lib().rb_pack_levels_dev(ptr(image), ptr(mask), image.numel(), int(Ng), ptr(lev), ptr(presence), ptr(status),
                                   stream()), "pack_levels")
    if int(status.item()) & 1:
        raise IndexError("gray level outside 1..Ng inside the mask")
    return lev, presence


def discretize(image: torch.Tensor, mask: torch.Tensor, /, all_reduce=None, **binning):
    """One image's gray-level discretisation on the device (the reference's binImage + the levels present in the ROI):
    bin (imageoperations.bin_image_device, binWidth / binCount in `binning`) -> Ng, the largest level -> pack_levels ->
    the gray levels that occur in the ROI.  `all_reduce` (torch.distributed.all_reduce's signature) makes a z-slab of a
    volume sharded over ranks use the whole ROI's min / max, Ng and levels.
    Returns (int32 levels, bin edges, packed levels, gray levels present as an int64 ndarray, Ng)."""
    minmax_reduce = None
    if all_reduce is not None:
        from torch.distributed import ReduceOp

        def minmax_reduce(mn, mx):                      # MIN of the minima as MAX of their negatives: one collective
            t = torch.tensor([-mn, mx], dtype=torch.float64, device=image.device)
            all_reduce(t, op=ReduceOp.MAX)
            neg_mn, mx = t.tolist()
            return -neg_mn, mx
    lev32, edges = imageoperations.bin_image_device(image, mask, minmax_reduce=minmax_reduce, **binning)
    Ng = lev32.max()
    if all_reduce is not None:
        Ng = Ng.to(torch.int64).reshape(1)
        all_reduce(Ng, op=ReduceOp.MAX)
    Ng = int(Ng.item())
    lev, presence = pack_levels(lev32, mask, max(Ng, 1))
    if all_reduce is not None:
        presence = presence.to(torch.int64)
        all_reduce(presence, op=ReduceOp.SUM)
    gray_levels = (torch.nonzero(presence).flatten() + 1).cpu().numpy().astype(np.int64)
    return lev32, edges, lev, gray_levels, Ng


def level_bytes(lev: torch.Tensor) -> int:
    return 1 if lev.dtype == torch.uint8 else 2


# the map types the texture kernels write: float64 (the reference's) or float32, each value rounded once from float64
MAP_DTYPES = (torch.float64, torch.float32)


def out_is_f32(out: torch.Tensor) -> int:
    """rb_voxel_features_dev's out_is_f32 for a map buffer; any other dtype raises TypeError"""
    if out.dtype not in MAP_DTYPES:
        raise TypeError(f"voxel feature maps are float64 or float32, not {out.dtype}")
    return int(out.dtype == torch.float32)


def glcm_alive_angles(lev, settings, centers=None):
    Z, Y, X = lev.shape
    alive = torch.zeros(_lib.ALIVE_WORDS, dtype=torch.int32, device=lev.device)
    check(lib().rb_glcm_alive_angles_dev(ptr(lev), level_bytes(lev), ptr(centers), Z, Y, X, C.byref(settings), ptr(alive),
                                         stream()), "glcm_alive_angles")
    return alive.cpu().numpy().view(np.uint32).copy()


def voxel_features(cls: str, lev: torch.Tensor, settings, *, centers=None, z0=0, z1=None, out=None, out_z0=None,
                   alive=None, status=None, dtype=torch.float64):
    """Launch the fused kernel of one class on planes [z0,z1) of `lev` (Z,Y,X).  Returns `out`:
    [F, z1-z0, Y, X] maps of type `dtype` (float64 or float32), allocated when None.  A given `out` is float64 or float32
    (its dtype decides; `dtype` is then ignored), with contiguous (Y, X) planes and any feature stride; plane z of the
    volume goes to out[:, z - out_z0].  Asynchronous on the current stream."""
    cid = CLASS_ID[cls]
    Z, Y, X = lev.shape
    z1 = Z if z1 is None else z1
    nf = lib().rb_num_features(cid)
    if out is None:
        out = torch.empty((nf, z1 - z0, Y, X), dtype=dtype, device=lev.device)
        out_z0 = z0
    f32 = out_is_f32(out)
    assert out.shape[0] == nf and out.shape[2:] == (Y, X) and out.stride()[1:] == (Y * X, X, 1)
    if out_z0 is None:
        out_z0 = z0
    if cls == "glcm" and alive is None:
        alive = glcm_alive_angles(lev, settings, centers)
    if status is None:
        status = torch.zeros(1, dtype=torch.int32, device=lev.device)
    check(lib().rb_voxel_features_dev(cid, ptr(lev), level_bytes(lev), ptr(centers), Z, Y, X, int(z0), int(z1),
                                      C.byref(settings), ptr(alive), ptr(out), f32, out.stride(0), int(out_z0), ptr(status),
                                      stream()), cls)
    return out


def extract_maps(image, mask, classes=CLASSES, **kw):
    """Convenience: discretised int volume + mask (numpy or CUDA tensors) -> {class: {feature: map}}
    with maps as float64 CUDA tensors (Z,Y,X).  `image` must already hold gray levels 1..Ng inside
    the mask (see imageoperations.bin_image for the discretisation kernel)."""
    dev = torch.device("cuda", torch.cuda.current_device())
    img = torch.as_tensor(np.ascontiguousarray(image) if isinstance(image, np.ndarray) else image).to(dev)
    msk = torch.as_tensor(np.ascontiguousarray(mask) if isinstance(mask, np.ndarray) else mask).to(dev)
    if img.ndim == 2:
        img, msk = img[None], msk[None]
        if kw.get("force2D"):
            kw = dict(kw, force2Ddimension=kw.get("force2Ddimension", 0) + 1)
    Ng = int(torch.where(msk != 0, img, torch.zeros_like(img)).max().item())
    lev, presence = pack_levels(img, msk, Ng)
    n_levels = int((presence > 0).sum().item())
    settings = _lib.make_settings(Ng, n_levels, **kw)
    res = {}
    for cls in classes:
        out = voxel_features(cls, lev, settings)
        res[cls] = {name: out[i] for i, name in enumerate(_lib.feature_names(cls))}
    return res


FIRSTORDER_NF = 18


def roi_box(roi: torch.Tensor):
    """the bounding box of the non-zero voxels of the CUDA tensor `roi` as a tuple of slices (one host copy)"""
    on = roi != 0
    first, last = [], []
    for d in range(on.ndim):
        idx = torch.nonzero(on.any(dim=tuple(k for k in range(on.ndim) if k != d))).flatten()
        first.append(idx[0])
        last.append(idx[-1])
    lo, hi = torch.stack([torch.stack(first), torch.stack(last)]).tolist()
    return tuple(slice(int(a), int(b) + 1) for a, b in zip(lo, hi))


def roi_extent(roi):
    """per-axis size of the bounding box of the non-zero voxels of `roi` (an ndarray or a CUDA tensor, 2-D or 3-D)"""
    if isinstance(roi, torch.Tensor):
        return [s.stop - s.start for s in roi_box(roi)]
    m = np.asarray(roi) != 0
    size = []
    for d in range(m.ndim):
        on = np.flatnonzero(m.any(axis=tuple(k for k in range(m.ndim) if k != d)))
        size.append(int(on[-1] - on[0] + 1))
    return size


def firstorder_radii(kernelRadius, shape, roi=None, force2D=False, force2Ddimension=0):
    """The window radii of voxel-based first order, one per axis of `shape`, as the reference forms them: kernelRadius
    clipped to the ROI's bounding-box size - 1 (`roi`: non-zero = in the ROI; None, an unmasked kernel: to the image
    size - 1), 0 on the force2D axis."""
    size = list(shape) if roi is None else roi_extent(roi)
    rad = [int(min(int(kernelRadius), s - 1)) for s in size]
    if force2D:
        rad[int(force2Ddimension)] = 0
    return rad


def voxel_volume(spacing_zyx):
    """the product of the voxel spacing, multiplied in x, y, z order as the reference's np.multiply.reduce(pixelSpacing)"""
    return float(np.multiply.reduce(np.asarray(spacing_zyx, dtype=np.float64)[::-1]))


def firstorder_launch(image, lev, kmask, radii, *, centers=None, voxelArrayShift=0, voxel_volume=1.0, initValue=0):
    """the `launch(za, zb, buf, out_z0=za)` of rb_firstorder_voxel_dev: the first-order maps of planes [za,zb) of the
    (Z,Y,X) volume into the float64 `buf` [18, ..., Y, X] (plane z at buf[:, z - out_z0]) on the current stream.
    `image`: raw or derived intensities (any device pixel type), `lev`: packed levels (0 = not in the kernel), `kmask`:
    the voxels that enter windows (None: every voxel), `centers`: the voxels that get maps (None: kmask), `radii`:
    (rz, ry, rx)."""
    Z, Y, X = lev.shape
    assert image.shape == lev.shape and image.is_contiguous() and lev.is_contiguous()
    assert kmask is None or (kmask.shape == lev.shape and kmask.dtype == torch.uint8 and kmask.is_contiguous())
    assert centers is None or (centers.shape == lev.shape and centers.dtype == torch.uint8 and centers.is_contiguous())
    rz, ry, rx = (int(r) for r in radii)

    def launch(za, zb, buf, out_z0=None):
        if buf.dtype != torch.float64:
            raise TypeError(f"first-order maps leave the kernel as float64, not {buf.dtype}")
        assert buf.shape[0] == FIRSTORDER_NF and buf.stride()[1:] == (Y * X, X, 1)
        check(lib().rb_firstorder_voxel_dev(ptr(image), _lib.TORCH_DTYPE_CODE[image.dtype], ptr(kmask), ptr(centers), ptr(lev),
                                            level_bytes(lev), Z, Y, X, rz, ry, rx, float(voxelArrayShift),
                                            float(voxel_volume), float(initValue), ptr(buf), buf.stride(0), int(za), int(zb),
                                            int(za if out_z0 is None else out_z0),
                                            torch.cuda.current_stream(lev.device).cuda_stream), "firstorder")
    return launch


def firstorder_features(image: torch.Tensor, lev: torch.Tensor, roi, *, kernelRadius=1, force2D=False, force2Ddimension=0,
                        voxelArrayShift=0, initValue=0, spacing_zyx=(1.0, 1.0, 1.0), centers=None, z0=0, z1=None, out=None,
                        out_z0=None, dtype=torch.float64, zchunk=16):
    """The device-resident first-order maps, the counterpart of voxel_features: planes [z0,z1) of the (Z,Y,X) CUDA
    volumes `image` (raw or derived intensities, any device pixel type), `lev` (packed levels, 0 outside the ROI) and
    `roi` (the kernel mask: the voxels that enter windows; None = every voxel, an unmasked kernel).  `centers` (CUDA,
    non-zero = gets maps) defaults to `roi`; other voxels get `initValue`.  The radii follow firstorder_radii.
    Returns `out`: [18, z1-z0, Y, X] in feature_names("firstorder") order, of type `dtype` (float64 or float32),
    allocated when None; a given `out` decides the type by its dtype and has contiguous (Y, X) planes, plane z at
    out[:, z - out_z0].  Float32 maps are the float64 maps rounded once: the kernel writes z-chunks of `zchunk` planes
    into a float64 scratch that converts on the device.  Asynchronous on the current stream."""
    Z, Y, X = lev.shape
    z1 = Z if z1 is None else int(z1)
    z0 = int(z0)
    if out is None:
        out = torch.empty((FIRSTORDER_NF, z1 - z0, Y, X), dtype=dtype, device=lev.device)
        out_z0 = z0
    f32 = out_is_f32(out)
    assert out.shape[0] == FIRSTORDER_NF and out.shape[2:] == (Y, X) and out.stride()[1:] == (Y * X, X, 1)
    out_z0 = z0 if out_z0 is None else int(out_z0)
    image = image.contiguous()
    kmask = None if roi is None else (roi != 0).to(torch.uint8).contiguous()
    cen = None if centers is None else (centers != 0).to(torch.uint8).contiguous()
    radii = firstorder_radii(kernelRadius, lev.shape, kmask, force2D, force2Ddimension)
    launch = firstorder_launch(image, lev, kmask, radii, centers=cen, voxelArrayShift=voxelArrayShift,
                               voxel_volume=voxel_volume(spacing_zyx), initValue=initValue)
    if not f32:
        launch(z0, z1, out, out_z0)
        return out
    plane = Y * X
    zc = max(1, min(int(zchunk), z1 - z0))
    scratch = torch.empty((FIRSTORDER_NF, zc, Y, X), dtype=torch.float64, device=lev.device)
    st = torch.cuda.current_stream(lev.device).cuda_stream
    for za in range(z0, z1, zc):
        zb = min(za + zc, z1)
        launch(za, zb, scratch, za)
        check(lib().rb_maps_to_f32_dev(ptr(scratch), scratch.stride(0), out.data_ptr() + (za - out_z0) * plane * 4,
                                       out.stride(0), (zb - za) * plane, FIRSTORDER_NF, st), "maps_to_f32")
    return out


def firstorder_segment(image: torch.Tensor, lev: torch.Tensor, roi: torch.Tensor, *, voxelArrayShift=0,
                       spacing_zyx=(1.0, 1.0, 1.0)):
    """Segment-based first order on the device, the counterpart of firstorder_features: the 18 features of the ROI
    (`roi` non-zero) of the CUDA intensities `image` (raw or derived, any device pixel type), with Entropy / Uniformity
    from the packed levels `lev` (rb_pack_levels_dev, e.g. discretize's), all of one 2-D or 3-D shape.  Runs on the
    current stream with no host copy of the volumes (rb_firstorder_segment_dev) and returns {feature: np.float64} in
    feature_names("firstorder") order.  ValueError for an empty ROI."""
    assert image.is_cuda and lev.is_cuda and roi.is_cuda and image.shape == lev.shape == roi.shape and image.ndim in (2, 3)
    Z, Y, X = ((1,) + tuple(image.shape)) if image.ndim == 2 else tuple(image.shape)
    image = image.contiguous()
    lev = lev.contiguous()
    roi = (roi != 0).to(torch.uint8).contiguous()
    if not bool(roi.any()):                  # before any launch of the reduction (it would only report it at its end)
        raise ValueError("first order: the ROI is empty")
    out = (C.c_double * FIRSTORDER_NF)()
    check(lib().rb_firstorder_segment_dev(ptr(image), _lib.TORCH_DTYPE_CODE[image.dtype], ptr(roi), ptr(lev),
                                          level_bytes(lev), Z, Y, X, float(voxelArrayShift), voxel_volume(spacing_zyx), out,
                                          torch.cuda.current_stream(lev.device).cuda_stream), "firstorder")
    return {n: np.float64(out[k]) for k, n in enumerate(_lib.feature_names("firstorder"))}


def _runs(idx):
    """[(first feature index, count, position in idx)] for every run of consecutive indices"""
    out, k = [], 0
    while k < len(idx):
        j = k
        while j + 1 < len(idx) and idx[j + 1] == idx[j] + 1:
            j += 1
        out.append((idx[k], j - k + 1, k))
        k = j + 1
    return out


def texture_launch(cls: str, lev: torch.Tensor, settings, *, centers=None, alive=None, status=None):
    """the `launch(za, zb, buf)` of maps_to_host for the fused kernel of one texture class: planes [za,zb) of `lev` into
    `buf` [F, >= zb-za, Y, X] (plane za at buf[:, 0], float64 or float32 maps as buf's dtype) on the current stream"""
    cid = CLASS_ID[cls]
    Z, Y, X = lev.shape
    if cls == "glcm" and alive is None:
        alive = glcm_alive_angles(lev, settings, centers)
    if status is None:
        status = torch.zeros(1, dtype=torch.int32, device=lev.device)

    def launch(za, zb, buf):
        check(lib().rb_voxel_features_dev(cid, ptr(lev), level_bytes(lev), ptr(centers), Z, Y, X, int(za), int(zb),
                                          C.byref(settings), ptr(alive), ptr(buf), out_is_f32(buf), buf.stride(0), int(za),
                                          ptr(status), torch.cuda.current_stream(lev.device).cuda_stream), cls)
    return launch


def class_maps_to_host(cls: str, lev: torch.Tensor, settings, feature_idx=None, *, centers=None, alive=None, z0=0, z1=None,
                       zchunk=64, out_dtype=torch.float64, host=None, copy_stream=None, status=None, progress=None, sync=True):
    """Output assembly of one texture class (the reference's per-batch `featureMaps[tuple(voxelCoords)] = ...`,
    radiomics/base.py:205-209,232-234, without the batch loop): maps_to_host over the class's fused kernel
    (texture_launch)."""
    launch = texture_launch(cls, lev, settings, centers=centers, alive=alive, status=status)
    return maps_to_host(launch, lib().rb_num_features(CLASS_ID[cls]), lev.shape, lev.device, feature_idx, z0=z0, z1=z1,
                        zchunk=zchunk, out_dtype=out_dtype, host=host, copy_stream=copy_stream, progress=progress, sync=sync,
                        map_dtypes=MAP_DTYPES)


def maps_to_host(launch, nf, shape, dev, feature_idx=None, *, z0=0, z1=None, zchunk=64, out_dtype=torch.float64,
                 host=None, copy_stream=None, progress=None, sync=True, map_dtypes=(torch.float64,)):
    """The voxel-map driver of every voxel class: `launch(za, zb, buf)` enqueues the `nf` maps of planes [za,zb) of a
    (Z,Y,X) = `shape` volume into `buf` [nf, >= zb-za, Y, X] on the current stream of device `dev`.  Planes [z0,z1) run
    in z-chunks into a two-slot device ring; every finished chunk leaves for the host on `copy_stream` -- ONE strided DMA
    per run of consecutive selected features (rb_memcpy2d_async) -- while the next chunk computes.  Only the maps in
    `feature_idx` (default: all) are copied.  `map_dtypes` are the map types `launch` writes (the texture kernels:
    MAP_DTYPES): an `out_dtype` among them is the ring's type, so float32 maps go from the kernel to the host with no
    float64 copy on the device; otherwise the ring is float64 and float32 converts on the device before the copy (half
    the PCIe bytes either way).
    Returns the page-locked host tensor [len(feature_idx), z1-z0, Y, X] (allocated from torch's caching pinned
    allocator when `host` is None: the caller owns it, dropping it recycles the block).  sync=False returns without
    waiting for the last copies (the caller synchronises `copy_stream` before touching `host`), so a following class
    starts computing while this one's tail is still on the wire."""
    Z, Y, X = shape
    z1 = Z if z1 is None else int(z1)
    nz = z1 - int(z0)
    idx = list(range(nf)) if feature_idx is None else [int(k) for k in feature_idx]
    if host is None:
        host = torch.empty((len(idx), nz, Y, X), dtype=out_dtype, pin_memory=True)
    assert host.shape == (len(idx), nz, Y, X) and host.dtype == out_dtype and host.is_contiguous()
    if not idx or nz <= 0:
        return host
    cur = torch.cuda.current_stream(dev)
    copy_stream = copy_stream or torch.cuda.Stream(device=dev)
    zc = max(1, min(int(zchunk), nz))
    plane = Y * X
    native = out_dtype in map_dtypes
    ring = [torch.empty((nf, zc, Y, X), dtype=out_dtype if native else torch.float64, device=dev)
            for _ in range(2 if nz > zc else 1)]
    f32 = out_dtype == torch.float32 and not native         # convert float64 maps on the device
    ring32 = [torch.empty((len(idx), zc, Y, X), dtype=torch.float32, device=dev) for _ in ring] if f32 else None
    esz = host.element_size()
    for t in ring + (ring32 or []):
        t.record_stream(copy_stream)                     # the caching allocator must not recycle them under the DMA
    copied = [None, None]
    L = lib()
    for i, za in enumerate(range(int(z0), z1, zc)):
        zb = min(za + zc, z1)
        slot = i % len(ring)
        if copied[slot] is not None:
            cur.wait_event(copied[slot])                 # the DMA of the chunk that used this slot has finished
        buf = ring[slot]
        launch(za, zb, buf)
        width = (zb - za) * plane
        if f32:
            for first, count, pos in _runs(idx):
                check(L.rb_maps_to_f32_dev(buf.data_ptr() + first * buf.stride(0) * 8, buf.stride(0),
                                           ring32[slot].data_ptr() + pos * ring32[slot].stride(0) * 4, ring32[slot].stride(0),
                                           width, count, cur.cuda_stream), "maps_to_f32")
        done = torch.cuda.Event()
        done.record(cur)
        copy_stream.wait_event(done)
        off = (za - int(z0)) * plane
        if f32:
            src = ring32[slot]
            check(L.rb_memcpy2d_async(host.data_ptr() + off * 4, host.stride(0) * 4, ptr(src), src.stride(0) * 4, width * 4,
                                      len(idx), 2, copy_stream.cuda_stream), "memcpy2d")
        else:
            for first, count, pos in _runs(idx):
                check(L.rb_memcpy2d_async(host.data_ptr() + (pos * host.stride(0) + off) * esz, host.stride(0) * esz,
                                          buf.data_ptr() + first * buf.stride(0) * esz, buf.stride(0) * esz, width * esz,
                                          count, 2, copy_stream.cuda_stream), "memcpy2d")
        ev = torch.cuda.Event()
        ev.record(copy_stream)
        copied[slot] = ev
        if progress is not None:
            progress(zb - za)
    if sync:
        copy_stream.synchronize()
    return host


class HostExtractor:
    """End-to-end voxel-based extraction with HOST buffers (what a pyradiomics user holds):
    int32 gray levels + mask in, float64 (or `out_dtype` float32) feature maps out, all transfers inside.  Pinned staging is
    allocated once and reused.  The 80 GB of result maps is what bounds this path (PCIe), so the
    device->host stream is kept busy from the first milliseconds: classes run in order of
    (bytes out / compute time), every class is cut into z-chunks (class_maps_to_host), and a chunk's
    maps are copied on a second stream while the next chunk / class computes.

    `shape` is the (Z,Y,X) block handed to this GPU; `z0:z1` (default everything) selects the
    planes whose maps are computed and returned -- a multi-GPU caller passes its slab plus halo
    planes read from the host volume and keeps only the interior (no collective needed)."""

    ORDER = ("gldm", "glszm", "glrlm", "ngtdm", "glcm")      # cheap-and-wide first, GLCM last

    def __init__(self, shape, classes=CLASSES, device=None, z0=0, z1=None, zchunk=64, out_dtype=torch.float64):
        self.shape = tuple(int(s) for s in shape)
        self.classes = tuple(c for c in self.ORDER if c in classes)
        self.dev = torch.device("cuda", torch.cuda.current_device()) if device is None else device
        self.z0, self.z1 = int(z0), int(self.shape[0] if z1 is None else z1)
        self.zchunk = int(zchunk)
        self.out_dtype = out_dtype
        self.out_shape = (self.z1 - self.z0,) + self.shape[1:]
        self.nf = {c: lib().rb_num_features(CLASS_ID[c]) for c in self.classes}
        n = int(np.prod(self.shape))
        self.d_img = torch.empty(self.shape, dtype=torch.int32, device=self.dev)
        self.d_msk = torch.empty(self.shape, dtype=torch.uint8, device=self.dev)
        self.h_img = torch.empty(self.shape, dtype=torch.int32, pin_memory=True)
        self.h_msk = torch.empty(self.shape, dtype=torch.uint8, pin_memory=True)
        self.h_out = {c: torch.empty((self.nf[c],) + self.out_shape, dtype=out_dtype, pin_memory=True) for c in self.classes}
        self.copy_stream = torch.cuda.Stream(device=self.dev)
        self.h2d_bytes = n * 5
        self.d2h_bytes = sum(self.nf.values()) * int(np.prod(self.out_shape)) * (4 if out_dtype == torch.float32 else 8)

    def run(self, image: np.ndarray, mask: np.ndarray, Ng: int, n_roi_levels: int, alive=None, **kw):
        """returns {class: pinned tensor [F, z1-z0, Y, X]} (valid until the next run())."""
        self.h_img.numpy()[...] = image
        self.h_msk.numpy()[...] = mask
        self.d_img.copy_(self.h_img, non_blocking=True)
        self.d_msk.copy_(self.h_msk, non_blocking=True)
        lev, _ = pack_levels(self.d_img, self.d_msk, Ng)
        settings = _lib.make_settings(Ng, n_roi_levels, **kw)
        if alive is None and "glcm" in self.classes:
            from . import distributed as D
            alive = D.allreduce_alive(glcm_alive_angles(lev, settings), self.dev)   # OR over the slabs' ranks
        for c in self.classes:
            class_maps_to_host(c, lev, settings, None, alive=alive if c == "glcm" else None, z0=self.z0, z1=self.z1,
                               zchunk=self.zchunk, out_dtype=self.out_dtype, host=self.h_out[c], copy_stream=self.copy_stream,
                               sync=False)
        self.copy_stream.synchronize()
        torch.cuda.current_stream(self.dev).synchronize()
        return self.h_out


def extract_to_nrrd(lev: torch.Tensor, settings, out_dir, classes=CLASSES, prefix="original", spacing_xyz=(1.0, 1.0, 1.0),
                    origin_xyz=(0.0, 0.0, 0.0), compress=True, level=1, workers=8, out_dtype=torch.float64, centers=None,
                    zchunk=64, features=None, image=None, voxelArrayShift=0):
    """Voxel driver + output assembly in one pipeline (the reference: extractor.execute(..., voxelBased=True) then one
    sitk.WriteImage(map, target, True) per map, radiomics/scripts/voxel.py:62-72): the fused kernels of one class stream
    their maps chunk by chunk into page-locked host memory (class_maps_to_host) while a pool of writer threads gzips the
    PREVIOUS class's maps into <prefix>_<class>_<Feature>.nrrd files (zlib releases the GIL), so compression and disk
    overlap the GPU and the PCIe stream.  `features` = {class: [names]} restricts what is copied and written.
    "firstorder" in `classes` also writes the first-order maps of `image` (the CUDA intensities `lev` was binned from;
    `voxelArrayShift` as the reference's setting): its kernel mask is `lev != 0`, or every voxel when `centers` is given
    (an unmasked kernel), its radii, force2D and initValue come from `settings`, the voxel volume from `spacing_xyz`.
    Returns {feature key: path}."""
    import concurrent.futures as cf
    import os

    from . import nrrd
    fo_launch = None
    if "firstorder" in classes:
        if image is None:
            raise ValueError("first-order maps need the intensity image (image=...)")
        kmask = (lev != 0).to(torch.uint8) if centers is None else None
        radii = firstorder_radii(settings.kernelRadius, lev.shape, kmask, settings.force2D, settings.force2Ddimension)
        cen = None if centers is None else (centers != 0).to(torch.uint8).contiguous()
        fo_launch = firstorder_launch(image.contiguous(), lev, kmask, radii, centers=cen, voxelArrayShift=voxelArrayShift,
                                      voxel_volume=voxel_volume(tuple(spacing_xyz)[::-1]), initValue=settings.initValue)
    os.makedirs(out_dir, exist_ok=True)
    jobs, keep = {}, []
    copy_stream = torch.cuda.Stream(device=lev.device)
    with cf.ThreadPoolExecutor(max_workers=max(1, int(workers))) as ex:
        for c in [c for c in HostExtractor.ORDER if c in classes] + (["firstorder"] if fo_launch else []):
            names = _lib.feature_names(c)
            want = names if not features or c not in features else [n for n in names if n in set(features[c])]
            idx = [names.index(n) for n in want]
            if not idx:
                continue
            if c == "firstorder":
                host = maps_to_host(fo_launch, FIRSTORDER_NF, lev.shape, lev.device, idx, zchunk=zchunk, out_dtype=out_dtype,
                                    copy_stream=copy_stream, sync=True)
            else:
                host = class_maps_to_host(c, lev, settings, idx, centers=centers, zchunk=zchunk, out_dtype=out_dtype,
                                          copy_stream=copy_stream, sync=True)
            keep.append(host)
            arr = host.numpy()
            for pos, n in enumerate(want):
                key = f"{prefix}_{c}_{n}"
                jobs[key] = ex.submit(nrrd.write_nrrd, os.path.join(out_dir, key + ".nrrd"), arr[pos], spacing_xyz, origin_xyz,
                                      compress, level)
        return {k: j.result() for k, j in jobs.items()}
