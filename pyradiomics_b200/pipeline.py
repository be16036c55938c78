"""Device-resident end-to-end pipelines over the hot path (BASELINE.json configs 4 and 5):

* ``voxel_suite_with_filters`` -- Original + wavelet (8 sub-bands) + LoG (one per sigma) derived
  images (+ the square / squareroot / logarithm / exponential / gradient and 3-D LBP images on
  request) -> per-image gray-level discretisation -> the five fused voxel-based texture kernels,
  everything on one GPU without host round trips (what ``RadiomicsFeatureExtractor.execute(...,
  voxelBased=True)`` does image type by image type, reference radiomics/featureextractor.py:371-392).
* ``segment_batch`` -- segment-based matrices + features for a list of independent cases, sharded
  round-robin over the ranks of the process group with no collective (the reference's own
  parallel model: one case per worker, radiomics/scripts/__init__.py:393-404).
"""
from __future__ import annotations

import torch

from . import _lib, featureclasses as FC, imageoperations as IO, voxel
from ._lib import CLASSES


IMAGE_TYPES = ("square", "squareroot", "logarithm", "exponential", "gradient")


def derived_images(x: torch.Tensor, spacing_zyx=(1.0, 1.0, 1.0), wavelet="coif1", sigmas=(1.0, 2.0, 3.0),
                   original=True, lbp3d=None, mask=None, image_types=(), gradient_use_spacing=True):
    """yields (name, CUDA tensor) like the reference's imageType generators.  `image_types`: names out of IMAGE_TYPES,
    yielded after LoG in the caller's order as float64 images (one max|x| reduction serves every per-voxel type;
    `gradient_use_spacing` is getGradientImage's gradientUseSpacing).  `lbp3d`: a settings dict (lbp3DLevels,
    lbp3DIcosphereRadius, lbp3DIcosphereSubdivision; {} = the defaults) adds the 3-D LBP level maps and kurtosis map of
    the ROI `mask` (non-zero voxels) after those, as getLBP3DImage names them; None (default) leaves them out."""
    unknown = [t for t in image_types if t not in IMAGE_TYPES]
    if unknown:
        raise ValueError(f"unknown image types {unknown} (known: {IMAGE_TYPES})")
    if original:
        yield "original", x
    if wavelet:
        lo, hi = IO.wavelet_filters(wavelet)
        xp, crop = IO._wrap_pad_even(x.to(torch.float64), (2, 1, 0))
        dec = IO.swt_level1_device(xp, (2, 1, 0), lo, hi)
        for key, t in dec.items():
            if key != "aaa":
                yield "wavelet-" + key.replace("a", "L").replace("d", "H"), t[crop]
        yield "wavelet-LLL", dec["aaa"][crop]
    for s in sigmas or ():
        yield f"log-sigma-{str(float(s)).replace('.', '-')}-mm-3D", IO.log_filter_device(x, float(s), spacing_zyx)
    max_abs = None
    for t in image_types:
        if t == "gradient":
            yield t, IO.gradient_magnitude_device(x, spacing_zyx if gradient_use_spacing else None)
            continue
        if max_abs is None:
            max_abs = IO.image_max_abs(x)
        yield t, IO.pointwise_image_device(x, t, max_abs)
    if lbp3d is not None:
        if mask is None:
            raise ValueError("the LBP 3-D images need the ROI mask")
        levels = int(lbp3d.get("lbp3DLevels", 2))
        maps = IO.lbp3d_device(x, mask, levels, lbp3d.get("lbp3DIcosphereRadius", 1),
                               int(lbp3d.get("lbp3DIcosphereSubdivision", 1)))
        for n in range(levels):
            yield f"lbp-3D-m{n + 1}", maps[n]
        yield "lbp-3D-k", maps[levels]


def voxel_suite_with_filters(image: torch.Tensor, mask: torch.Tensor, classes=CLASSES, spacing_zyx=(1.0, 1.0, 1.0),
                             wavelet="coif1", sigmas=(1.0, 2.0, 3.0), consume=None, lbp3d=None, image_types=(),
                             gradient_use_spacing=True, normalize=None, resegment=None, **kw):
    """image: CUDA tensor (Z,Y,X) of raw intensities, mask: CUDA uint8/bool.  For every derived
    image (`image_types`, `gradient_use_spacing`, `lbp3d`: see derived_images): bin (binWidth/binCount in kw) -> pack ->
    fused kernels.
    `normalize` (a dict with normalizeScale, removeOutliers; {} = the defaults) normalises the whole image first and every
    derived image comes from the normalised one; `resegment` (a dict with resegmentRange, resegmentMode) then resegments
    the mask against that image, and binning, the texture kernels and the LBP 3-D ROI use the resegmented mask -- the
    reference's order (featureextractor.py:316-392).  None (default) skips either step.
    `consume(name, cls, maps)` is called with each float64 [F,Z,Y,X] result (maps are reused buffers unless consume keeps
    them); returns the list of (image name, Ng, number of levels)."""
    if normalize is not None:
        image = IO.normalize_image_device(image, normalize.get("normalizeScale", 1), normalize.get("removeOutliers"))
    msk = (mask != 0).to(torch.uint8).contiguous()
    if resegment is not None:
        msk, _, _ = IO.resegment_mask_device(image, msk, resegment["resegmentRange"],
                                             resegment.get("resegmentMode", "absolute"))
    outs = {}
    info = []
    for name, img in derived_images(image, spacing_zyx, wavelet, sigmas, lbp3d=lbp3d, mask=msk, image_types=image_types,
                                    gradient_use_spacing=gradient_use_spacing):
        lev32, _ = IO.bin_image_device(img.contiguous(), msk, **kw)
        Ng = int(lev32.max().item())
        lev, presence = voxel.pack_levels(lev32, msk, Ng)
        nlev = int((presence > 0).sum().item())
        s = _lib.make_settings(Ng, nlev, spacing_zyx=spacing_zyx, **kw)
        for c in classes:
            nf = _lib.lib().rb_num_features(_lib.CLASS_ID[c])
            if c not in outs:
                outs[c] = torch.empty((nf,) + tuple(lev.shape), dtype=torch.float64, device=lev.device)
            maps = voxel.voxel_features(c, lev, s, out=outs[c], out_z0=0)
            if consume is not None:
                consume(name, c, maps)
        info.append((name, Ng, nlev))
    return info


def segment_batch(cases, classes=tuple(FC.FEATURE_CLASSES), rank=0, world=1, **kw):
    """cases: sequence of (image ndarray, mask ndarray).  Rank `rank` of `world` processes the cases
    k with k % world == rank on its current CUDA device; returns {case index: {class: {feature: value}}}."""
    res = {}
    for k, (img, msk) in enumerate(cases):
        if k % world != rank:
            continue
        res[k] = {c: {f: float(v) for f, v in FC.FEATURE_CLASSES[c](img, msk, **kw).execute().items()} for c in classes}
    return res


# ---------------------------------------------------------------------------------------------- multi-GPU pre-filters
def derived_images_slab(own: torch.Tensor, Z: int, rank: int, world: int, spacing_zyx=(1.0, 1.0, 1.0), wavelet="coif1",
                        sigmas=(1.0, 2.0, 3.0), original=True):
    """`derived_images` for a volume that is sharded into z-slabs over the ranks of the default process group
    (SURVEY.md section 8e): yields (name, this rank's slab of the derived image).  No LBP 3-D here: its B-spline
    prefilter is a recursion over whole lines along z.  No square / squareroot / logarithm / exponential / gradient
    either: the per-voxel types would need max|x| all-reduced over the ranks, the gradient a replicated edge plane at
    the volume's global z faces.
      * wavelet: the transform is periodic, so the slab gets (F-1-F/2) planes from the rank below and F/2 from the rank
        above, ring-closed between rank 0 and the last rank (distributed.SlabHalo(periodic=True)); an odd global Z is
        wrap-padded by handing the last rank a copy of rank 0's first plane, like the reference pads before transforming;
      * LoG: the recursive Gaussian along z is a sequential scan over whole lines -- z-slabs are transposed to y-slabs
        for that pass and back (distributed.zslab_to_yslab); the x and y passes are local.  Bit-identical to one GPU."""
    import torch.distributed as dist
    from . import distributed as D
    if original:
        yield "original", own
    nz, Y, X = own.shape
    if wavelet:
        lo, hi = IO.wavelet_filters(wavelet)
        F = int(lo.size)
        low, up = F - 1 - F // 2, F // 2
        x64 = own.to(torch.float64)
        last = world - 1
        if Z % 2 and world > 1:                     # global wrap-pad along z: the last rank appends global plane 0
            if rank == 0:
                dist.send(x64[0:1].contiguous(), last)
            if rank == last:
                first = torch.empty_like(x64[0:1])
                dist.recv(first, 0)
                x64 = torch.cat([x64, first], 0)
        elif Z % 2:
            x64 = torch.cat([x64, x64[0:1]], 0)
        xp, crop = IO._wrap_pad_even(x64, (2, 1))           # y, x: local
        slab = D.SlabHalo(xp, low, rank, world, hi=up, periodic=True)
        slab.exchange()
        dec = IO.swt_level1_device(slab.buf, (2, 1, 0), lo, hi, z_range=(low, low + xp.shape[0]))
        crop = (slice(0, nz),) + tuple(crop[1:])
        for key, t in dec.items():
            if key != "aaa":
                yield "wavelet-" + key.replace("a", "L").replace("d", "H"), t[crop]
        yield "wavelet-LLL", dec["aaa"][crop]

    def z_pass(t, sigma_vox, order, scale):
        ys = D.zslab_to_yslab(t, Z, rank, world)
        return D.yslab_to_zslab(IO._rg_pass(ys.contiguous(), 0, sigma_vox, order, scale=scale), Y, rank, world)

    for s in sigmas or ():
        yield (f"log-sigma-{str(float(s)).replace('.', '-')}-mm-3D",
               IO.log_filter_device(own, float(s), spacing_zyx, z_pass=z_pass if world > 1 else None))


def voxel_suite_with_filters_slab(own: torch.Tensor, own_mask: torch.Tensor, Z: int, rank: int, world: int, classes=CLASSES,
                                  spacing_zyx=(1.0, 1.0, 1.0), wavelet="coif1", sigmas=(1.0, 2.0, 3.0), consume=None, **kw):
    """BASELINE.json config 4 on z-slabs: every derived image is binned with the WHOLE ROI's edges (all-reduced min / max
    and gray-level presence), the packed levels exchange one halo plane per face, and the fused texture kernels run on
    the slab.  `consume(name, cls, maps[F, nz, Y, X])` sees each result; returns [(image name, Ng, number of levels)]."""
    import torch.distributed as dist
    from . import distributed as D
    msk = (own_mask != 0).to(torch.uint8).contiguous()
    dev = own.device
    r = int(kw.get("kernelRadius", 1))

    def reduce_minmax(mn, mx):
        if world == 1:
            return mn, mx
        t = torch.tensor([-mn, mx], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return -float(t[0].item()), float(t[1].item())

    info, outs = [], {}
    nz = own.shape[0]
    for name, img in derived_images_slab(own, Z, rank, world, spacing_zyx, wavelet, sigmas):
        lev32, _ = IO.bin_image_device(img.contiguous(), msk, minmax_reduce=reduce_minmax, **kw)
        ngt = lev32.max().to(torch.int64).reshape(1)
        if world > 1:
            dist.all_reduce(ngt, op=dist.ReduceOp.MAX)
        Ng = int(ngt.item())
        lev, presence = voxel.pack_levels(lev32, msk, Ng)
        pres = presence.to(torch.int64)
        if world > 1:
            dist.all_reduce(pres, op=dist.ReduceOp.SUM)
        nlev = int((pres > 0).sum().item())
        s = _lib.make_settings(Ng, nlev, spacing_zyx=spacing_zyx, **kw)
        slab = D.SlabHalo(lev, r, rank, world)
        slab.exchange()
        alive = D.allreduce_alive(voxel.glcm_alive_angles(slab.buf, s), dev) if "glcm" in classes else None
        for c in classes:
            nf = _lib.lib().rb_num_features(_lib.CLASS_ID[c])
            if c not in outs:
                outs[c] = torch.empty((nf, nz) + tuple(lev.shape[1:]), dtype=torch.float64, device=dev)
            maps = voxel.voxel_features(c, slab.buf, s, z0=r, z1=r + nz, out=outs[c], out_z0=r, alive=alive if c == "glcm" else None)
            if consume is not None:
                consume(name, c, maps)
        info.append((name, Ng, nlev))
    return info
