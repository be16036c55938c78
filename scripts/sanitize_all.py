"""compute-sanitizer target: ONE small invocation of every kernel family of the library (fused voxel fast
paths, the generic voxel kernel, the cMatrices builders in segment and voxel-batch mode, discretisation,
wavelet, LoG, shape, first-order, 3-D LBP, the square / squareroot / logarithm / exponential / gradient
image types, normalisation and resegmentation).  Run as
    compute-sanitizer --tool memcheck|racecheck|initcheck|synccheck python scripts/sanitize_all.py [N] [family ...]
The families are independent so a slow tool can be pointed at one of them."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from pyradiomics_b200 import _lib, cmatrices, cshape, featureclasses as FC, image as I, imageoperations as IO, voxel

args = [a for a in sys.argv[1:]]
N = int(args.pop(0)) if args and args[0].isdigit() else 20
N16 = N - N % 16 if N >= 16 else N
fams = args or ["fast", "generic", "matrix", "filters", "shape", "firstorder", "lbp3d", "imagetypes", "preprocess"]
rng = np.random.default_rng(0)


def volumes():
    lev_u = rng.integers(1, 33, (N, N + 1, N + 2)).astype(np.int32)
    f = torch.randn(1, 1, N, N + 1, N + 2)
    f = torch.nn.functional.conv3d(f, torch.ones(1, 1, 5, 5, 5) / 125, padding=2)[0, 0].numpy()
    q = np.quantile(f, np.linspace(0, 1, 33)[1:-1])
    lev_s = (np.digitize(f, q) + 1).astype(np.int32)
    return {"uniform": lev_u, "smooth": lev_s}


vols = volumes()
mask_full = np.ones(vols["uniform"].shape, bool)
mask_rag = rng.random(mask_full.shape) < 0.8

if "fast" in fams:
    for kind, lev in vols.items():
        for m in (mask_full, mask_rag):
            res = voxel.extract_maps(lev, m)
            torch.cuda.synchronize()
            print("fast", kind, "ok", float(res["glcm"]["MCC"].nanmean().item()), flush=True)

if "generic" in fams:
    os.environ["B200_RADIOMICS_FORCE_GENERIC"] = "1"
    n = min(N, 12)
    lev = vols["smooth"][:n, :n, :n]
    for kw in ({}, {"kernelRadius": 2, "distances": [1, 2]}, {"weightingNorm": "euclidean"}, {"symmetricalGLCM": False},
               {"kernelRadius": 3, "symmetricalGLCM": False}, {"force2D": True, "force2Ddimension": 0}):
        res = voxel.extract_maps(lev, mask_rag[:n, :n, :n], **kw)
        torch.cuda.synchronize()
        print("generic", kw, "ok", flush=True)
    del os.environ["B200_RADIOMICS_FORCE_GENERIC"]

if "matrix" in fams:
    lev = vols["smooth"]
    for m in (mask_full, mask_rag):
        P, _ = cmatrices.calculate_glcm(lev, m, [1], 32, False, -1)
        cmatrices.calculate_glrlm(lev, m, 32, max(lev.shape), False, -1)
        cmatrices.calculate_glszm(lev, m, 32, int(m.sum()), False, -1)
        cmatrices.calculate_gldm(lev, m, [1], 32, 0, False, -1)
        cmatrices.calculate_ngtdm(lev, m, [1], 32, False, -1)
        vox = np.array(np.where(m))[:, ::37].astype(np.int32)
        cmatrices.calculate_glcm(lev, m, [1], 32, False, -1, 1, vox)
        cmatrices.calculate_glrlm(lev, m, 32, max(lev.shape), False, -1, 1, vox)
        cmatrices.calculate_glszm(lev, m, 32, 27, False, -1, 1, vox)
        cmatrices.calculate_gldm(lev, m, [1], 32, 0, False, -1, 1, vox)
        cmatrices.calculate_ngtdm(lev, m, [1], 32, False, -1, 1, vox)
        print("matrix ok", float(P.sum()), flush=True)
    # a row pitch that is a multiple of 16 bytes: the fused tile kernel stages its boxes by TMA (else cooperative loads)
    lt, mt = np.ascontiguousarray(lev[:, :, :N16]), np.ascontiguousarray(mask_rag[:, :, :N16])
    for tma in ("1", "0"):
        os.environ["B200_SEG_TMA"] = tma
        cmatrices.calculate_glcm(lt, mt, [1, 2], 32, False, -1)
        cmatrices.calculate_gldm(lt, mt, [1], 32, 1, False, -1)
        cmatrices.calculate_ngtdm(lt, mt, [1], 32, False, -1)
        levd, _ = voxel.pack_levels(torch.as_tensor(lt).cuda(), torch.as_tensor(mt).cuda(), 32)
        cmatrices.segment_texture_device(levd, [1], 32, 0, False, -1)
        cmatrices.calculate_glrlm_device(levd, 32, max(lt.shape), False, -1)
        cmatrices.calculate_glszm_device(levd, 32, False, -1)
    del os.environ["B200_SEG_TMA"]
    print("matrix tma/coop ok", flush=True)
    cmatrices.calculate_glcm(lev[3], mask_rag[3], [1, 2], 32, False, -1)          # 2-D
    cmatrices.calculate_glszm(lev[3], mask_rag[3], 32, int(mask_rag[3].sum()), False, -1)
    # the direct segment kernel: 16-bit levels (all three matrices in one pass), and offsets > 3 in 2-D
    levd, _ = voxel.pack_levels(torch.as_tensor(lev + 268).cuda(), torch.as_tensor(mask_rag).cuda(), 300)
    cmatrices.segment_texture_device(levd, [1, 2], 300, 0, False, -1)
    cmatrices.calculate_glcm(lev[3], mask_rag[3], [1, 4], 32, False, -1)
    print("matrix direct ok", flush=True)

if "filters" in fams:
    raw = (vols["smooth"].astype(np.float64) - 1) * 25 + rng.random(mask_full.shape) * 20
    for arr in (raw, raw.astype(np.float32), raw.astype(np.int16)):
        IO.binImage(arr, mask_rag, binWidth=25)
        IO.binImage(arr, mask_rag, binCount=16)
    odd = raw[: N - 1 if N % 2 == 0 else N, :, :]
    for im in (raw, odd):
        names = [n for _, n, _ in IO.getWaveletImage(im, None)]
        names += [n for _, n, _ in IO.getLoGImage(im, None, sigma=[1.0, 2.0])]
    torch.cuda.synchronize()
    ri, rm = IO.resampleImage(raw.astype(np.int16), mask_rag.astype(np.uint8), resampledPixelSpacing=[1.6, 1.6, 1.6], padDistance=2)
    torch.cuda.synchronize()
    print("filters ok", len(names), "resampled", ri.array.shape, flush=True)

if "shape" in fams:
    zz, yy, xx = np.indices(mask_full.shape)
    ball = ((zz - N / 2) ** 2 + (yy - N / 2) ** 2 + (xx - N / 2) ** 2) < (N / 2.5) ** 2
    print("shape", cshape.calculate_coefficients(np.pad(ball & mask_rag, 1), (1.0, 0.8, 0.7)), flush=True)
    print("shape2D", cshape.calculate_coefficients2D(np.pad((ball & mask_rag)[N // 2], 1), (0.8, 0.7)), flush=True)

if "firstorder" in fams:
    raw = (vols["smooth"].astype(np.float64) - 1) * 25 + rng.random(mask_full.shape) * 20
    r = FC.RadiomicsFirstOrder(raw, mask_rag.astype(np.int32), voxelBased=True, binWidth=25).execute()
    print("firstorder ok", len(r), flush=True)
    # segment mode (rb_firstorder_segment_dev): 8-bit levels on the ragged ROI, 16-bit levels, a sparse ROI of 3 voxels
    sparse = np.zeros(mask_full.shape, bool)
    sparse.reshape(-1)[[0, mask_full.size // 2, mask_full.size - 1]] = True
    img_t = torch.from_numpy(raw).cuda()
    for m, bw in ((mask_rag, 25), (mask_rag, 0.05), (sparse, 25)):
        m_t = torch.from_numpy(m.astype(np.uint8)).cuda()
        _, _, lev, _, _ = voxel.discretize(img_t, m_t, binWidth=bw)
        f = voxel.firstorder_segment(img_t, lev, m_t, voxelArrayShift=10)
        print("firstorder segment ok", lev.dtype, f["Median"], flush=True)
if "lbp3d" in fams:
    raw = ((vols["smooth"] - 1) * 25 + 3).astype(np.int16)
    for kw in ({}, {"lbp3DLevels": 4, "lbp3DIcosphereRadius": 1.5, "lbp3DIcosphereSubdivision": 2}):
        names = [n for _, n, _ in IO.getLBP3DImage(raw, mask_rag.astype(np.uint8), **kw)]
    torch.cuda.synchronize()
    print("lbp3d ok", names, flush=True)
if "imagetypes" in fams:
    raw = ((vols["smooth"] - 1) * 25 - 300).astype(np.int16)
    names = []
    for img in (raw, raw[0].astype(np.uint8), raw.astype(np.float32) / 7):
        for gen in (IO.getSquareImage, IO.getSquareRootImage, IO.getLogarithmImage, IO.getExponentialImage,
                    IO.getGradientImage):
            names += [n for _, n, _ in gen(I.ArrayImage(img, (0.7, 1.1, 2.0)[:img.ndim]), None)]
    torch.cuda.synchronize()
    print("imagetypes ok", names[:5], flush=True)
if "preprocess" in fams:
    raw = ((vols["smooth"] - 1) * 25 - 300).astype(np.int16)
    kept = []
    for img in (raw, raw.astype(np.float32) / 7):
        nimg = IO.normalizeImage(I.ArrayImage(img), normalizeScale=100, removeOutliers=3)
        for rng_, mode in (([-300], "absolute"), ([0.2, 0.8], "relative"), ([-2, 2], "sigma")):
            out = IO.resegmentMask(nimg if mode == "sigma" else I.ArrayImage(img), I.ArrayImage(mask_rag.astype(np.uint8)),
                                   resegmentRange=rng_, resegmentMode=mode)
            kept.append(int((I.as_array(out) != 0).sum()))
    torch.cuda.synchronize()
    print("preprocess ok", kept, flush=True)
print("sanitize_all done")
