"""Per-class GPU time of the fused voxel kernels on the benchmark's volumes: every class (GLCM, GLRLM, GLSZM, GLDM,
NGTDM) timed with CUDA events around one whole-volume call, after warm-up, over several calls.  Prints one JSON line
(with the card's name and power limit and the library that ran; B200_RADIOMICS_LIB selects another build).

    python scripts/prof_small_classes.py [--size 256] [--kinds uniform smooth] [--reps 5] [--out FILE]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the benchmark's volume generator and card description)


def time_classes(kind, n, reps):
    import numpy as np
    import torch

    from pyradiomics_b200 import _lib, voxel

    lev = torch.as_tensor(bench.synth_volume(n, kind).astype("uint8")).cuda()
    s = _lib.make_settings(32, 32)
    res = {}
    for cname in _lib.CLASSES:
        out = voxel.voxel_features(cname, lev, s)
        for _ in range(2):
            voxel.voxel_features(cname, lev, s, out=out, out_z0=0)
        torch.cuda.synchronize()
        ms = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            voxel.voxel_features(cname, lev, s, out=out, out_z0=0)
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        res[cname] = {"ms_median": round(float(np.median(ms)), 3), "ms_min": round(min(ms), 3), "ms_max": round(max(ms), 3)}
        del out
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--kinds", nargs="+", default=["uniform", "smooth"])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also append the JSON line to this file")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        sys.exit("prof_small_classes.py needs a CUDA device")
    from pyradiomics_b200 import _lib

    line = {"what": "per-class voxel-kernel time, CUDA events, one whole-volume call each", "size": args.size,
            "reps": args.reps, "gpu": bench.gpu_info(torch.cuda.current_device()), "lib": os.path.basename(_lib.LIB_PATH)}
    for kind in args.kinds:
        line[kind] = time_classes(kind, args.size, args.reps)
    text = json.dumps(line)
    print(text)
    if args.out:
        with open(args.out, "a") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
