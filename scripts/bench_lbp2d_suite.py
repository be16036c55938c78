#!/usr/bin/env python
"""bench_lbp2d_suite.py -- the 2-D LBP image type inside the device-resident voxel suite on one GPU.

Workload: the int16 intensities of bench.py's smooth --size^3 volume (raw_from_levels(synth_volume(n, "smooth"))), the
whole volume as ROI, getLBP2DImage's defaults (uniform, P = 8, R = 1, slices along axis 0).  Prints ONE JSON line:
  cast_kernel_ms     : CUDA-event time of imageoperations.lbp2d_device(out_dtype=int16) (one rb_lbp2d_cast_dev launch,
                       the codes stored as int16), median over --steps calls after --warmup; float64_kernel_ms the same for
                       rb_lbp2d_dev's float64 volume, in the same run
  bytes, gb_per_s    : the ideal traffic of the cast kernel, the int16 read once and written once (4 B per voxel)
  host_path_ms       : wall time of getLBP2DImage on the NumPy volume followed by the upload of its int16 result (what a
                       suite caller did before), median over --gen-steps
  suite_ms           : wall time (ending in a synchronise) of pipeline.voxel_suite_with_filters(wavelet=None, sigmas=(),
                       lbp2d={}), binCount 10 (the ten
                       uniform codes, one level each), the five texture classes: 'original' then 'lbp-2D', median over --suite-steps
                       after one warm-up run
  parity             : OUTSIDE the timed region, the cast kernel's volume against getLBP2DImage's, bit for bit
  deterministic      : a repeat suite run's lbp-2D maps against the first run's, bit for bit
  gpu                : card name and power limit, read in the same run
Writes nothing to the tree.  Run from the repository root:  python scripts/bench_lbp2d_suite.py
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "scripts")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench import gpu_info, raw_from_levels, synth_volume  # noqa: E402
from bench_lbp2d import device_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--gen-steps", type=int, default=5)
    ap.add_argument("--suite-steps", type=int, default=3)
    args = ap.parse_args()

    import torch
    from pyradiomics_b200 import image as I, imageoperations as IO, pipeline as PL
    n = args.size
    raw = raw_from_levels(synth_volume(n, "smooth"))
    assert raw.dtype == np.int16
    torch.cuda.set_device(0)
    img = torch.from_numpy(raw).cuda()
    mask = torch.ones(img.shape, dtype=torch.uint8, device=img.device)

    cast_ms, cast_all, out = device_ms(lambda: IO.lbp2d_device(img, 0, 8, 1, "uniform", out_dtype=torch.int16),
                                       args.steps, args.warmup)
    f64_ms, _, _ = device_ms(lambda: IO.lbp2d_device(img, 0, 8, 1, "uniform"), args.steps, args.warmup)

    host = []
    for _ in range(args.gen_steps):
        t0 = time.perf_counter()
        (im, _, _), = IO.getLBP2DImage(raw, None)
        up = IO._to_device(I.as_array(im))
        torch.cuda.synchronize()
        host.append((time.perf_counter() - t0) * 1e3)
    parity = bool(torch.equal(out, up))
    del out, up

    first = {}

    def keep(name, cls, maps):
        if name == "lbp-2D":
            first[cls] = maps.clone()
    same = []

    def compare(name, cls, maps):
        if name == "lbp-2D":
            same.append(torch.equal(first[cls].view(torch.int64), maps.view(torch.int64)))

    def suite(consume=None):
        return PL.voxel_suite_with_filters(img, mask, wavelet=None, sigmas=(), lbp2d={}, consume=consume, binCount=10)

    info = suite(keep)
    torch.cuda.synchronize()
    suite_all = []
    for _ in range(args.suite_steps):
        t0 = time.perf_counter()
        suite()
        torch.cuda.synchronize()
        suite_all.append((time.perf_counter() - t0) * 1e3)
    suite(compare)
    torch.cuda.synchronize()

    nbytes = raw.size * 4
    line = {
        "metric": "ms lbp2d cast kernel (uniform, P 8, R 1, axis 0, int16 out)", "value": cast_ms, "unit": "ms", "n_gpus": 1,
        "gpu": gpu_info(0), "steps": args.steps, "warmup": args.warmup, "higher_is_better": False, "dtype": "i16",
        "config": {"volume": f"raw_from_levels(synth_volume({n}, 'smooth')), int16, ROI = every voxel",
                   "cast_step": "imageoperations.lbp2d_device(out_dtype=torch.int16): one rb_lbp2d_cast_dev launch",
                   "suite": "pipeline.voxel_suite_with_filters(wavelet=None, sigmas=(), lbp2d={}, binCount=10), "
                            "glcm glrlm glszm gldm ngtdm, float64 maps",
                   "ideal_traffic": "2 B read + 2 B written per voxel"},
        "cast_kernel_ms": cast_ms, "cast_kernel_ms_all": cast_all, "float64_kernel_ms": f64_ms, "bytes": nbytes,
        "gb_per_s": nbytes / (cast_ms * 1e-3) / 1e9,
        "host_path_ms": float(np.median(host)), "host_path_ms_all": host,
        "suite_ms": float(np.median(suite_all)), "suite_ms_all": suite_all,
        "suite_images": [{"name": nm, "Ng": ng, "levels": nl} for nm, ng, nl in info],
        "parity": {"cast_kernel_vs_getLBP2DImage": parity},
        "deterministic": bool(same) and all(same),
    }
    print(json.dumps(line))


if __name__ == "__main__":
    main()
