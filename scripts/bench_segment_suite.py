"""Segment-based first order and the segment suite on the GPU: one JSON line.

* 256^3 bench volumes (bench.synth_volume "uniform" and "smooth", raw int16 intensities (level - 1) * 25 + 3), with a full
  ROI and an ellipsoid ROI: CUDA-event time of voxel.firstorder_segment (binned once beforehand, --reps runs after a
  warm-up) next to the host path RadiomicsFirstOrder(...).execute() on the same case (one run, host clock), and the
  largest difference between the two relative to the value; once more with binWidth 1 (Ng > 255: 16-bit levels);
  for the full ROIs, the device time of each kernel from torch.profiler in a run of its own.
* pipeline.segment_suite_with_filters on bench.py's config-4 volume (smoothed float64, 256^3, ellipsoid ROI):
  original + wavelet (8) + LoG (sigma 1, 2, 3) + shape, all six classes, binWidth 25: total ms (host clock around
  work that ends in a synchronise), a per-image breakdown (original alone, the wavelet sub-bands, each LoG sigma), and
  a repeat compared bit for bit (the keys whose values differ between runs are listed).
* The card's name and power limit, before and after.

    python scripts/bench_segment_suite.py [--reps 5] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

import bench  # noqa: E402  (the bench volumes, the card's name and power limit)


def ellipsoid(n):
    g = np.meshgrid(*[np.linspace(-1, 1, n)] * 3, indexing="ij")
    return (g[0] ** 2 / 0.8 + g[1] ** 2 / 0.6 + g[2] ** 2 / 0.9) < 1


def kernel_profile(raw, lev, roi):
    """device time per kernel of one voxel.firstorder_segment call (torch.profiler, a run of its own)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from pyradiomics_b200 import voxel
    voxel.firstorder_segment(raw, lev, roi)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        voxel.firstorder_segment(raw, lev, roi)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if "seg_" in e.key:
            name = e.key.split("seg_")[1].split("(")[0]
            out[name] = {"calls": e.count, "total_us": round(e.device_time_total, 1)}
    return out


def firstorder_times(kind, roi_kind, reps, binWidth=25):
    import torch
    from pyradiomics_b200 import featureclasses as FC, image as I, voxel
    vol = bench.synth_volume(256, kind)
    raw_np = bench.raw_from_levels(vol)
    roi_np = np.ones(vol.shape, bool) if roi_kind == "full" else ellipsoid(256)
    raw = torch.from_numpy(raw_np).cuda()
    roi = torch.from_numpy(roi_np.astype(np.uint8)).cuda()
    _, _, lev, _, _ = voxel.discretize(raw, roi, binWidth=binWidth)
    got = voxel.firstorder_segment(raw, lev, roi)            # warm-up
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        again = voxel.firstorder_segment(raw, lev, roi)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
        assert all(np.float64(again[k]).tobytes() == np.float64(got[k]).tobytes() for k in got)
    t0 = time.perf_counter()
    host = FC.RadiomicsFirstOrder(I.ArrayImage(raw_np), I.ArrayImage(roi_np.astype(np.uint8)), binWidth=binWidth).execute()
    host_s = time.perf_counter() - t0
    rel = max(abs(float(got[k]) - float(v)) / max(abs(float(v)), 1e-300) for k, v in host.items())
    prof = kernel_profile(raw, lev, roi) if roi_kind == "full" else None
    return {"roi_voxels": int(roi_np.sum()), "level_bytes": voxel.level_bytes(lev), "kernels": prof, "device_ms": [round(x, 3) for x in ms], "device_ms_min": round(min(ms), 3),
            "host_execute_s": round(host_s, 3), "max_rel_diff_vs_host": rel}


def suite(reps):
    import torch
    from pyradiomics_b200 import pipeline as PL
    from bench_firstorder import config4_volume
    img = torch.as_tensor(config4_volume(256)).cuda()
    mask = torch.from_numpy(ellipsoid(256).astype(np.uint8)).cuda()
    kw = dict(binWidth=25, spacing_zyx=(1.0, 1.0, 1.0))

    def timed(**k):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = PL.segment_suite_with_filters(img, mask, **kw, **k)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, out

    timed()                                                   # warm-up of every shape
    totals, outs = [], []
    for _ in range(reps):
        t, out = timed()
        totals.append(t)
        outs.append(out)
    same_keys = all(list(o) == list(outs[0]) for o in outs[1:])
    differing = sorted({k for o in outs[1:] for k in o if np.float64(o[k]).tobytes() != np.float64(outs[0][k]).tobytes()})
    parts = {"shape": timed(classes=(), wavelet=None, sigmas=())[0],
             "original": timed(shape=False, wavelet=None, sigmas=())[0],
             "wavelet_8": timed(shape=False, sigmas=())[0] - timed(shape=False, wavelet=None, sigmas=())[0]}
    for s in (1.0, 2.0, 3.0):
        parts[f"log_sigma_{s}"] = timed(shape=False, wavelet=None, sigmas=(s,))[0] - parts["original"]
    return {"volume": "256^3 bench config-4 volume (smoothed float64), ellipsoid ROI", "features": len(outs[0]),
            "total_ms": [round(t, 1) for t in totals], "total_ms_min": round(min(totals), 1),
            "breakdown_ms": {k: round(v, 1) for k, v in parts.items()}, "repeat_same_keys": bool(same_keys),
            "repeat_bit_identical": not differing, "repeat_differing_keys": differing}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    line = {"what": "segment first order + segment suite", "gpu": bench.gpu_info(0)}
    for kind in ("uniform", "smooth"):
        for roi_kind in ("full", "ellipsoid"):
            line[f"firstorder_256_{kind}_{roi_kind}"] = firstorder_times(kind, roi_kind, args.reps)
    # binWidth 1 on the uniform volume's intensities (0..778): 32 levels 25 apart, Ng 776 -> 16-bit levels
    line["firstorder_256_uniform_full_16bit"] = firstorder_times("uniform", "full", args.reps, binWidth=1)
    line["suite_256"] = suite(args.reps)
    line["gpu_after"] = bench.gpu_info(0)
    txt = json.dumps(line)
    print(txt)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
