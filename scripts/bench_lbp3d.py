#!/usr/bin/env python
"""bench_lbp3d.py -- voxels/s of the 3-D LBP image type (imageoperations.getLBP3DImage's device step) on one GPU.

Workload: the int16 intensities of bench.py's smooth --size^3 volume (raw_from_levels(synth_volume(n, "smooth"))), a full
mask, the reference's default settings (2 levels, 42 sphere vertices of radius 1).  Prints ONE JSON line:
  value          : voxels / device-event time of imageoperations.lbp3d_device per step (float64 copy, exact B-spline
                   prefilter, per-voxel kernel -> 3 maps), median over --steps after --warmup
  gpu            : card name and power limit the number was measured under
  parity_sample  : OUTSIDE the timed region, --parity-voxels voxels from bench.sample_voxels (a quarter on faces / edges /
                   corners) against the NumPy / SciPy oracle oracle/lbp3d_np.py, with the tolerances of
                   tests/test_lbp3d_cpu.py; oracle_cpu is the oracle's one-core rate on that sample
  deterministic  : two more runs compared bit for bit with the timed one
Writes nothing to the tree.  Run from the repository root:  python scripts/bench_lbp3d.py
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

from bench import gpu_info, raw_from_levels, sample_voxels, synth_volume  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--parity-voxels", type=int, default=20480)
    args = ap.parse_args()

    import torch
    import lbp3d_np
    from pyradiomics_b200 import imageoperations as IO
    n = args.size
    raw = raw_from_levels(synth_volume(n, "smooth"))
    torch.cuda.set_device(0)
    img = torch.from_numpy(raw).cuda()
    roi = torch.ones(raw.shape, dtype=torch.uint8, device="cuda")
    for _ in range(args.warmup):
        IO.lbp3d_device(img, roi)
    torch.cuda.synchronize()
    ms = []
    for _ in range(args.steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = IO.lbp3d_device(img, roi)
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    step_ms = float(np.median(ms))
    again = [IO.lbp3d_device(img, roi) for _ in range(2)]
    deterministic = all(torch.equal(out.view(torch.int64), a.view(torch.int64)) for a in again)
    vox = sample_voxels(n, args.parity_voxels, 7)
    idx = [torch.as_tensor(v).long().cuda() for v in vox]
    got = out[:, idx[0], idx[1], idx[2]].cpu().numpy()
    del out, again
    t0 = time.perf_counter()
    coef = lbp3d_np.prefilter(raw)
    t1 = time.perf_counter()
    o = lbp3d_np.lbp3d(raw, None, IO._icosphere(1, 1.0), 2, 1.0, coef=coef, coords=vox)
    t2 = time.perf_counter()
    ref = o["maps"]
    bad = np.zeros(vox.shape[1], bool)
    for lv in range(2):                              # the tolerances of tests/test_lbp3d_cpu.py
        bad |= ~np.isclose(got[lv], ref[lv], rtol=1e-12, atol=1e-12 * max(float(np.nanmax(np.abs(ref[lv]))), 1.0))
    bad |= np.isnan(got[2]) != np.isnan(ref[2])
    settled = ~np.isnan(ref[2]) & (o["m2"] > 1e3 * (np.finfo(np.float64).eps * o["mean"]) ** 2)
    bad |= settled & ~np.isclose(got[2], ref[2], rtol=1e-10, atol=1e-10)
    line = {
        "metric": "voxels/s lbp3d image type", "value": n ** 3 / (step_ms * 1e-3), "unit": "voxels/s", "n_gpus": 1,
        "gpu": gpu_info(0), "steps": args.steps, "warmup": args.warmup, "ms_per_step": step_ms, "ms_all_steps": ms,
        "higher_is_better": True, "dtype": "f64",
        "config": {"volume": f"raw_from_levels(synth_volume({n}, 'smooth')), int16, full mask",
                   "settings": {"lbp3DLevels": 2, "lbp3DIcosphereRadius": 1, "lbp3DIcosphereSubdivision": 1},
                   "step": "imageoperations.lbp3d_device: float64 copy, exact B-spline prefilter, per-voxel kernel -> 3 maps"},
        "parity_sample": {"voxels": int(vox.shape[1]), "outside_tolerance": int(bad.sum()),
                          "nan_kurtosis": int(np.isnan(ref[2]).sum()),
                          "oracle": "oracle/lbp3d_np.py (scipy.ndimage.map_coordinates, scipy.stats.kurtosis, sph_harm_y)",
                          "tolerance": "level maps 1e-12 relative, kurtosis 1e-10 where m2 is not near zero, NaN positions"},
        "oracle_cpu": {"voxels_per_s": vox.shape[1] / (t2 - t1), "prefilter_s": t1 - t0, "cores": 1,
                       "note": "NumPy / SciPy restatement on the sample, whole-volume spline prefilter timed apart"},
        "deterministic": bool(deterministic),
    }
    print(json.dumps(line))


if __name__ == "__main__":
    main()
