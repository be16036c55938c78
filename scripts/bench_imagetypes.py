#!/usr/bin/env python
"""bench_imagetypes.py -- the square, squareroot, logarithm, exponential and gradient image types on one GPU.

Workload: the int16 intensities of bench.py's smooth --size^3 volume (raw_from_levels(synth_volume(n, "smooth"))), 1 mm
isotropic spacing.  A step is what pipeline.derived_images(image_types=<all five>) runs: one max|x| reduction
(imageoperations.image_max_abs, shared by the four per-voxel types) and the five filters, each writing a float64 image.
Prints ONE JSON line:
  ms_per_step / value : device-event time of the whole step (median over --steps after --warmup), voxels / that time
  per_type           : per filter (and the reduction) the median event time, voxels/s, the bytes it has to move
                       (computed from the shapes: the input read once, the float64 output written once) and the
                       resulting GB/s against the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s, not a measured peak)
  gpu                : card name and power limit the number was measured under
  parity             : OUTSIDE the timed region, every voxel of the last step's five images against the NumPy oracle
                       oracle/imagetypes_np.py with the tolerances of tests/test_imagetypes_gpu.py (square, squareroot,
                       gradient bit for bit; logarithm, exponential 1e-15 relative; NaN positions identical)
  deterministic      : two more steps compared bit for bit with the timed one
Writes nothing to the tree.  Run from the repository root:  python scripts/bench_imagetypes.py
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

from bench import gpu_info, raw_from_levels, synth_volume  # noqa: E402

TYPES = ("square", "squareroot", "logarithm", "exponential", "gradient")
HBM_DATASHEET_GBS = 3350.0
SPACING_ZYX = (1.0, 1.0, 1.0)


def step(IO, x, torch):
    """the five images plus event stamps: [start, after the reduction, after each type]"""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(TYPES) + 2)]
    ev[0].record()
    m = IO.image_max_abs(x)
    ev[1].record()
    out = {}
    for k, t in enumerate(TYPES):
        out[t] = IO.gradient_magnitude_device(x, SPACING_ZYX) if t == "gradient" else IO.pointwise_image_device(x, t, m)
        ev[k + 2].record()
    return out, ev


def outside_tolerance(got, ref, kind):
    nan_ref, nan_got = np.isnan(ref), np.isnan(got)
    bad = nan_ref != nan_got
    both = ~nan_ref & ~nan_got
    if kind in ("logarithm", "exponential"):
        bad[both] |= ~np.isclose(got[both], ref[both], rtol=1e-15, atol=0)
    else:
        bad[both] |= (got[both] != ref[both]) | (np.signbit(got[both]) != np.signbit(ref[both]))
    return int(bad.sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import torch
    import imagetypes_np as O
    from pyradiomics_b200 import imageoperations as IO
    n = args.size
    raw = raw_from_levels(synth_volume(n, "smooth"))
    nvox = raw.size
    torch.cuda.set_device(0)
    x = torch.from_numpy(raw).cuda()
    for _ in range(args.warmup):
        step(IO, x, torch)
    torch.cuda.synchronize()
    total, per = [], {k: [] for k in ("max_abs",) + TYPES}
    for _ in range(args.steps):
        out, ev = step(IO, x, torch)
        ev[-1].synchronize()
        total.append(ev[0].elapsed_time(ev[-1]))
        per["max_abs"].append(ev[0].elapsed_time(ev[1]))
        for k, t in enumerate(TYPES):
            per[t].append(ev[k + 1].elapsed_time(ev[k + 2]))
    step_ms = float(np.median(total))
    again = [step(IO, x, torch)[0] for _ in range(2)]
    deterministic = all(torch.equal(out[t].view(torch.int64), a[t].view(torch.int64)) for a in again for t in TYPES)
    got = {t: out[t].cpu().numpy() for t in TYPES}
    del out, again

    t0 = time.perf_counter()
    ref = {t: O.gradient(raw, SPACING_ZYX) if t == "gradient" else O.pointwise(raw, t) for t in TYPES}
    oracle_s = time.perf_counter() - t0
    bad = {t: outside_tolerance(got[t], ref[t], t) for t in TYPES}

    item = raw.dtype.itemsize
    nbytes = {"max_abs": nvox * item, **{t: nvox * (item + 8) for t in TYPES}}
    per_type = {}
    for k, v in per.items():
        ms = float(np.median(v))
        per_type[k] = {"ms": ms, "voxels_per_s": nvox / (ms * 1e-3), "bytes": nbytes[k],
                       "achieved_GBps": nbytes[k] / (ms * 1e-3) / 1e9,
                       "fraction_of_datasheet_hbm": nbytes[k] / (ms * 1e-3) / 1e9 / HBM_DATASHEET_GBS}
    all_bytes = sum(nbytes.values())
    line = {
        "metric": "voxels/s square+squareroot+logarithm+exponential+gradient image types", "value": nvox / (step_ms * 1e-3),
        "unit": "voxels/s", "n_gpus": 1, "gpu": gpu_info(0), "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": step_ms, "ms_all_steps": total, "higher_is_better": True, "dtype": "f64",
        "config": {"volume": f"raw_from_levels(synth_volume({n}, 'smooth')), int16", "spacing_zyx": SPACING_ZYX,
                   "step": "imageoperations.image_max_abs (one rb_minmax_dev + a 32-byte copy to the host), then "
                           "pointwise_image_device x 4 and gradient_magnitude_device -> five float64 images"},
        "per_type": per_type,
        "bytes_per_step": all_bytes, "achieved_GBps": all_bytes / (step_ms * 1e-3) / 1e9,
        "hbm_datasheet": {"GBps": HBM_DATASHEET_GBS, "note": "H100 SXM data-sheet HBM3 bandwidth, not measured here",
                          "floor_ms": all_bytes / (HBM_DATASHEET_GBS * 1e9) * 1e3,
                          "fraction": all_bytes / (step_ms * 1e-3) / 1e9 / HBM_DATASHEET_GBS},
        "parity": {"voxels_per_type": nvox, "outside_tolerance": bad, "outside_tolerance_total": sum(bad.values()),
                   "oracle": "oracle/imagetypes_np.py (NumPy, whole volume)",
                   "tolerance": "square, squareroot, gradient bit for bit; logarithm, exponential 1e-15 relative; "
                                "NaN positions identical"},
        "oracle_cpu": {"s": oracle_s, "voxels_per_s": nvox / oracle_s, "cores": 1,
                       "note": "the NumPy restatement of all five types on the whole volume"},
        "deterministic": bool(deterministic),
    }
    print(json.dumps(line))


if __name__ == "__main__":
    main()
