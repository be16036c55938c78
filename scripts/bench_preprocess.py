#!/usr/bin/env python
"""bench_preprocess.py -- image normalisation and mask resegmentation on one GPU.

Workload: the int16 intensities of bench.py's smooth --size^3 volume (raw_from_levels(synth_volume(n, "smooth"))) and
an ellipsoid ROI of about half the volume (uint8 mask).  Three steps, each timed by device events around the whole
call (they end in a small device-to-host copy, so the host waits for the device):
  normalize        imageoperations.normalize_image_device(x, scale=100, outliers=3): the two-pass whole-image moments
                   (rb_roi_moments_dev), then rb_normalize_dev writing a float64 image
  resegment_sigma  resegment_mask_device(x, roi, [-3, 3], "sigma"): two-pass ROI moments, then rb_resegment_dev
  resegment_rel    resegment_mask_device(x, roi, [0.2, 0.8], "relative"): one-pass ROI maximum, then rb_resegment_dev
Prints ONE JSON line:
  ms_per_step / value : the three steps together (median over --steps after --warmup), voxels / that time
  per_step            : per step the median event time, the bytes it has to move (computed from the shapes: every pass
                        reads the image, and the mask where there is one; the output is written once) and the resulting
                        GB/s against the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s, not a measured peak)
  gpu                 : card name and power limit the number was measured under
  parity              : OUTSIDE the timed region, every voxel against oracle/preprocess_np.py: the normalised image bit for
                        bit given the device's statistics, each resegmented mask voxel for voxel with NumPy's own
                        statistics
  deterministic       : two more steps compared bit for bit with the timed one
Writes nothing to the tree.  Run from the repository root:  python scripts/bench_preprocess.py
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

HBM_DATASHEET_GBS = 3350.0
STEPS = ("normalize", "resegment_sigma", "resegment_rel")
RESEGMENT = {"resegment_sigma": ([-3, 3], "sigma"), "resegment_rel": ([0.2, 0.8], "relative")}


def ellipsoid(n):
    z, y, x = np.ogrid[:n, :n, :n]
    c = (n - 1) / 2
    return ((((z - c) / (0.45 * n)) ** 2 + ((y - c) / (0.4 * n)) ** 2 + ((x - c) / (0.5 * n)) ** 2) <= 1).astype(np.uint8)


def step(IO, x, roi, torch):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(STEPS) + 1)]
    ev[0].record()
    out = {"normalize": IO.normalize_image_device(x, 100, 3)}
    ev[1].record()
    for k, name in enumerate(STEPS[1:]):
        rng, mode = RESEGMENT[name]
        out[name] = IO.resegment_mask_device(x, roi, rng, mode)[0]
        ev[k + 2].record()
    return out, ev


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import torch
    import preprocess_np as O
    from pyradiomics_b200 import imageoperations as IO
    n = args.size
    raw = raw_from_levels(synth_volume(n, "smooth"))
    mask = ellipsoid(n)
    nvox, nroi = raw.size, int(mask.sum())
    torch.cuda.set_device(0)
    x, roi = torch.from_numpy(raw).cuda(), torch.from_numpy(mask).cuda()
    for _ in range(args.warmup):
        step(IO, x, roi, torch)
    torch.cuda.synchronize()
    total, per = [], {k: [] for k in STEPS}
    for _ in range(args.steps):
        out, ev = step(IO, x, roi, torch)
        ev[-1].synchronize()
        total.append(ev[0].elapsed_time(ev[-1]))
        for k, name in enumerate(STEPS):
            per[name].append(ev[k].elapsed_time(ev[k + 1]))
    step_ms = float(np.median(total))
    again = [step(IO, x, roi, torch)[0] for _ in range(2)]
    deterministic = all(torch.equal(out[k].view(torch.uint8), a[k].view(torch.uint8)) for a in again for k in STEPS)
    _, _, mean, std, _ = IO.roi_moments_device(x, ddof=1)
    got = {k: out[k].cpu().numpy() for k in STEPS}
    del out, again

    t0 = time.perf_counter()
    ref = {"normalize": O.normalize(raw, 100, 3, stats=(mean, std))}
    for name, (rng, mode) in RESEGMENT.items():
        ref[name] = O.resegment(raw, mask, rng, mode)[0]
    oracle_s = time.perf_counter() - t0
    g, r = got["normalize"], ref["normalize"]
    bad = {"normalize": int(((g.view(np.int64) != r.view(np.int64)) & ~(np.isnan(g) & np.isnan(r))).sum())}
    for name in RESEGMENT:
        bad[name] = int((got[name].astype(bool) != ref[name]).sum())

    item = raw.dtype.itemsize
    nbytes = {"normalize": nvox * (2 * item + item + 8),                       # two reduction passes, read + write
              "resegment_sigma": nvox * (2 * (item + 1) + item + 1 + 1),       # two masked passes, masked threshold
              "resegment_rel": nvox * ((item + 1) + item + 1 + 1)}             # one masked pass, masked threshold
    per_step = {}
    for k, v in per.items():
        ms = float(np.median(v))
        per_step[k] = {"ms": ms, "voxels_per_s": nvox / (ms * 1e-3), "bytes": nbytes[k],
                       "bytes_per_voxel": nbytes[k] / nvox, "achieved_GBps": nbytes[k] / (ms * 1e-3) / 1e9,
                       "datasheet_floor_ms": nbytes[k] / (HBM_DATASHEET_GBS * 1e9) * 1e3,
                       "fraction_of_datasheet_hbm": nbytes[k] / (ms * 1e-3) / 1e9 / HBM_DATASHEET_GBS}
    all_bytes = sum(nbytes.values())
    line = {
        "metric": "voxels/s normalisation + sigma and relative resegmentation", "value": nvox / (step_ms * 1e-3),
        "unit": "voxels/s", "n_gpus": 1, "gpu": gpu_info(0), "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": step_ms, "ms_all_steps": total, "higher_is_better": True,
        "config": {"volume": f"raw_from_levels(synth_volume({n}, 'smooth')), int16",
                   "roi": f"ellipsoid, {nroi} of {nvox} voxels",
                   "normalize": {"normalizeScale": 100, "removeOutliers": 3},
                   "resegment": {k: {"resegmentRange": v[0], "resegmentMode": v[1]} for k, v in RESEGMENT.items()}},
        "per_step": per_step,
        "bytes_per_step": all_bytes, "achieved_GBps": all_bytes / (step_ms * 1e-3) / 1e9,
        "hbm_datasheet": {"GBps": HBM_DATASHEET_GBS, "note": "H100 SXM data-sheet HBM3 bandwidth, not measured here",
                          "floor_ms": all_bytes / (HBM_DATASHEET_GBS * 1e9) * 1e3,
                          "fraction": all_bytes / (step_ms * 1e-3) / 1e9 / HBM_DATASHEET_GBS},
        "parity": {"voxels_per_step": nvox, "outside_tolerance": bad, "outside_tolerance_total": sum(bad.values()),
                   "oracle": "oracle/preprocess_np.py (NumPy, whole volume)",
                   "tolerance": "normalised image bit for bit given the device's mean / std (NaN positions identical); "
                                "resegmented masks equal, the oracle using NumPy's own ROI statistics"},
        "oracle_cpu": {"s": oracle_s, "voxels_per_s": 3 * nvox / oracle_s, "cores": 1,
                       "note": "the NumPy restatement of the three steps on the whole volume"},
        "deterministic": bool(deterministic),
    }
    print(json.dumps(line))


if __name__ == "__main__":
    main()
