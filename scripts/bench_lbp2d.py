#!/usr/bin/env python
"""bench_lbp2d.py -- time of the 2-D LBP image type (imageoperations.getLBP2DImage) on one GPU.

Workload: the int16 intensities of bench.py's smooth --size^3 volume (raw_from_levels(synth_volume(n, "smooth"))), sliced
along axis 0, in two settings: lbp2DMethod 'uniform' with P = 8, R = 1 (the reference's defaults) and 'default' with
P = 24, R = 3.  Prints ONE JSON line; per setting:
  device_ms       : CUDA-event time of imageoperations.lbp2d_device (one rb_lbp2d_dev launch), median over --steps calls
                    after --warmup; axis2_device_ms the same with the slices cut along x (columns = z)
  bytes, gb_per_s : the ideal traffic, the int16 read once (2 B) and the float64 written once (8 B) per voxel, over
                    device_ms; floor_ms is that traffic at the data sheet's 3.35 TB/s
  generator_ms    : wall time of the whole getLBP2DImage on the NumPy volume (upload, kernel, download, the per-slice cast
                    to int16 on the host), median over --gen-steps
  parity_planes   : OUTSIDE the timed region, --planes planes compared bit for bit with the NumPy oracle
                    oracle/lbp2d_np.py (NaN positions identical)
  deterministic   : two more device runs compared bit for bit with the timed one
  gpu             : card name and power limit, read in the same run
Writes nothing to the tree.  Run from the repository root:  python scripts/bench_lbp2d.py
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

HBM_TB_S = 3.35                                    # H100 SXM5 80 GB data sheet


def device_ms(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return float(np.median(ms)), ms, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--gen-steps", type=int, default=5)
    ap.add_argument("--planes", type=int, default=3)
    args = ap.parse_args()

    import torch
    import lbp2d_np
    from pyradiomics_b200 import imageoperations as IO
    n = args.size
    raw = raw_from_levels(synth_volume(n, "smooth"))
    assert raw.dtype == np.int16
    torch.cuda.set_device(0)
    img = torch.from_numpy(raw).cuda()
    nbytes = raw.size * (raw.itemsize + 8)
    planes = np.linspace(0, n - 1, args.planes).round().astype(int)
    results = {}
    for method, P, R in [("uniform", 8, 1), ("default", 24, 3)]:
        run = lambda axis=0: IO.lbp2d_device(img, axis, P, R, method)        # noqa: E731
        ms, all_ms, out = device_ms(run, args.steps, args.warmup)
        ms2, _, _ = device_ms(lambda: run(2), args.steps, args.warmup)
        again = [run() for _ in range(2)]
        deterministic = all(torch.equal(out.view(torch.int64), a.view(torch.int64)) for a in again)
        got = out[torch.as_tensor(planes).cuda()].cpu().numpy()
        del out, again
        gen = []
        for _ in range(args.gen_steps):
            t0 = time.perf_counter()
            (im, _, _), = IO.getLBP2DImage(raw, None, lbp2DSamples=P, lbp2DRadius=R, lbp2DMethod=method, force2D=True)
            gen.append((time.perf_counter() - t0) * 1e3)
        t0 = time.perf_counter()
        ref = np.stack([lbp2d_np.local_binary_pattern(raw[p], P, R, method) for p in planes])
        t_oracle = time.perf_counter() - t0
        same = np.array_equal(np.isnan(got), np.isnan(ref)) and \
            np.array_equal(np.where(np.isnan(got), 0, got).view(np.int64), np.where(np.isnan(ref), 0, ref).view(np.int64))
        results[f"{method}_P{P}_R{R}"] = {
            "device_ms": ms, "device_ms_all": all_ms, "axis2_device_ms": ms2, "bytes": nbytes,
            "gb_per_s": nbytes / (ms * 1e-3) / 1e9, "floor_ms": nbytes / (HBM_TB_S * 1e12) * 1e3,
            "generator_ms": float(np.median(gen)), "generator_ms_all": gen,
            "parity_planes": {"planes": planes.tolist(), "bit_identical": bool(same),
                              "oracle": "oracle/lbp2d_np.py (NumPy restatement of skimage local_binary_pattern)",
                              "oracle_cpu_s_per_plane": t_oracle / len(planes)},
            "deterministic": bool(deterministic),
        }
    head = results["uniform_P8_R1"]
    line = {
        "metric": "ms lbp2d image type (uniform, P 8, R 1, axis 0)", "value": head["device_ms"], "unit": "ms", "n_gpus": 1,
        "gpu": gpu_info(0), "steps": args.steps, "warmup": args.warmup, "higher_is_better": False, "dtype": "f64",
        "config": {"volume": f"raw_from_levels(synth_volume({n}, 'smooth')), int16",
                   "step": "imageoperations.lbp2d_device: one rb_lbp2d_dev launch, every slice -> float64 volume",
                   "ideal_traffic": "2 B read + 8 B written per voxel", "hbm_tb_per_s": HBM_TB_S},
        "runs": results,
    }
    print(json.dumps(line))


if __name__ == "__main__":
    main()
