"""Per-kernel GPU time of the fused GLCM path on the benchmark volumes: phase A (glcm_fast_kernel), every phase-B
solve launch (glcm_fast_solve_kernel<KIND>, one launch per size group) and the finish kernel, from torch.profiler with
CUDA activities in a run of its own.  Prints one JSON line (with the card's name and power limit).

    python scripts/prof_glcm_phases.py [--size 256] [--kinds uniform smooth] [--steps 3] [--out FILE]
"""
import argparse
import collections
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the benchmark's volume generator and card description)


def phase_of(name):
    if "glcm_fast_kernel" in name:
        return "phaseA"
    m = re.search(r"glcm_fast_solve_kernel<(\d)>", name)
    if m:
        return f"solve{m.group(1)}"
    if "glcm_fast_finish_kernel" in name:
        return "finish"
    return None


def profile(kind, n, steps):
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile

    from pyradiomics_b200 import _lib, voxel

    lev = torch.as_tensor(bench.synth_volume(n, kind).astype("uint8")).cuda()
    s = _lib.make_settings(32, 32)
    out = voxel.voxel_features("glcm", lev, s)
    for _ in range(2):
        voxel.voxel_features("glcm", lev, s, out=out, out_z0=0)
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            voxel.voxel_features("glcm", lev, s, out=out, out_z0=0)
        torch.cuda.synchronize()
    per = collections.defaultdict(float)
    launches = collections.Counter()
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        ph = phase_of(ev.name)
        if ph is None:
            continue
        per[ph] += ev.device_time / 1e3            # us -> ms
        launches[ph] += 1
    res = {k: round(v / steps, 3) for k, v in sorted(per.items())}
    res["total"] = round(sum(per.values()) / steps, 3)
    return {"ms_per_volume": res, "launches_per_volume": {k: v // steps for k, v in sorted(launches.items())}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--kinds", nargs="+", default=["uniform", "smooth"])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also append the JSON line to this file")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        sys.exit("prof_glcm_phases.py needs a CUDA device")
    from pyradiomics_b200 import _lib

    line = {"what": "GLCM per-kernel time, torch.profiler (CUDA activities)", "size": args.size, "steps": args.steps,
            "gpu": bench.gpu_info(torch.cuda.current_device()), "lib": os.path.basename(_lib.LIB_PATH)}
    for kind in args.kinds:
        line[kind] = profile(kind, args.size, args.steps)
    text = json.dumps(line)
    print(text)
    if args.out:
        with open(args.out, "a") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
