"""GLCM's Lanczos eigen-solve launches (glcm_fast_solve_kernel<2>, one launch per size group 18 / 16 / 14 and queue
chunk) on the benchmark volumes: per-launch GPU time from torch.profiler (CUDA activities, in a run of its own), the
eigen-task count per size group (host count of phase A's rule, tests/mcc_class.py, on a random sample of centres scaled
to the volume), and what the GLCM maps of each build are, so builds can be compared value for value.

Each build named by --libs NAME=PATH runs in its own process (B200_RADIOMICS_LIB selects it), the builds alternating for
--rounds rounds.  Prints one JSON line per build and round and, with two or more builds, one comparison line: the largest
|MCC| difference against the first build and whether the other 23 GLCM maps are bit-identical.

    python scripts/prof_glcm_lanczos.py [--size 256] [--kinds uniform smooth] [--steps 3] [--rounds 2]
                                        [--libs parent=PATH pr=PATH] [--out FILE]
"""
import argparse
import collections
import hashlib
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the benchmark's volume generator and card description)

GROUPS = (18, 16, 14)          # glcm_fast_run launches the Lanczos size groups in this order in every chunk


def group_of(nlev):
    return 14 if nlev <= 14 else 16 if nlev <= 16 else 18


def task_counts(kind, n, sample, seed=0):
    """eigen-tasks per size group of the Lanczos kind (13..18 levels; only the three axis angles reach them), from a host
    count over `sample` random centres, scaled to the n^3 volume"""
    import numpy as np

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import mcc_class as M

    lev = bench.synth_volume(n, kind)
    rng = np.random.default_rng(seed)
    cen = rng.integers(0, n, (sample, 3))
    W = M.windows_of(lev, cen)
    cnt = collections.Counter()
    for slot in range(3):
        cls, nlev, _, _ = M.classify(W, slot)
        for g in GROUPS:
            cnt[g] += int(((cls == M.TASK) & (nlev >= 13) & (np.vectorize(group_of)(nlev) == g)).sum())
    scale = n ** 3 / sample
    return {str(g): {"per_voxel": round(cnt[g] / sample, 4), "per_volume": int(round(cnt[g] * scale))} for g in GROUPS}


def one_build(kind, n, steps, dump):
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
    evs = sorted((ev for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA
                  and "glcm_fast_solve_kernel<2>" in ev.name), key=lambda ev: ev.time_range.start)
    per_launch = [ev.device_time / 1e3 for ev in evs]            # us -> ms, in launch order
    nl = len(per_launch) // steps
    per_group = collections.defaultdict(float)
    for i, t in enumerate(per_launch):
        per_group[GROUPS[i % len(GROUPS)]] += t / steps
    first = per_launch[:nl]                                     # the launches of one volume: [chunk][group]
    res = {"lanczos_ms_per_volume": round(sum(per_launch) / steps, 3),
           "ms_per_group": {str(g): round(per_group[g], 3) for g in GROUPS},
           "ms_per_launch_first_volume": [round(t, 3) for t in first], "launches_per_volume": nl}
    names = _lib.feature_names("glcm")
    mcc_i = names.index("MCC")
    h = hashlib.sha256()
    for k in range(len(names)):
        if k != mcc_i:
            h.update(out[k].cpu().numpy().tobytes())
    res["sha256_other_maps"] = h.hexdigest()
    if dump:
        import numpy as np

        np.save(dump, out[mcc_i].cpu().numpy())
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--kinds", nargs="+", default=["uniform", "smooth"])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--sample", type=int, default=40000)
    ap.add_argument("--libs", nargs="*", default=[], metavar="NAME=PATH")
    ap.add_argument("--one", nargs=2, metavar=("KIND", "DUMP"), help=argparse.SUPPRESS)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        sys.exit("prof_glcm_lanczos.py needs a CUDA device")
    if args.one:
        print(json.dumps(one_build(args.one[0], args.size, args.steps, args.one[1] or None)))
        return
    libs = [tuple(x.split("=", 1)) for x in args.libs] or [("this", "")]
    gpu = bench.gpu_info(torch.cuda.current_device())
    lines = []
    with tempfile.TemporaryDirectory() as tmp:
        for kind in args.kinds:
            counts = task_counts(kind, args.size, args.sample)
            for r in range(args.rounds):
                for name, path in libs:
                    env = dict(os.environ)
                    if path:
                        env["B200_RADIOMICS_LIB"] = os.path.abspath(path)
                    dump = os.path.join(tmp, f"{kind}_{name}.npy") if r == 0 else ""
                    p = subprocess.run([sys.executable, os.path.abspath(__file__), "--size", str(args.size), "--steps",
                                        str(args.steps), "--one", kind, dump], env=env, capture_output=True, text=True)
                    if p.returncode:
                        sys.exit(p.stderr[-3000:])
                    res = json.loads(p.stdout.strip().splitlines()[-1])
                    lines.append({"what": "GLCM Lanczos launches (glcm_fast_solve_kernel<2>), torch.profiler", "size": args.size,
                                  "kind": kind, "round": r, "build": name, "gpu": gpu, "steps": args.steps,
                                  "tasks_per_group_host_count": counts, **res})
                    print(json.dumps(lines[-1]), flush=True)
            if len(libs) > 1:
                import numpy as np

                base = np.load(os.path.join(tmp, f"{kind}_{libs[0][0]}.npy"))
                for name, _ in libs[1:]:
                    other = np.load(os.path.join(tmp, f"{kind}_{name}.npy"))
                    same_nan = bool(np.array_equal(np.isnan(base), np.isnan(other)))
                    d = np.abs(base - other)
                    sh = {ln["build"]: ln["sha256_other_maps"] for ln in lines if ln["kind"] == kind and ln.get("round") == 0}
                    lines.append({"what": f"GLCM maps of {name} against {libs[0][0]}", "kind": kind,
                                  "mcc_max_abs_diff": float(np.nanmax(d)), "mcc_voxels_differing": int((d > 0).sum()),
                                  "mcc_nan_mask_equal": same_nan,
                                  "other_23_maps_bit_identical": sh.get(name) == sh.get(libs[0][0])})
                    print(json.dumps(lines[-1]), flush=True)
    if args.out:
        with open(args.out, "a") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
