"""GLCM phase A's MCC classification on the benchmark volumes: how many level graphs still need the connectivity sweep,
and what phase A costs with each library build.

Two parts, each printing one JSON line (appended to --out if given):

* ``--counts`` (CPU only): per angle group (3 axes, 6 face diagonals, 4 body diagonals) of the full-window voxels, the
  share of (voxel, angle) level graphs, and of warps (32 consecutive voxels of a row, as the phase-A kernel maps them),
  that enter the sweep -- before the distinct-edge count (every graph with two or more levels) and after it (only graphs
  with at least nlev distinct level pairs: fewer leave a disconnected graph or a tree).
* ``--libs NAME=PATH ...`` (GPU): phase-A time per volume (torch.profiler, CUDA activities, the same harness as
  prof_glcm_phases.py) for each library build, alternated over --rounds rounds, each run in a fresh process
  (B200_RADIOMICS_LIB selects the build), with a SHA-256 over the raw bytes of the 24 float64 GLCM maps of every volume.

    python scripts/prof_glcm_mcc_class.py --counts [--size 256]
    python scripts/prof_glcm_mcc_class.py --libs parent=/path/a.so this=pyradiomics_b200/libb200radiomics.so [--rounds 3]
"""
import argparse
import collections
import hashlib
import itertools
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402

import bench  # noqa: E402  (the benchmark's volume generator and card description)

GROUPS = ("axis", "face", "body")


def angle_offsets():
    """the 13 distance-1 angles, grouped by the number of moving dimensions (phase A's slot order)"""
    angs = [a for a in itertools.product((1, 0, -1), repeat=3)][:13]
    return {g: [a for a in angs if sum(c != 0 for c in a) == k] for k, g in zip((1, 2, 3), GROUPS)}


def sweep_counts(lev):
    """per group: graphs / warps of full-window voxels that enter the sweep with and without the distinct-edge count"""
    Z, Y, X = lev.shape
    assert X % 32 == 0
    lev = lev.astype(np.int64)
    res = {}
    for g, angs in angle_offsets().items():
        c = collections.Counter()
        for z in range(1, Z - 1):
            # level pairs of every window centred on plane z (interior rows and columns: the full-window voxels)
            before = np.zeros((len(angs), Y, X), bool)
            after = np.zeros((len(angs), Y, X), bool)
            for k, (dz, dy, dx) in enumerate(angs):
                ends, codes = [], []
                for wz, wy, wx in itertools.product(range(-1, 2), repeat=3):
                    qz, qy, qx = wz + dz, wy + dy, wx + dx
                    if max(abs(qz), abs(qy), abs(qx)) > 1:
                        continue
                    a = lev[z + wz, 1 + wy:Y - 1 + wy, 1 + wx:X - 1 + wx]
                    b = lev[z + qz, 1 + qy:Y - 1 + qy, 1 + qx:X - 1 + qx]
                    ends.append((np.int64(1) << a) | (np.int64(1) << b))
                    codes.append(np.minimum(a, b) * 256 + np.maximum(a, b))
                nlev = np.bitwise_count(np.bitwise_or.reduce(np.stack(ends), axis=0)).astype(np.int64)
                s = np.sort(np.stack(codes, axis=-1), axis=-1)
                edges = 1 + (np.diff(s, axis=-1) != 0).sum(-1)
                before[k, 1:-1, 1:-1] = nlev >= 2
                after[k, 1:-1, 1:-1] = (nlev >= 2) & (edges >= nlev)
            lanes = np.zeros((Y, X), bool)
            lanes[1:-1, 1:-1] = True
            w_lanes = lanes.reshape(Y, X // 32, 32).any(-1)
            c["graphs"] += len(angs) * int(lanes.sum())
            c["graphs_sweep_before"] += int(before.sum())
            c["graphs_sweep_after"] += int(after.sum())
            c["warps"] += len(angs) * int(w_lanes.sum())
            c["warps_sweep_before"] += int(before.reshape(len(angs), Y, X // 32, 32).any(-1).sum())
            c["warps_sweep_after"] += int(after.reshape(len(angs), Y, X // 32, 32).any(-1).sum())
        res[g] = {"graphs_per_voxel": len(angs),
                  "share_graphs_sweep_before": round(c["graphs_sweep_before"] / c["graphs"], 4),
                  "share_graphs_sweep_after": round(c["graphs_sweep_after"] / c["graphs"], 4),
                  "share_warps_sweep_before": round(c["warps_sweep_before"] / c["warps"], 4),
                  "share_warps_sweep_after": round(c["warps_sweep_after"] / c["warps"], 4)}
    return res


def one_run(kinds, size, steps):
    """this process's library: phase-A ms per volume and the hash of the GLCM maps, per volume kind"""
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile

    from prof_glcm_phases import phase_of
    from pyradiomics_b200 import _lib, voxel

    line = {"lib": _lib.LIB_PATH}
    for kind in kinds:
        lev = torch.as_tensor(bench.synth_volume(size, kind).astype("uint8")).cuda()
        s = _lib.make_settings(32, 32)
        out = voxel.voxel_features("glcm", lev, s)
        for _ in range(2):
            voxel.voxel_features("glcm", lev, s, out=out, out_z0=0)
        torch.cuda.synchronize()
        digest = hashlib.sha256(out.cpu().numpy().tobytes()).hexdigest()
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                voxel.voxel_features("glcm", lev, s, out=out, out_z0=0)
            torch.cuda.synchronize()
        per = collections.defaultdict(float)
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA and phase_of(ev.name):
                per[phase_of(ev.name)] += ev.device_time / 1e3
        line[kind] = {"phaseA_ms": round(per["phaseA"] / steps, 3),
                      "glcm_ms": round(sum(per.values()) / steps, 3), "maps_sha256": digest}
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--kinds", nargs="+", default=["uniform", "smooth"])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--counts", action="store_true")
    ap.add_argument("--libs", nargs="*", default=[], metavar="NAME=PATH")
    ap.add_argument("--one", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if args.one:
        print(json.dumps(one_run(args.kinds, args.size, args.steps)))
        return
    lines = []
    if args.counts:
        lines.append({"what": "share of (voxel, angle) level graphs and of warps (32 consecutive voxels) of the "
                              "full-window voxels that enter the connectivity sweep, before and after the distinct-edge "
                              "count (host count of the kernel's rule)", "size": args.size,
                      **{k: sweep_counts(bench.synth_volume(args.size, k)) for k in args.kinds}})
    if args.libs:
        import torch

        if not torch.cuda.is_available():
            sys.exit("prof_glcm_mcc_class.py --libs needs a CUDA device")
        gpu = bench.gpu_info(torch.cuda.current_device())
        libs = [x.split("=", 1) for x in args.libs]
        runs = []
        for r in range(args.rounds):
            for name, path in libs:
                env = dict(os.environ, B200_RADIOMICS_LIB=os.path.abspath(path))
                cmd = [sys.executable, os.path.abspath(__file__), "--one", "--size", str(args.size), "--steps",
                       str(args.steps), "--kinds", *args.kinds]
                res = json.loads(subprocess.check_output(cmd, env=env, cwd=ROOT).decode().strip().splitlines()[-1])
                runs.append({"round": r + 1, "build": name, **{k: res[k] for k in args.kinds}})
                print(json.dumps(runs[-1]), flush=True)
        summary = {}
        for kind in args.kinds:
            summary[kind] = {name: {"phaseA_ms": [x[kind]["phaseA_ms"] for x in runs if x["build"] == name],
                                    "glcm_ms": [x[kind]["glcm_ms"] for x in runs if x["build"] == name]}
                             for name, _ in libs}
            summary[kind]["maps_identical"] = len({x[kind]["maps_sha256"] for x in runs}) == 1
        lines.append({"what": "GLCM phase-A ms per volume (torch.profiler, CUDA activities, mean of --steps volumes "
                              "after 2 warm-up volumes), builds alternated in fresh processes; SHA-256 of the 24 "
                              "float64 GLCM maps", "size": args.size, "steps": args.steps, "gpu": gpu,
                      "runs": runs, "summary": summary})
    for line in lines:
        text = json.dumps(line)
        print(text)
        if args.out:
            with open(args.out, "a") as f:
                f.write(text + "\n")


if __name__ == "__main__":
    main()
