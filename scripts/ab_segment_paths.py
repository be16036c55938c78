"""A/B of two builds of the library on the segment-mode GLCM / GLDM / NGTDM paths that have no benchmark workload.

    python scripts/ab_segment_paths.py A.so B.so [--names a b] [--rounds 3] [--repeat 3] [--out FILE]

Each round runs every build once, alternating, in its own process (B200_RADIOMICS_LIB selects the build).  A case is
timed on the host around calls that end in a device synchronise: one warm-up call, then the median of --repeat calls.
Cases:
  dev16_256     256^3 random levels 1..300 (16-bit level volume), GLCM + GLDM + NGTDM by segment_texture_device
  host16_256    the same volume through calculate_glcm, calculate_gldm and calculate_ngtdm (sum of the three)
  dev2d_4096    4096^2 2-D uint8 levels 1..32, distances [1, 4], segment_texture_device
  host2d_4096   the same image through calculate_glcm, calculate_gldm and calculate_ngtdm
  tile8_256     control: the benchmark's 256^3 uint8 case (levels 1..32, distance 1) by segment_texture_device
One JSON line with the card's name and power limit goes to stdout (and to --out)."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def worker(repeat):
    import numpy as np
    import torch
    sys.path.insert(0, ROOT)
    from pyradiomics_b200 import cmatrices as B, voxel

    rng = np.random.default_rng(0)
    l16 = rng.integers(1, 301, (256, 256, 256)).astype(np.int32)
    l2d = rng.integers(1, 33, (4096, 4096)).astype(np.int32)
    l8 = rng.integers(1, 33, (256, 256, 256)).astype(np.int32)
    m3, m2 = np.ones(l16.shape, bool), np.ones(l2d.shape, bool)

    def dev(lev, msk, dist, Ng):
        levd, _ = voxel.pack_levels(torch.as_tensor(lev).cuda(), torch.as_tensor(msk).cuda(), Ng)
        return lambda: B.segment_texture_device(levd, dist, Ng, 0, False, -1)

    def host(lev, msk, dist, Ng):
        return lambda: (B.calculate_glcm(lev, msk, dist, Ng, False, -1), B.calculate_gldm(lev, msk, dist, Ng, 0, False, -1),
                        B.calculate_ngtdm(lev, msk, dist, Ng, False, -1))

    cases = {"dev16_256": dev(l16, m3, [1], 300), "host16_256": host(l16, m3, [1], 300),
             "dev2d_4096": dev(l2d, m2, [1, 4], 32), "host2d_4096": host(l2d, m2, [1, 4], 32),
             "tile8_256": dev(l8, m3, [1], 32)}
    res = {}
    for name, fn in cases.items():
        fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(repeat):
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - t0) * 1e3)
        res[name] = round(statistics.median(ts), 3)
    print(json.dumps(res), flush=True)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, check=True).stdout.splitlines()[0]
    name, limit = (x.strip() for x in q.split(","))
    return {"name": name, "power_limit_w": float(limit)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs=2)
    ap.add_argument("--names", nargs=2, default=["a", "b"])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--out")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args.repeat)
    runs = {n: [] for n in args.names}
    for _ in range(args.rounds):
        for name, lib in zip(args.names, args.libs):
            env = dict(os.environ, B200_RADIOMICS_LIB=os.path.abspath(lib))
            out = subprocess.run([sys.executable, os.path.abspath(__file__), *args.libs, "--worker", "--repeat", str(args.repeat)],
                                 env=env, capture_output=True, text=True, check=True).stdout
            runs[name].append(json.loads(out.strip().splitlines()[-1]))
    cases = list(runs[args.names[0]][0])
    line = {"what": "segment-mode GLCM + GLDM + NGTDM paths without a benchmark workload, builds alternated per round",
            "gpu": gpu_info(), "unit": "ms, median of --repeat calls after one warm-up, host clock around a device synchronise",
            "rounds": args.rounds, "repeat": args.repeat,
            "ms": {c: {n: [r[c] for r in runs[n]] for n in args.names} for c in cases}}
    print(json.dumps(line), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
