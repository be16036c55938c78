"""A/B of two or more builds of the library on the flagship benchmark: bench.py --gpus 1 --no-e2e --no-cpu-baseline
--no-secondary per volume kind, the builds alternating round by round, each run in its own process (B200_RADIOMICS_LIB
selects the build).  Prints one JSON line per run (with the card's name and power limit) and a summary line per kind
and build: median, min and max of the benchmark value and of the GLCM ms.

    python scripts/ab_bench.py --libs parent=PATH pr=PATH [--kinds uniform smooth] [--rounds 3] [--steps 5]
                               [--warmup 3] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--libs", nargs="+", required=True, metavar="NAME=PATH")
    ap.add_argument("--kinds", nargs="+", default=["uniform", "smooth"])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    libs = [tuple(x.split("=", 1)) for x in args.libs]
    lines = []
    for kind in args.kinds:
        flags = ["--gpus", "1", "--steps", str(args.steps), "--warmup", str(args.warmup), "--kind", kind, "--no-e2e",
                 "--no-cpu-baseline", "--no-secondary"]
        what = "bench.py " + " ".join(flags) + ", builds alternated in one session (B200_RADIOMICS_LIB)"
        runs = []
        for r in range(args.rounds):
            for name, path in libs:
                env = dict(os.environ, B200_RADIOMICS_LIB=os.path.abspath(path))
                p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), *flags], env=env, capture_output=True,
                                   text=True, cwd=ROOT)
                if p.returncode:
                    sys.exit(p.stderr[-3000:])
                res = json.loads(p.stdout.strip().splitlines()[-1])
                line = {"what": what, "order": r, "build": name, "kind": kind, "gpu": res.get("gpu"),
                        "value": res.get("value"), "ms_per_step": res.get("ms_per_step"),
                        "per_class_ms": (res.get("roofline") or {}).get("per_class_ms"), "deterministic": res.get("deterministic"),
                        "parity_ok": (res.get("parity_sample") or {}).get("ok")}
                runs.append(line)
                lines.append(line)
                print(json.dumps(line), flush=True)
        for name, _ in libs:
            v = [x["value"] for x in runs if x["build"] == name]
            g = [x["per_class_ms"]["glcm"] for x in runs if x["build"] == name and x["per_class_ms"]]
            lines.append({"what": "summary: " + what, "kind": kind, "build": name, "runs": len(v),
                          "value_median": statistics.median(v), "value_min": min(v), "value_max": max(v),
                          "glcm_ms_median": statistics.median(g) if g else None,
                          "glcm_ms_min": min(g) if g else None, "glcm_ms_max": max(g) if g else None})
            print(json.dumps(lines[-1]), flush=True)
    if args.out:
        with open(args.out, "a") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
