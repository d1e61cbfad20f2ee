"""A/B comparison of two builds of liblimovelo_b200.so on one GPU, in one session.

Runs `bench.py --no-cpu --dump-outputs` for every config, alternating the two libraries (LV_LIB_PATH) run by run, so
that both see the same machine state.  Prints each config's ms_per_step (median, min, max, spread = max - min) per
build and compares every dumped array (state, covariance, per-evaluation log) of the two builds with np.array_equal.
The card's name and power limit are read with `nvidia-smi --query-gpu`, nothing is changed on the device.

    python tools/ab_bench.py LIB_A LIB_B [--runs 3] [--configs cfg0,cfg1,cfg2,cfg3] [--steps 200] [--warmup 5] [--json OUT]

Exit status 1 when a dumped array differs between the builds.
"""
import argparse
import glob
import json
import os
import statistics
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "nvidia-smi: no output"
    except Exception as e:             # the numbers stay valid, only their label is missing
        return "nvidia-smi unavailable (%s)" % e


def run_bench(lib, cfg, steps, warmup, dump_dir):
    env = dict(os.environ, LV_LIB_PATH=os.path.abspath(lib))
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--no-cpu", "--config", cfg,
           "--steps", str(steps), "--warmup", str(warmup), "--dump-outputs", dump_dir]
    p = subprocess.run(cmd, env=env, capture_output=True, text=True)
    if p.returncode != 0:
        raise SystemExit("bench.py failed (%s, %s):\n%s" % (lib, cfg, p.stderr[-4000:]))
    line = [l for l in p.stdout.splitlines() if l.startswith("{")][-1]
    return json.loads(line)


def load_dump(d):
    return {os.path.basename(f)[:-4]: np.load(f) for f in sorted(glob.glob(os.path.join(d, "*.npy")))}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("lib_a")
    ap.add_argument("lib_b")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--configs", default="cfg0,cfg1,cfg2,cfg3")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", default="", help="also write the results to this file")
    args = ap.parse_args()
    libs = {"A": args.lib_a, "B": args.lib_b}
    card = gpu_info()
    print("card (name, power limit, max SM clock):", card)
    print("A =", libs["A"])
    print("B =", libs["B"])
    results, identical = {}, True
    with tempfile.TemporaryDirectory(prefix="lv_ab_") as tmp:
        for cfg in args.configs.split(","):
            ms = {"A": [], "B": []}
            dumps = {"A": [], "B": []}
            for r in range(args.runs):
                for tag in (("A", "B") if r % 2 == 0 else ("B", "A")):        # alternate, and alternate who goes first
                    d = os.path.join(tmp, "%s_%s_%d" % (cfg, tag, r))
                    ms[tag].append(run_bench(libs[tag], cfg, args.steps, args.warmup, d)["ms_per_step"])
                    dumps[tag].append(load_dump(d))
            ref = dumps["A"][0]
            diff = []
            for tag in ("A", "B"):
                for k, dd in enumerate(dumps[tag]):
                    if sorted(dd) != sorted(ref):
                        diff.append("%s run %d: arrays %s vs %s" % (tag, k, sorted(dd), sorted(ref)))
                        continue
                    diff += ["%s run %d: %s" % (tag, k, name) for name in ref if not np.array_equal(dd[name], ref[name])]
            identical = identical and not diff
            row = {}
            for tag in ("A", "B"):
                v = ms[tag]
                row[tag] = {"ms_per_step": v, "median": statistics.median(v), "min": min(v), "max": max(v),
                            "spread": max(v) - min(v)}
            row["B_vs_A"] = row["B"]["median"] / row["A"]["median"] - 1.0
            row["arrays"] = sorted(ref)
            row["identical"] = not diff
            row["differences"] = diff
            results[cfg] = row
            print("%s  A %.4f ms [%.4f..%.4f, spread %.4f]  B %.4f ms [%.4f..%.4f, spread %.4f]  B/A-1 %+.1f %%  outputs %s" % (
                cfg, row["A"]["median"], row["A"]["min"], row["A"]["max"], row["A"]["spread"],
                row["B"]["median"], row["B"]["min"], row["B"]["max"], row["B"]["spread"], 100 * row["B_vs_A"],
                "bit-identical (%d arrays x %d runs)" % (len(ref), 2 * args.runs) if not diff else "DIFFER: " + "; ".join(diff)),
                flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": card, "libs": libs, "steps": args.steps, "warmup": args.warmup, "runs": args.runs,
                       "results": results}, f, indent=1)
    sys.exit(0 if identical else 1)


if __name__ == "__main__":
    main()
