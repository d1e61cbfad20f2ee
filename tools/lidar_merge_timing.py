"""Device time per message of the time-ordered merge into the LiDAR buffer (lv_lidar_merge_device_async) against the plain push
(lv_lidar_push_device_async) at 24 000 and 240 000 points (a Livox Avia / Mid-70 message at 10 Hz, and ten of them), for a message
that does not reach back into the buffer, one that reaches back over half a message, and one that reaches back over a whole one.

Each timed call follows the same set-up on the handle's stream: the buffer is cleared and one message A of n points over 0.1 s is
pushed; the timed message B (n points over 0.1 s) starts at A's end, in A's middle or just before A's start, so T_tail holds 0,
n / 2 or n points.  CUDA events around B's call alone, --iters times per run, --runs runs, plain push and merge alternated; the
median of the per-call times is reported, with the spread over runs.  Both calls are given the count on the device, as in the tick.
The card's name and power limit are read in the same run.  Prints one JSON line per shape and writes them to
OUT/lidar_merge_timing.json.
    python tools/lidar_merge_timing.py [--runs 9] [--iters 40] [--warmup 5] [--out DIR]   (DIR defaults to <tmp>/lidar_merge_timing)
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as G  # noqa: E402

OVERLAPS = {"none": 0.0, "half": 0.5, "whole": 1.0}


def message(n, start, seed):
    """n points over 0.1 s from `start`, time-sorted, as the message front end leaves them"""
    rng = np.random.default_rng(seed)
    t = start + np.sort(rng.uniform(0.0, 0.1, n))
    return rng.normal(0, 20, (n, 3)).astype(np.float32), t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=9)
    ap.add_argument("--iters", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "lidar_merge_timing"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("lidar_merge_timing: no CUDA device (there is nothing to measure without one)")
    os.makedirs(a.out, exist_ok=True)
    lv = G.load_package()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    stream = torch.cuda.Stream()
    prm = lv.default_params(max_points=1 << 12, max_map_points=1 << 12)
    prm.stream = stream.cuda_stream
    loc = lv.Localizer(prm)
    T = lv._transform12(np.array([0.0, -1.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.3, -0.2, 0.1], np.float32))
    results = []
    for n in (24_000, 240_000):
        loc.lidar_reserve(3 * n)
        loc.lidar_reserve_merge(n)
        xa, ta = message(n, 10.0, 1)
        d_a = [loc.upload(xa), loc.upload(ta), loc.upload(np.array([n], np.int64))]
        for name, frac in OVERLAPS.items():
            start = ta[-1] - frac * 0.1 if frac < 1.0 else ta[0] - 1e-6
            xb, tb = message(n, start, 2)
            d_b = [loc.upload(xb), loc.upload(tb), d_a[2]]
            calls = {
                "push": lambda: loc.lidar_push_async(*d_b, n),
                "merge": lambda: loc.lidar_merge_async(*d_b, n),
                "merge_T": lambda: loc.lidar_merge_async(*d_b, n, T),
            }
            per_call = {k: [] for k in calls}
            for rep in range(a.warmup + a.runs):
                for key, call in calls.items():                          # alternated, so all see the same machine state
                    ev = []
                    for _ in range(a.iters):
                        loc.lidar_clear_async(float("inf"))
                        loc.lidar_push_async(*d_a, n)
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record(stream)
                        call()
                        e1.record(stream)
                        ev.append((e0, e1))
                    ev[-1][1].synchronize()
                    if rep >= a.warmup:
                        per_call[key].append(float(np.median([e0.elapsed_time(e1) * 1e3 for e0, e1 in ev])))
            st = loc.async_status()
            assert st == (lv.OK, ""), st
            assert loc.lidar_info()["points"] == 2 * n
            r = dict(points=n, overlap=name, t_tail=int((ta > tb[0]).sum()), card=card,
                     us_per_message={k: float(np.median(v)) for k, v in per_call.items()},
                     us_spread={k: float(np.max(v) - np.min(v)) for k, v in per_call.items()})
            print(json.dumps(r))
            results.append(r)
            for d in d_b[:2]:
                loc.device_free(d)
        for d in d_a:
            loc.device_free(d)
        loc.lidar_clear_async(float("inf"))
    loc.close()
    with open(os.path.join(a.out, "lidar_merge_timing.json"), "w") as f:
        json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
