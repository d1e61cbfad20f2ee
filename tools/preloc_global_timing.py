"""Cost of finding the start pose anywhere in a saved map on one GPU: lv_prelocalize_global over a whole-map window, pruned
and exhaustive (LV_PRELOC_NO_PRUNE=1), on SynthWorld maps of 1 M and 10 M points; and lv_prelocalize against
lv_prelocalize_global at the recommended +-5 m window.

    python tools/preloc_global_timing.py [--sizes 1000000,10000000] [--reps 25] [--reps-exhaustive 25] [--json OUT]

Both calls synchronise, so a time is the wall time of the call, the median (and min .. max) of --reps calls after two
warm-up calls.  The whole-map window covers every occupied voxel from the map's centre (lv_map_extent, INTEGRATION.md B7),
every heading, 0.4 m / 2 degrees, 2048 scored points; the sweep is taken at the road position 60 m and the start is the
map's centre turned by 100 degrees.  One line per configuration; stats are lv_preloc_stats.  The card's name, power limit
and maximum SM clock are read with `nvidia-smi --query-gpu` in the same run; nothing is changed on the device.
"""
import argparse
import json
import math
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import __graft_entry__ as G  # noqa: E402
from preloc_timing import gpu_info  # noqa: E402


def timed(fn, reps, warm=2):
    for _ in range(warm):
        fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(t), min(t), max(t)


def axes(x):
    g = np.asarray(x[23:26], np.float64)
    g = g / np.linalg.norm(g)
    e = np.array([0.0, 1.0, 0.0]) if abs(g[0]) > 0.9 else np.array([1.0, 0.0, 0.0])
    u = e - e.dot(g) * g
    u /= np.linalg.norm(u)
    return u, np.cross(g, u)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1000000,10000000")
    ap.add_argument("--reps", type=int, default=25)
    ap.add_argument("--reps-exhaustive", type=int, default=25)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    lv = G.load_package()
    pi32 = float(np.float32(math.pi))
    rec = dict(radius=5.0, step=0.4, yaw_range=pi32, yaw_step=math.radians(2.0), max_points=2048)
    res = dict(gpu=gpu_info(), rows=[])
    print("gpu:", res["gpu"], flush=True)
    for m in [int(s) for s in a.sizes.split(",")]:
        prm = lv.params_from_yaml(os.path.join(lv.CONFIG_DIR, "xaloc.yaml"), max_map_points=m + (m >> 4), max_points=1 << 15)
        world = lv.SynthWorld(20261016, m)
        mp = world.map()
        truth = world.pose(60.0, prm)
        sweep = world.sweep(truth, rings=32, azimuths=256, elev=(-10.0, 15.0), seed=3)
        loc = lv.Localizer(prm)
        try:
            loc.map_build(mp)
            loc.init_state()
            _, P0 = loc.get_state()
            d = loc.upload(np.ascontiguousarray(sweep, np.float32))
            lo, hi = loc.map_extent()
            u, v = axes(truth)
            g = np.asarray(truth[23:26]) / np.linalg.norm(truth[23:26])
            # the start: the map's centre, the truth's attitude turned by 100 degrees about gravity
            th = math.radians(100.0)
            q = np.array([*(math.sin(th / 2) * g), math.cos(th / 2)])
            r = truth[3:7]
            start = truth.copy()
            start[3:7] = [q[3] * r[0] + q[0] * r[3] + q[1] * r[2] - q[2] * r[1], q[3] * r[1] + q[1] * r[3] + q[2] * r[0] - q[0] * r[2],
                          q[3] * r[2] + q[2] * r[3] + q[0] * r[1] - q[1] * r[0], q[3] * r[3] - q[0] * r[0] - q[1] * r[1] - q[2] * r[2]]
            start[0:2] = 0.5 * (lo[0:2] + hi[0:2])
            corners = np.array([[x, y, z] for x in (lo[0], hi[0]) for y in (lo[1], hi[1]) for z in (lo[2], hi[2])]) - start[0:3]
            radius = float(np.max(np.abs(np.concatenate([corners @ u, corners @ v]))))
            whole = dict(rec, radius=radius)

            def glob(win, x0, out):
                def call():
                    loc.set_state(x0, P0)
                    st, o, s = loc.prelocalize_global(d, len(sweep), **win)
                    assert st == lv.OK
                    out[:] = [o, s]
                return call

            def brute(win, x0, out):
                def call():
                    loc.set_state(x0, P0)
                    st, o = loc.prelocalize(d, len(sweep), **win)
                    assert st == lv.OK
                    out[:] = [o, None]
                return call

            o = [None, None]
            t = timed(glob(whole, start, o), a.reps)
            row = dict(map_points=len(mp), config="whole-map pruned", window=whole, ms=t, stats=o[1], winner=o[0]["index"],
                       score=o[0]["score"], pos_err_m=float(np.linalg.norm(np.asarray(o[0]["x"])[0:3] - truth[0:3])))
            print(json.dumps(row), flush=True)
            res["rows"].append(row)
            os.environ["LV_PRELOC_NO_PRUNE"] = "1"
            try:
                o2 = [None, None]
                t = timed(glob(whole, start, o2), a.reps_exhaustive, warm=1)
            finally:
                del os.environ["LV_PRELOC_NO_PRUNE"]
            row = dict(map_points=len(mp), config="whole-map exhaustive", window=whole, ms=t, stats=o2[1], winner=o2[0]["index"],
                       score=o2[0]["score"], same_winner=o2[0]["index"] == o[0]["index"],
                       probes_per_s=o2[1]["probes"] / (t[0] * 1e-3))
            print(json.dumps(row), flush=True)
            res["rows"].append(row)
            for name, fn in (("recommended lv_prelocalize", brute), ("recommended lv_prelocalize_global", glob)):
                o3 = [None, None]
                t = timed(fn(rec, truth, o3), a.reps)
                row = dict(map_points=len(mp), config=name, window=rec, ms=t, winner=o3[0]["index"], score=o3[0]["score"])
                if o3[1] is not None:
                    row["stats"] = o3[1]
                print(json.dumps(row), flush=True)
                res["rows"].append(row)
            loc.device_free(d)
        finally:
            loc.close()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
