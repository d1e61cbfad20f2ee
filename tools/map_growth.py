"""Cost of growing the device map (lv_map_reserve / lv_map_set_growth), on one GPU.

1. One growth: a handle holding a SynthWorld surface map at capacity C is reserved to 2 C.  Wall time around the call
   between two lv_synchronize (allocation + re-hash + arena copy + the frees), and the bytes the kernels move: the old
   tables read, the new tables initialised and filled, the arena's used prefix read and written.  C = 1 M and 8 M points.
2. The device tick (lv_correct_device + lv_map_add_last_sweep) at cfg1 sizes (65 536-point sweeps) over --sweeps sweeps
   along the road, from an empty map: handle G starts at 1/8 of the capacity it ends at, with growth on; handle B is born
   at G's final capacity.  Per tick: host time to enqueue, and the tick's wall time with a synchronisation after it (the
   GPU time of the tick, launch latency included); growths and host waits.  Ticks in which G grew are reported apart.
   A second pass enqueues every tick without synchronising (the driver's steady state) for the host time and the waits.

Prints one JSON object.  Run from the repository root after __graft_entry__.build().
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as G  # noqa: E402
import bench  # noqa: E402


def one_growth(lv, cap):
    world = lv.SynthWorld(bench.SEED + 5, cap)
    mp = world.map()
    prm = bench.config_params(lv, "cfg1", max_map_points=cap)
    loc = lv.Localizer(prm)
    loc.map_build(mp)
    loc.map_status()
    a = loc.map_info()
    loc.synchronize()
    t0 = time.perf_counter()
    loc.map_reserve(2 * cap)
    loc.synchronize()
    ms = (time.perf_counter() - t0) * 1e3
    b = loc.map_info()
    moved = (32 * a["voxel_slots"] + 16 * a["block_slots"]            # old tables read
             + 2 * (32 * b["voxel_slots"] + 16 * b["block_slots"])    # new tables initialised, then written (upper bound)
             + 2 * 16 * a["arena_top"])                               # arena prefix read + written
    loc.close()
    return dict(capacity_from=cap, capacity_to=2 * cap, map_points=int(a["points"]), ms=round(ms, 3),
                bytes_moved=int(moved), gb_per_s=round(moved / ms / 1e6, 1), map_bytes_before=int(a["bytes"]),
                map_bytes_after=int(b["bytes"]))


def road(lv, O, n):
    prm = bench.config_params(lv, "cfg1")
    world = lv.SynthWorld(bench.SEED + 1, 200_000)
    rng = np.random.default_rng(11)
    sweeps, xs = [], []
    for i in range(n):
        truth = world.pose(15.0 + 1.5 * i, prm)
        sweeps.append(world.sweep(truth, rings=bench.RINGS, azimuths=bench.AZIMUTHS, min_dist=4.0, seed=1000 + i))
        d = np.zeros(23)
        d[0:3] = rng.uniform(-0.05, 0.05, 3)
        d[3:6] = rng.uniform(-0.5, 0.5, 3) * np.pi / 180.0
        xs.append(truth if i == 0 else O.boxplus(truth, d))
    return sweeps, xs


def ticks(lv, sweeps, xs, cap, grow_limit, sync):
    prm = bench.config_params(lv, "cfg1", max_map_points=cap)
    loc = lv.Localizer(prm)
    if grow_limit:
        loc.map_set_growth(grow_limit)
    _, P0 = lv.init_state_host(prm)
    d = [loc.upload(s) for s in sweeps]
    loc.synchronize()
    host, wall, grew = [], [], []
    for i, s in enumerate(sweeps):
        loc.set_state(xs[i], P0)
        g0 = loc.map_info()["growths"] if sync else 0
        t0 = time.perf_counter()
        loc.correct_device(d[i], len(s), time=0.1 * i)
        loc.map_add_last_sweep(downsample=True)
        t1 = time.perf_counter()
        if sync:
            loc.synchronize()
        t2 = time.perf_counter()
        host.append((t1 - t0) * 1e3)
        wall.append((t2 - t0) * 1e3)
        grew.append(sync and loc.map_info()["growths"] != g0)
    loc.synchronize()
    loc.map_status()
    info = loc.map_info()
    for p in d:
        loc.device_free(p)
    loc.close()
    return np.array(host), np.array(wall), np.array(grew, bool), info


def summary(host, wall, grew, info, sync):
    steady = ~grew
    out = dict(host_enqueue_ms_median=round(float(np.median(host[steady])), 4), host_enqueue_ms_max=round(float(host[steady].max()), 4),
               growths=int(info["growths"]), host_waits=int(info["host_waits"]), final_capacity=int(info["capacity_points"]),
               map_points=int(info["points"]), map_bytes=int(info["bytes"]))
    if sync:
        out.update(tick_ms_median=round(float(np.median(wall[steady])), 4), tick_ms_max=round(float(wall[steady].max()), 4))
        if grew.any():
            out.update(growth_ticks=int(grew.sum()), growth_tick_ms=[round(float(v), 3) for v in wall[grew]],
                       growth_tick_host_ms=[round(float(v), 3) for v in host[grew]])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sweeps", type=int, default=300)
    ap.add_argument("--skip-big", action="store_true", help="skip the 8 M -> 16 M growth (about 45 GB of device memory)")
    a = ap.parse_args()
    lv, O = G.load_package(), G.load_oracle()
    import subprocess
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = dict(gpu=gpu, growth=[one_growth(lv, 1 << 20)])
    if not a.skip_big:
        res["growth"].append(one_growth(lv, 1 << 23))
    sweeps, xs = road(lv, O, a.sweeps)
    # pass 0 finds the final capacity; G then starts at 1/8 of it
    _, _, _, probe = ticks(lv, sweeps, xs, 1 << 17, 1 << 24, False)
    final = int(probe["capacity_points"])
    for sync in (True, False):
        g = ticks(lv, sweeps, xs, max(final // 8, 1 << 16), 1 << 24, sync)
        b = ticks(lv, sweeps, xs, final, 0, sync)
        key = "tick_synchronised" if sync else "tick_streamed"
        res[key] = dict(grown=summary(*g, sync), born_final=summary(*b, sync))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
