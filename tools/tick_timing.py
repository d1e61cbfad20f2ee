"""The device tick with host waits (the synchronous calls) against the stream-ordered tick (the _async calls), in one run,
alternating them round by round.  One tick is main.cpp:76-105 on the device from a PointCloud2 message already in HBM:

    process (decode, decimate, time sort) -> compensate (deskew) -> voxel grid -> MAX_POINTS2MATCH gate -> update -> map add
    -> the state read back (main.cpp:85-88 publishes it every tick; both chains end with lv_get_state)

  sync   lv_process_cloud_device, lv_compensate_device, lv_voxelgrid_downsample_device (each waits for its count), the host
         applies the gate, lv_correct_device, lv_map_add_last_sweep, lv_get_state
  async  the same with lv_process_cloud_device_async, lv_compensate_device_async, lv_voxelgrid_downsample_device_async,
         lv_correct_device_async (counts stay on the device), lv_map_add_last_sweep, lv_get_state

Shapes: cfg1 (Velodyne 64 x 1024 = 65 536-point windows, one per message) and cfg2 (13 107-point windows, ten per message as
bench.py's cfg2 / kitti.yaml's 0.01 s windows).  Per tick it reports
  host_blocked_ms  host time inside the tick's calls before the state read (enqueue, plus every wait of the sync calls)
  wall_ms          host time of the whole tick, state read included, ticks back to back
  device_ms        CUDA events on the handle's stream around the tick's work (the handle runs on a torch stream)
as the median over --rounds rounds of --ticks ticks each, after --warmup ticks.  The card's name and power limit are read in
the same run.  Prints one JSON line per shape and writes them to OUT/tick_timing.json.
    python tools/tick_timing.py [--rounds 5] [--ticks 50] [--warmup 10] [--out DIR]   (DIR defaults to <tmp>/tick_timing)
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as G  # noqa: E402

VELO = np.dtype({"names": ["x", "y", "z", "intensity", "ring", "time"], "formats": ["<f4", "<f4", "<f4", "<f4", "<u2", "<f4"],
                 "offsets": [0, 4, 8, 16, 20, 24], "itemsize": 32})
SHAPES = {"cfg1_65536_per_window": ("xaloc.yaml", 65536), "cfg2_13107_per_window": ("kitti.yaml", 13107)}
LEAF, MIN_POINTS, FRT = 0.25, 20, 0.1


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return out[0] if out else "nvidia-smi: no output"


def message(lv, world, prm, n, s=8.0):
    """a Velodyne message of the synthetic world, ring-major (time order != message order), stamped 10 s"""
    rings, cols = 64, 1024
    x = world.pose(s, prm)
    sw = world.sweep(x, rings=rings, azimuths=cols, seed=3)
    xyz = sw.reshape(cols, rings, 3).transpose(1, 0, 2).reshape(-1, 3)
    p = np.zeros(len(xyz), VELO)
    p["x"], p["y"], p["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    p["ring"] = np.repeat(np.arange(rings), cols)
    p["time"] = np.tile(np.arange(cols) * (0.099 / (cols - 1)), rings).astype(np.float32)
    return p[:n].copy(), x


def path_for(lv, prm, x):
    """a deskew path (Compensator::upsample) around [10.0, 10.1] at the sweep's pose"""
    imu_t = np.arange(9.99, 10.105, 2.5e-3)
    a = np.tile(np.array([0.3, -0.2, 9.8], np.float32), (len(imu_t), 1))
    w = np.tile(np.array([0.0, 0.0, 0.2], np.float32), (len(imu_t), 1))
    states = [lv.state_from_ikfom(prm, x, ts, a[0], w[0]) for ts in (9.99, 10.03, 10.06, 10.099)]
    path = lv.compensator_upsample(states, a, w, imu_t)
    return path, lv.compensator_get_t2(path, 10.1)


class Chain:
    def __init__(self, lv, prm, world, msg, x, asyn):
        self.lv, self.asyn, self.msg = lv, asyn, msg
        self.stream = torch.cuda.Stream()
        prm.stream = self.stream.cuda_stream
        self.loc = lv.Localizer(prm)
        self.loc.map_build(world.map())
        x0, P0 = self.loc.get_state()
        self.loc.set_state(x, P0)
        self.path, self.x2 = path_for(lv, prm, x)
        n = len(msg)
        self.n = n
        self.lay = lv.cloud_layout("velodyne", msg.dtype)
        self.d_msg = self.loc.upload(msg)
        self.d_xyz, self.d_t, self.d_ds = self.loc.device_alloc(12 * n), self.loc.device_alloc(8 * n), self.loc.device_alloc(12 * n)
        self.d_k, self.d_m = self.loc.device_alloc(8), self.loc.device_alloc(8)
        self.x, self.P = np.zeros(lv.STATE_LEN), np.zeros((lv.DOF, lv.DOF))

    def tick(self, t):
        loc, n = self.loc, self.n
        if self.asyn:
            loc.process_cloud_device_async("velodyne", self.lay, self.d_msg, self.msg.nbytes, n, 10_000_000, True, True, FRT, 1, 1.0,
                                           self.d_xyz, self.d_t, self.d_k)
            loc.compensate_device_async(self.path, self.x2, self.d_xyz, self.d_t, self.d_k, n, self.d_xyz)
            loc.voxelgrid_downsample_device_async(self.d_xyz, self.d_k, n, LEAF, self.d_ds, self.d_m)
            loc.correct_device_async(self.d_ds, self.d_m, n, MIN_POINTS, t)
            loc.map_add_last_sweep(True)
        else:
            k = loc.process_cloud_device("velodyne", self.lay, self.d_msg, self.msg.nbytes, n, 10_000_000, True, True, FRT, 1, 1.0,
                                         self.d_xyz, self.d_t)
            loc.compensate_device(self.path, self.x2, self.d_xyz, self.d_t, k, self.d_xyz)
            m = loc.voxelgrid_downsample_device(self.d_xyz, k, LEAF, self.d_ds)
            if m >= MIN_POINTS:                                   # main.cpp:81
                loc.correct_device(self.d_ds, m, t)
                loc.map_add_last_sweep(True)

    def read_state(self):
        self.lv._check(self.loc.L.lv_get_state(self.loc.h, self.lv._d(self.x), self.lv._d(self.P)))

    def run(self, ticks, t0):
        blocked, ev = [], []
        torch.cuda.synchronize()
        w0 = time.perf_counter()
        for i in range(ticks):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(self.stream)
            h0 = time.perf_counter()
            self.tick(t0 + 0.01 * i)
            blocked.append(1e3 * (time.perf_counter() - h0))
            b.record(self.stream)
            self.read_state()
            ev.append((a, b))
        wall = 1e3 * (time.perf_counter() - w0) / ticks
        torch.cuda.synchronize()
        dev = [a.elapsed_time(b) for a, b in ev]
        st = self.loc.async_status() if self.asyn else (self.lv.OK, "")
        assert st[0] == self.lv.OK, st
        return statistics.median(blocked), wall, statistics.median(dev)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--ticks", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "tick_timing"))
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    lv = G.load_package()
    lines = []
    for name, (yaml, n) in SHAPES.items():
        world = lv.SynthWorld(20260924, 200000)
        prm = lv.params_from_yaml(os.path.join(lv.CONFIG_DIR, yaml), max_map_points=1 << 20, max_points=1 << 16)
        msg, x = message(lv, world, prm, n)
        chains = {"sync": Chain(lv, prm, world, msg, x, False), "async": Chain(lv, prm, world, msg, x, True)}
        for c in chains.values():
            c.run(args.warmup, 10.1)
        res = {k: {"host_blocked_ms": [], "wall_ms": [], "device_ms": []} for k in chains}
        for r in range(args.rounds):
            for k in (("sync", "async") if r % 2 == 0 else ("async", "sync")):
                hb, wall, dev = chains[k].run(args.ticks, 20.0 + r)
                res[k]["host_blocked_ms"].append(hb)
                res[k]["wall_ms"].append(wall)
                res[k]["device_ms"].append(dev)
        xs, xa = chains["sync"].x.copy(), chains["async"].x.copy()
        row = {"shape": name, "points_per_window": n, "card": card(), "rounds": args.rounds, "ticks": args.ticks,
               "same_final_state": bool((xs == xa).all())}
        for k, v in res.items():
            row[k] = {m: {"median": statistics.median(s), "min": min(s), "max": max(s)} for m, s in v.items()}
        line = json.dumps(row)
        print(line, flush=True)
        lines.append(row)
        for c in chains.values():
            c.loc.close()
    with open(os.path.join(args.out, "tick_timing.json"), "w") as f:
        json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
