"""The windowed device tick with the LiDAR buffer in HBM against the same tick fed by a host-side deque, in one run, alternating
them round by round.  Velodyne 64 x 1024 messages arrive at 10 Hz; the tick localizes on windows [t2 - delta, t2] much shorter
than a message (kitti.yaml's 0.01 s, xaloc's 0.02 s), as main.cpp:61-122 does:

  device  receive: lv_process_cloud_device_async -> lv_lidar_push_device_async (no host wait)
          tick:    lv_lidar_get_points_device_async -> compensate -> voxel grid -> lv_correct_device_async (MAX_POINTS2MATCH gate)
                   -> lv_map_add_last_sweep -> lv_lidar_clear_async -> lv_get_state
  host    receive: lv_process_cloud_device, the kept points downloaded into a host deque of messages
          tick:    the window cut on the host (searchsorted: the deque is time-sorted here), uploaded with its count, then the same
                   stream-ordered stages, the clear on the host deque, lv_get_state

Per tick it reports
  host_blocked_ms  host time inside the tick's calls before the state read (the host chain's cut and upload included)
  wall_ms          host time of the whole tick, state read included, ticks back to back (receives included, amortised)
  device_ms        CUDA events on the handle's stream around the tick's work (the handle runs on a torch stream)
as the median over --rounds rounds of --ticks ticks each, after --warmup ticks.  The card's name and power limit are read in
the same run.  Prints one JSON line per window length and writes them to OUT/window_timing.json.
    python tools/window_timing.py [--rounds 5] [--ticks 50] [--warmup 10] [--out DIR]   (DIR defaults to <tmp>/window_timing)
"""
import argparse
import collections
import ctypes as C
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import __graft_entry__ as G  # noqa: E402
from tick_timing import card, message  # noqa: E402

DELTAS = {"kitti_0.01s": ("kitti.yaml", 0.01), "xaloc_0.02s": ("xaloc.yaml", 0.02)}
LEAF, MIN_POINTS, FRT, EMPTY_LIDAR_TIME, N_MAX = 0.25, 20, 0.1, 0.3, 1 << 16


def path_for(lv, prm, x, t1, t2):
    """a deskew path (Compensator::upsample) around [t1, t2] at the sweep's pose"""
    imu_t = np.arange(t1 - 0.01, t2 + 0.006, 2.5e-3)
    a = np.tile(np.array([0.3, -0.2, 9.8], np.float32), (len(imu_t), 1))
    w = np.tile(np.array([0.0, 0.0, 0.2], np.float32), (len(imu_t), 1))
    states = [lv.state_from_ikfom(prm, x, ts, a[0], w[0]) for ts in np.linspace(t1 - 0.01, t2 + 0.002, 3)]
    path = lv.compensator_upsample(states, a, w, imu_t)
    return path, lv.compensator_get_t2(path, t2)


class Chain:
    def __init__(self, lv, prm, world, msg, x, delta, device):
        self.lv, self.msg, self.delta, self.device = lv, msg, delta, device
        self.stream = torch.cuda.Stream()
        prm.stream = self.stream.cuda_stream
        self.loc = lv.Localizer(prm)
        self.loc.map_build(world.map())
        x0, P0 = self.loc.get_state()
        self.loc.set_state(x, P0)
        self.prm, self.xs = prm, x
        self.n = len(msg)
        self.lay = lv.cloud_layout("velodyne", msg.dtype)
        self.d_msg = self.loc.upload(msg)
        a = self.loc.device_alloc
        self.d_pxyz, self.d_pt, self.d_k = a(12 * self.n), a(8 * self.n), a(8)
        self.d_wxyz, self.d_wt, self.d_w = a(12 * N_MAX), a(8 * N_MAX), a(8)
        self.d_ds, self.d_m = a(12 * N_MAX), a(8)
        if device:
            self.loc.lidar_reserve(6 * self.n)
        self.deque = collections.deque()                          # host chain: (xyz, time) per message, newest first
        self.k, self.received = 0, 0
        self.paths = {}
        self.x, self.P = np.zeros(lv.STATE_LEN), np.zeros((lv.DOF, lv.DOF))

    def window(self, k):
        t2 = 10.0 + self.delta * (k + 1)
        t1 = t2 - self.delta
        if k not in self.paths:
            self.paths[k] = path_for(self.lv, self.prm, self.xs, t1, t2)
        return t1, t2, self.paths[k]

    def receive(self, j):
        loc, stamp = self.loc, 10_000_000 + 100_000 * j
        args = ("velodyne", self.lay, self.d_msg, self.msg.nbytes, self.n, stamp, True, True, FRT, 1, 1.0, self.d_pxyz, self.d_pt)
        if self.device:
            loc.process_cloud_device_async(*args, self.d_k)
            loc.lidar_push_async(self.d_pxyz, self.d_pt, self.d_k, self.n)
        else:
            k = loc.process_cloud_device(*args)
            self.deque.appendleft((loc.download(self.d_pxyz, np.empty((k, 3), np.float32)), loc.download(self.d_pt, np.empty(k))))

    def tick(self, t1, t2, path, x2):
        loc = self.loc
        if self.device:
            loc.lidar_get_points_async(t1, t2, self.d_wxyz, self.d_wt, N_MAX, self.d_w)
        else:
            parts = []
            for xyz, t in reversed(self.deque):                   # oldest message first
                lo, hi = np.searchsorted(t, t1, "left"), np.searchsorted(t, t2, "right")
                if hi > lo:
                    parts.append((xyz[lo:hi], t[lo:hi]))
            xyz = np.ascontiguousarray(np.concatenate([p[0] for p in parts]) if parts else np.zeros((0, 3), np.float32))
            t = np.ascontiguousarray(np.concatenate([p[1] for p in parts]) if parts else np.zeros(0))
            cnt = np.array([len(t)], np.int64)
            for d, arr in ((self.d_wxyz, xyz), (self.d_wt, t), (self.d_w, cnt)):
                if arr.nbytes:
                    self.lv._check(loc.L.lv_memcpy_h2d(loc.h, d, arr.ctypes.data_as(C.c_void_p), arr.nbytes))
        loc.compensate_device_async(path, x2, self.d_wxyz, self.d_wt, self.d_w, N_MAX, self.d_wxyz)
        loc.voxelgrid_downsample_device_async(self.d_wxyz, self.d_w, N_MAX, LEAF, self.d_ds, self.d_m)
        loc.correct_device_async(self.d_ds, self.d_m, N_MAX, MIN_POINTS, t2)
        loc.map_add_last_sweep(True)
        if self.device:
            loc.lidar_clear_async(t2 - EMPTY_LIDAR_TIME)
        else:
            while self.deque and self.deque[-1][1][-1] <= t2 - EMPTY_LIDAR_TIME:
                self.deque.pop()

    def read_state(self):
        self.lv._check(self.loc.L.lv_get_state(self.loc.h, self.lv._d(self.x), self.lv._d(self.P)))

    def run(self, ticks):
        blocked, ev = [], []
        torch.cuda.synchronize()
        w0 = time.perf_counter()
        for _ in range(ticks):
            t1, t2, (path, x2) = self.window(self.k)
            while 10.0 + 0.1 * self.received < t2:                # the message that holds t2 has arrived
                self.receive(self.received)
                self.received += 1
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(self.stream)
            h0 = time.perf_counter()
            self.tick(t1, t2, path, x2)
            blocked.append(1e3 * (time.perf_counter() - h0))
            b.record(self.stream)
            self.read_state()
            ev.append((a, b))
            self.k += 1
        wall = 1e3 * (time.perf_counter() - w0) / ticks
        torch.cuda.synchronize()
        dev = [a.elapsed_time(b) for a, b in ev]
        st = self.loc.async_status()
        assert st[0] == self.lv.OK, st
        return statistics.median(blocked), wall, statistics.median(dev)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--ticks", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "window_timing"))
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    lv = G.load_package()
    lines = []
    for name, (yaml, delta) in DELTAS.items():
        world = lv.SynthWorld(20260924, 200000)
        prm = lv.params_from_yaml(os.path.join(lv.CONFIG_DIR, yaml), max_map_points=1 << 21, max_points=N_MAX)
        msg, x = message(lv, world, prm, 65536)
        chains = {"host_deque": Chain(lv, prm, world, msg, x, delta, False), "device_buffer": Chain(lv, prm, world, msg, x, delta, True)}
        for c in chains.values():
            c.loc.map_set_growth(1 << 23)
            for k in range(args.warmup + args.rounds * args.ticks):   # paths are host work outside the timed ticks
                c.window(k)
            c.run(args.warmup)
        res = {k: {"host_blocked_ms": [], "wall_ms": [], "device_ms": []} for k in chains}
        for r in range(args.rounds):
            for k in (("host_deque", "device_buffer") if r % 2 == 0 else ("device_buffer", "host_deque")):
                hb, wall, dev = chains[k].run(args.ticks)
                res[k]["host_blocked_ms"].append(hb)
                res[k]["wall_ms"].append(wall)
                res[k]["device_ms"].append(dev)
        row = {"window": name, "delta_s": delta, "points_per_message": len(msg), "card": card(), "rounds": args.rounds,
               "ticks": args.ticks}
        for k, v in res.items():
            row[k] = {m: {"median": statistics.median(s), "min": min(s), "max": max(s)} for m, s in v.items()}
        print(json.dumps(row), flush=True)
        lines.append(row)
        for c in chains.values():
            c.loc.close()
    with open(os.path.join(args.out, "window_timing.json"), "w") as f:
        json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
