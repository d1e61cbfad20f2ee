"""What carrying intensity, range and time through the device tick costs: the xyz-only chain against the full-point chain, in one
run, alternating them round by round.  Velodyne 64 x 1024 messages (float intensity) arrive at 10 Hz into the LiDAR buffer in HBM; the
tick localizes on xaloc's 0.02 s windows, maps online (lv_map_add_last_sweep) and publishes both clouds every tick:
global_ds_compensated (/limovelo/pcl) and, with high_quality_publish, global_compensated (/limovelo/full_pcl).

  xyz   lv_lidar_reserve / push / get, lv_voxelgrid_downsample_device_async, lv_sweep_to_world_device_async of both clouds; the
        publisher downloads each cloud's count and xyz
  full  lv_lidar_reserve_full / push_full / get_full (intensity and range lanes), lv_voxelgrid_downsample_full_device_async,
        the same transforms, lv_cloud_stamp_device_async of both clouds; the publisher downloads each cloud's count, xyz, time,
        intensity, range and the two header stamps

Everything else (process, compensate, lv_correct_device_async, clear) is shared.  Per tick it reports
  host_blocked_ms  host time inside the tick's calls before the state read
  wall_ms          host time of the whole tick, state read and both published clouds included, ticks back to back
  device_ms        CUDA events on the handle's stream around the tick's work (receives excluded)
as the median over --rounds rounds of --ticks ticks each, after --warmup ticks.  The card's name, power limit and maximum SM clock
are read in the same run.  Prints one JSON line and writes OUT/full_points_timing.json.
    python tools/full_points_timing.py [--rounds 5] [--ticks 50] [--warmup 10] [--out DIR]   (DIR: <tmp>/full_points_timing)
"""
import argparse
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
from window_timing import path_for  # noqa: E402

DELTA, LEAF, MIN_POINTS, FRT, EMPTY_LIDAR_TIME, N_MAX = 0.02, 0.25, 20, 0.1, 0.3, 1 << 17


class Chain:
    def __init__(self, lv, prm, world, msg, x, full):
        self.lv, self.msg, self.full = lv, msg, full
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
        self.d_p = [a(k * self.n) for k in (12, 8, 4, 4)]
        self.d_w = [a(k * N_MAX) for k in (12, 8, 4, 4)]
        self.d_ds = [a(k * N_MAX) for k in (12, 8, 4, 4)]
        self.d_pub, self.d_full = a(12 * N_MAX), a(12 * N_MAX)
        self.d_k, self.d_wn, self.d_m, self.d_pubn, self.d_fulln, self.d_stamps = a(8), a(8), a(8), a(8), a(8), a(16)
        (self.loc.lidar_reserve_full if full else self.loc.lidar_reserve)(6 * self.n)
        self.k, self.received = 0, 0
        self.paths = {}
        self.x, self.P = np.zeros(lv.STATE_LEN), np.zeros((lv.DOF, lv.DOF))
        self.host = [np.empty((N_MAX, 3), np.float32), np.empty(N_MAX), np.empty(N_MAX, np.float32), np.empty(N_MAX, np.float32)]
        self.cnt, self.stamps = np.zeros(1, np.int64), np.zeros(2, np.uint64)

    def path(self, t1, t2):
        key = (round(t1, 9), round(t2, 9))
        if key not in self.paths:
            self.paths[key] = path_for(self.lv, self.prm, self.xs, t1, t2)
        return self.paths[key]

    def receive(self, j):
        loc, stamp = self.loc, 10_000_000 + 100_000 * j
        if self.full:
            loc.process_cloud_device_async("velodyne", self.lay, self.d_msg, self.msg.nbytes, self.n, stamp, True, True, FRT, 1, 1.0,
                                           self.d_p[0], self.d_p[1], self.d_k, self.d_p[2], self.d_p[3])
            loc.lidar_push_full_async(*self.d_p, self.d_k, self.n)
        else:
            loc.process_cloud_device_async("velodyne", self.lay, self.d_msg, self.msg.nbytes, self.n, stamp, True, True, FRT, 1, 1.0,
                                           self.d_p[0], self.d_p[1], self.d_k)
            loc.lidar_push_async(self.d_p[0], self.d_p[1], self.d_k, self.n)

    def d2h(self, out, d, nbytes):
        if nbytes:
            self.lv._check(self.loc.L.lv_memcpy_d2h(self.loc.h, out.ctypes.data_as(C.c_void_p), C.c_void_p(d), nbytes))

    def tick(self, t2):
        loc, t1 = self.loc, t2 - DELTA
        path, x2 = self.path(t1, t2)
        if self.full:
            loc.lidar_get_points_full_async(t1, t2, *self.d_w, N_MAX, self.d_wn)
        else:
            loc.lidar_get_points_async(t1, t2, self.d_w[0], self.d_w[1], N_MAX, self.d_wn)
        loc.compensate_device_async(path, x2, self.d_w[0], self.d_w[1], self.d_wn, N_MAX, self.d_w[0])
        if self.full:
            loc.voxelgrid_downsample_full_async(*self.d_w[:3], self.d_wn, N_MAX, LEAF, *self.d_ds, self.d_m)
        else:
            loc.voxelgrid_downsample_device_async(self.d_w[0], self.d_wn, N_MAX, LEAF, self.d_ds[0], self.d_m)
        loc.correct_device_async(self.d_ds[0], self.d_m, N_MAX, MIN_POINTS, t2)
        loc.sweep_to_world_async(self.d_ds[0], self.d_m, N_MAX, self.d_pub, self.d_pubn)
        loc.sweep_to_world_async(self.d_w[0], self.d_wn, N_MAX, self.d_full, self.d_fulln)
        if self.full:
            loc.cloud_stamp_async(self.d_ds[1], self.d_pubn, N_MAX, self.d_stamps)
            loc.cloud_stamp_async(self.d_w[1], self.d_fulln, N_MAX, self.d_stamps + 8)
        loc.map_add_last_sweep(True)
        loc.lidar_clear_async(t2 - EMPTY_LIDAR_TIME)

    def publish(self):
        """the tick's state read, and both published clouds on the host"""
        self.lv._check(self.loc.L.lv_get_state(self.loc.h, self.lv._d(self.x), self.lv._d(self.P)))
        for d_xyz, d_n, lanes in ((self.d_pub, self.d_pubn, self.d_ds), (self.d_full, self.d_fulln, self.d_w)):
            self.d2h(self.cnt, d_n, 8)
            m = int(self.cnt[0])
            self.d2h(self.host[0], d_xyz, 12 * m)
            if self.full:
                for h, d, b in zip(self.host[1:], lanes[1:], (8, 4, 4)):
                    self.d2h(h, d, b * m)
        if self.full:
            self.d2h(self.stamps, self.d_stamps, 16)

    def run(self, ticks):
        blocked, ev = [], []
        torch.cuda.synchronize()
        w0 = time.perf_counter()
        for _ in range(ticks):
            t2 = 10.0 + DELTA * (self.k + 1) + 0.1
            while 10.0 + 0.1 * self.received < t2:                 # the message that holds t2 has arrived
                self.receive(self.received)
                self.received += 1
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(self.stream)
            h0 = time.perf_counter()
            self.tick(t2)
            blocked.append(1e3 * (time.perf_counter() - h0))
            b.record(self.stream)
            self.publish()
            ev.append((a, b))
            self.k += 1
        wall = 1e3 * (time.perf_counter() - w0) / ticks
        torch.cuda.synchronize()
        dev = [a.elapsed_time(b) for a, b in ev]
        st = self.loc.async_status()
        assert st[0] == self.lv.OK, st
        return dict(host_blocked_ms=statistics.median(blocked), wall_ms=wall, device_ms=statistics.median(dev))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--ticks", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "full_points_timing"))
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    lv = G.load_package()
    world = lv.SynthWorld(20260924, 200000)
    prm = lv.params_from_yaml(os.path.join(lv.CONFIG_DIR, "xaloc.yaml"), max_map_points=1 << 21, max_points=N_MAX)
    msg, x = message(lv, world, prm, 65536)
    msg["intensity"] = np.random.default_rng(1).uniform(0, 255, len(msg)).astype(np.float32)
    chains = {"xyz": Chain(lv, prm, world, msg, x, False), "full": Chain(lv, prm, world, msg, x, True)}
    for c in chains.values():
        c.loc.map_set_growth(1 << 23)
        c.run(args.warmup)
    res = {k: {} for k in chains}
    for r in range(args.rounds):
        for k in (("xyz", "full") if r % 2 == 0 else ("full", "xyz")):
            for m, v in chains[k].run(args.ticks).items():
                res[k].setdefault(m, []).append(v)
    same = all(np.array_equal(a, b) for a, b in zip(chains["xyz"].loc.get_state(), chains["full"].loc.get_state()))
    row = {"workload": "xaloc 0.02 s windows, mapping online, both clouds published every tick", "points_per_message": len(msg),
           "card": card(), "rounds": args.rounds, "ticks": args.ticks, "same_state": bool(same),
           "window_points_last_tick": int(chains["full"].cnt[0]), "stamps_last_tick": [int(v) for v in chains["full"].stamps]}
    for k, v in res.items():
        row[k] = {m: {"median": statistics.median(s), "min": min(s), "max": max(s)} for m, s in v.items()}
    print(json.dumps(row), flush=True)
    with open(os.path.join(args.out, "full_points_timing.json"), "w") as f:
        json.dump([row], f, indent=1)
    for c in chains.values():
        c.loc.close()


if __name__ == "__main__":
    main()
