"""The tick's output and mapping step (main.cpp:88-117) on the device against the same step through host round trips, in one run,
alternating them round by round.  Velodyne 64 x 1024 messages arrive at 10 Hz into the LiDAR buffer in HBM; the tick localizes on
xaloc's 0.02 s windows, publishes the full-resolution window in the world frame (high_quality_publish: global_compensated, the
cloud is downloaded for the publisher) and, with mapping_online false, maps the last full rotation every full_rotation_time:

  device  lv_sweep_to_world_device_async of the compensated window, its count and points downloaded;
          offline map: get_points(t2 - 0.1, t2) -> compensate -> lv_sweep_to_world_device_async -> voxel grid ->
          lv_map_add_device_async, counts on the device
  host    the compensated window and its count downloaded, the state read, the world frame computed on the host (the oracle's
          fp32 restatement of State.cpp:79-89, the reference's own arithmetic);
          offline map: the full rotation's count read back, compensated, downloaded, transformed on the host, lv_voxelgrid_downsample
          and lv_map_add on host buffers

Both chains share the rest of the tick (get, compensate, voxel grid, lv_correct_device_async, clear).  Per tick it reports
  host_blocked_ms  host time inside the tick's calls before the state read (host transforms and round trips included)
  wall_ms          host time of the whole tick, state read and published cloud included, ticks back to back (receives amortised)
  device_ms        CUDA events on the handle's stream around the tick's work
for all ticks and for the mapping ticks alone, as the median over --rounds rounds of --ticks ticks each, after --warmup ticks.  The
card's name, power limit and SM clock are read in the same run.  Prints one JSON line and writes OUT/world_clouds_timing.json.
    python tools/world_clouds_timing.py [--rounds 5] [--ticks 50] [--warmup 10] [--out DIR]   (DIR: <tmp>/world_clouds_timing)
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
    def __init__(self, lv, O, prm, world, msg, x, device):
        self.lv, self.O, self.msg, self.device = lv, O, msg, device
        self.stream = torch.cuda.Stream()
        prm.stream = self.stream.cuda_stream
        self.loc = lv.Localizer(prm)
        self.loc.map_build(world.map())
        x0, P0 = self.loc.get_state()
        self.loc.set_state(x, P0)
        self.prm, self.xs = prm, x
        self.oprm = O.make_params()
        self.omap = O.Map()
        self.omap.build(np.zeros((1, 3), np.float32))               # the oracle's match_all computes the world points of any state
        self.n = len(msg)
        self.lay = lv.cloud_layout("velodyne", msg.dtype)
        self.d_msg = self.loc.upload(msg)
        a = self.loc.device_alloc
        self.d_pxyz, self.d_pt, self.d_k = a(12 * self.n), a(8 * self.n), a(8)
        self.d_wxyz, self.d_wt, self.d_w = a(12 * N_MAX), a(8 * N_MAX), a(8)
        self.d_ds, self.d_m, self.d_pub, self.d_pubn = a(12 * N_MAX), a(8), a(12 * N_MAX), a(8)
        self.d_fxyz, self.d_ft, self.d_f, self.d_fds, self.d_fm = a(12 * N_MAX), a(8 * N_MAX), a(8), a(12 * N_MAX), a(8)
        self.loc.lidar_reserve(6 * self.n)
        self.k, self.received, self.last_map_time = 0, 0, -1.0
        self.paths = {}
        self.x, self.P = np.zeros(lv.STATE_LEN), np.zeros((lv.DOF, lv.DOF))
        self.pub = np.empty((N_MAX, 3), np.float32)
        self.cnt = np.zeros(1, np.int64)

    def path(self, t1, t2):
        key = (round(t1, 9), round(t2, 9))
        if key not in self.paths:
            self.paths[key] = path_for(self.lv, self.prm, self.xs, t1, t2)
        return self.paths[key]

    def receive(self, j):
        loc, stamp = self.loc, 10_000_000 + 100_000 * j
        loc.process_cloud_device_async("velodyne", self.lay, self.d_msg, self.msg.nbytes, self.n, stamp, True, True, FRT, 1, 1.0,
                                       self.d_pxyz, self.d_pt, self.d_k)
        loc.lidar_push_async(self.d_pxyz, self.d_pt, self.d_k, self.n)

    def d2h(self, out, d, nbytes):
        if nbytes:
            self.lv._check(self.loc.L.lv_memcpy_d2h(self.loc.h, out.ctypes.data_as(C.c_void_p), C.c_void_p(d), nbytes))

    def to_world_host(self, d_xyz, d_n=None, m=0):
        """the round trip: the count (unless the host has it), the points and the state come back; the world frame is computed on
        the host"""
        if d_n is not None:
            self.d2h(self.cnt, d_n, 8)
            m = int(self.cnt[0])
        pts = np.empty((m, 3), np.float32)
        self.d2h(pts, d_xyz, 12 * m)
        self.lv._check(self.loc.L.lv_get_state(self.loc.h, self.lv._d(self.x), None))
        return self.omap.match_all(self.x, self.oprm, pts)["g"] if m else pts

    def has_to_map(self, t2):                                      # Mapper::hasToMap (Mapper.cpp:58-61)
        if self.last_map_time < 0:
            self.last_map_time = t2
        return t2 - self.last_map_time >= FRT

    def tick(self, t2):
        """returns the published cloud (None: it is still on the device) and whether the tick mapped"""
        loc, t1 = self.loc, t2 - DELTA
        path, x2 = self.path(t1, t2)
        loc.lidar_get_points_async(t1, t2, self.d_wxyz, self.d_wt, N_MAX, self.d_w)
        loc.compensate_device_async(path, x2, self.d_wxyz, self.d_wt, self.d_w, N_MAX, self.d_wxyz)
        loc.voxelgrid_downsample_device_async(self.d_wxyz, self.d_w, N_MAX, LEAF, self.d_ds, self.d_m)
        loc.correct_device_async(self.d_ds, self.d_m, N_MAX, MIN_POINTS, t2)
        mapped = self.has_to_map(t2)
        if mapped:
            self.last_map_time = t2                                  # Mapper::add (Mapper.cpp:29)
        if self.device:
            loc.sweep_to_world_async(self.d_wxyz, self.d_w, N_MAX, self.d_pub, self.d_pubn)
            if mapped:
                fpath, fx2 = self.path(t2 - FRT, t2)
                loc.lidar_get_points_async(t2 - FRT, t2, self.d_fxyz, self.d_ft, N_MAX, self.d_f)
                loc.compensate_device_async(fpath, fx2, self.d_fxyz, self.d_ft, self.d_f, N_MAX, self.d_fxyz)
                loc.sweep_to_world_async(self.d_fxyz, self.d_f, N_MAX, self.d_fxyz, self.d_f)
                loc.voxelgrid_downsample_device_async(self.d_fxyz, self.d_f, N_MAX, LEAF, self.d_fds, self.d_fm)
                loc.map_add_device_async(self.d_fds, self.d_fm, N_MAX, True)
            loc.lidar_clear_async(t2 - EMPTY_LIDAR_TIME)
            return None, mapped
        pub = self.to_world_host(self.d_wxyz, self.d_w)
        if mapped:
            fpath, fx2 = self.path(t2 - FRT, t2)
            kf = loc.lidar_get_points(t2 - FRT, t2, self.d_fxyz, self.d_ft, N_MAX)
            loc.compensate_device(fpath, fx2, self.d_fxyz, self.d_ft, kf, self.d_fxyz)
            loc.map_add(loc.voxelgrid_downsample(self.to_world_host(self.d_fxyz, m=kf), LEAF), True)
        loc.lidar_clear_async(t2 - EMPTY_LIDAR_TIME)
        return pub, mapped

    def publish(self, pub):
        """the tick's state read, and the published cloud on the host"""
        self.lv._check(self.loc.L.lv_get_state(self.loc.h, self.lv._d(self.x), self.lv._d(self.P)))
        if pub is None:
            self.d2h(self.cnt, self.d_pubn, 8)
            self.d2h(self.pub, self.d_pub, 12 * int(self.cnt[0]))

    def run(self, ticks):
        blocked, ev, mapped_at = [], [], []
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
            pub, mapped = self.tick(t2)
            blocked.append(1e3 * (time.perf_counter() - h0))
            b.record(self.stream)
            self.publish(pub)
            ev.append((a, b))
            mapped_at.append(mapped)
            self.k += 1
        wall = 1e3 * (time.perf_counter() - w0) / ticks
        torch.cuda.synchronize()
        dev = [a.elapsed_time(b) for a, b in ev]
        st = self.loc.async_status()
        assert st[0] == self.lv.OK, st
        sel = lambda v: [x for x, m in zip(v, mapped_at) if m]
        return dict(host_blocked_ms=statistics.median(blocked), wall_ms=wall, device_ms=statistics.median(dev),
                    host_blocked_ms_mapping=statistics.median(sel(blocked)), device_ms_mapping=statistics.median(sel(dev)))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--ticks", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "world_clouds_timing"))
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    lv, O = G.load_package(), G.load_oracle()
    world = lv.SynthWorld(20260924, 200000)
    prm = lv.params_from_yaml(os.path.join(lv.CONFIG_DIR, "xaloc.yaml"), max_map_points=1 << 21, max_points=N_MAX)
    msg, x = message(lv, world, prm, 65536)
    chains = {"host_round_trip": Chain(lv, O, prm, world, msg, x, False), "device": Chain(lv, O, prm, world, msg, x, True)}
    for c in chains.values():
        c.loc.map_set_growth(1 << 23)
        c.run(args.warmup)
    res = {k: {} for k in chains}
    for r in range(args.rounds):
        for k in (("host_round_trip", "device") if r % 2 == 0 else ("device", "host_round_trip")):
            for m, v in chains[k].run(args.ticks).items():
                res[k].setdefault(m, []).append(v)
    row = {"workload": "xaloc 0.02 s windows, high_quality_publish, mapping_online false", "points_per_message": len(msg),
           "card": card(), "rounds": args.rounds, "ticks": args.ticks,
           "map_points": {k: c.loc.map_size() for k, c in chains.items()}}
    for k, v in res.items():
        row[k] = {m: {"median": statistics.median(s), "min": min(s), "max": max(s)} for m, s in v.items()}
    print(json.dumps(row), flush=True)
    with open(os.path.join(args.out, "world_clouds_timing.json"), "w") as f:
        json.dump([row], f, indent=1)
    for c in chains.values():
        c.loc.close()


if __name__ == "__main__":
    main()
