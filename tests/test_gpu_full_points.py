"""Full points through the device tick: intensity, range and time from the message to the published clouds.

The full voxel grid (lv_voxelgrid_downsample_full and its stream-ordered form) equals tests/full_points_ref.py bit for bit on every
family of tests/frontend_cases.py, and its xyz equals the xyz-only voxel grid's.  The LiDAR buffer with attribute lanes equals the
restated deque of whole Points on a ring that wraps several times, with 64-point ties at t2, late and overlapping messages, plain
pushes (lanes 0), re-reserves and a push that does not fit.  Windowed ticks from an empty map over Velodyne, Hesai and Ouster messages
run process -> full push -> full get -> compensate -> full voxel grid -> update -> world-frame clouds -> stamps on the device, and
match, tick for tick, a chain that decodes on the host, keeps the restated deque and runs the xyz-only synchronous calls: state, P,
logs, last_time_updated and the map bit for bit, the clouds' xyz as lv_match_all's world points, and their intensity, range, time,
counts and header stamps bit for bit."""
import ctypes as C

import numpy as np
import pytest

import frontend_cases as FC
import frontend_ref as F
import full_points_ref as P
from test_async_tick_args import BASE, CNT
from test_gpu_async_tick import Bufs, get_count, put_count
from test_gpu_cloud_frontend import FRT, host_process
from test_gpu_lidar_buffer import (COLS, EMPTY_LIDAR_TIME, IMU_ACC, IMU_GYRO, LEAF, MD, MIN_POINTS, RATE, RINGS, bits, velodyne_message,
                                   window_path)
from test_gpu_world_clouds import g_world, upload
from test_wire_format import DTYPES

pytestmark = pytest.mark.gpu
f32 = np.float32


@pytest.fixture(scope="module")
def loc(lv):
    h = lv.Localizer(lv.default_params(max_points=1 << 17, max_map_points=1 << 16))
    yield h
    h.close()


def attributes(rng, n):
    return rng.uniform(0, 1.7e9, n), rng.uniform(0, 255, n).astype(f32), rng.uniform(0, 120, n).astype(f32)


def same_full(got, ref, what):
    assert len(got[0]) == len(ref[0]), (what, len(got[0]), len(ref[0]))
    for name, a, b in zip(("xyz", "time", "intensity", "range"), got, ref):
        assert bits(a) == bits(b), (what, name)


# ---- the voxel grid ---------------------------------------------------------------------------------------------------------------
def test_voxelgrid_full_equals_the_restatement(lv, loc):
    rng = np.random.default_rng(17)
    seen = dict(overflow=0, leaves=0)
    for name, xyz, leaf in FC.voxel_cases():
        n = len(xyz)
        t, inten, rg = attributes(rng, n)
        ref = P.voxelgrid_full(xyz, t, inten, leaf)
        seen["overflow"] += F.voxel_cells(xyz, leaf)["overflow"]
        seen["leaves"] += len(ref[0])
        same_full(loc.voxelgrid_downsample_full(xyz, t, inten, leaf), ref, ("host", name))
        b = Bufs(loc)
        hi = n + 37                                                   # every range of n_max points must lie in its own buffer
        ins = [b(k * hi) for k in (12, 8, 4)]
        for d, a in zip(ins, (xyz, t, inten)):
            upload(loc, d, a)
        d_n, d_m, d_k = b(8), b(8), b(8)
        outs = [b(k * hi) for k in (12, 8, 4, 4)]
        d_plain = b(12 * hi)
        for n_max in (n, hi):
            put_count(loc, d_n, n)
            put_count(loc, d_m, -3)
            loc.voxelgrid_downsample_full_async(*ins, d_n, n_max, leaf, *outs, d_m)
            loc.voxelgrid_downsample_device_async(ins[0], d_n, n_max, leaf, d_plain, d_k)
            m = get_count(loc, d_m)
            assert m == len(ref[0]) == get_count(loc, d_k), (name, m)
            got = tuple(loc.download(d, np.empty((m, 3) if k == 0 else m, dt)) for k, (d, dt) in
                        enumerate(zip(outs, (f32, np.float64, f32, f32))))
            same_full(got, ref, ("device", name, n_max))
            assert bits(loc.download(d_plain, np.empty((m, 3), f32))) == bits(got[0]), name      # the xyz-only form's centroids
        assert loc.async_status() == (lv.OK, ""), name
        b.free()
    assert seen["overflow"] >= 1 and seen["leaves"] > 10000, seen


def test_voxelgrid_full_optional_outputs_counts_and_bound(lv, loc):
    rng = np.random.default_rng(2)
    xyz = rng.normal(0, 15, (5000, 3)).astype(f32)
    t, inten, rg = attributes(rng, 5000)
    b = Bufs(loc)
    ins = [b.upload(a) for a in (xyz, t, inten)]
    d_n, d_m = b(8), b(8)
    d_out, d_i = b(12 * 5000), b(4 * 5000)
    for k in (0, 1, 17, 3210):
        put_count(loc, d_n, k)
        loc.voxelgrid_downsample_full_async(*ins, d_n, 5000, 0.5, d_out, None, d_i, None, d_m)   # time and range not wanted
        ref = P.voxelgrid_full(xyz[:k], t[:k], inten[:k], 0.5)
        m = get_count(loc, d_m)
        assert m == len(ref[0]), k
        assert bits(loc.download(d_out, np.empty((m, 3), f32))) == bits(ref[0])
        assert bits(loc.download(d_i, np.empty(m, f32))) == bits(ref[2])
    assert loc.async_status() == (lv.OK, "")
    put_count(loc, d_n, 5001)                                         # a count above n_max: clamped and reported
    loc.voxelgrid_downsample_full_async(*ins, d_n, 5000, 0.5, d_out, None, None, None, d_m)
    assert get_count(loc, d_m) == len(P.voxelgrid_full(xyz, t, inten, 0.5)[0])
    st, msg = loc.async_status()
    assert st == lv.ERR_ARG and "outside [0, n_max]" in msg
    L = loc.L
    far = [BASE + (k << 30) for k in range(3)]                         # never dereferenced: refused before any device work
    assert L.lv_voxelgrid_downsample_full_device_async(loc.h, *far, CNT, (1 << 17) + 1, C.c_float(0.5), BASE + (8 << 30), None, None,
                                                       None, CNT + 8) == lv.ERR_ARG
    assert L.lv_last_error() == b"voxel grid full: n_max above max_points"
    b.free()


# ---- the buffer ---------------------------------------------------------------------------------------------------------------------
class FullBuffer:
    """the handle's buffer with lanes, with staging for messages and windows"""

    def __init__(self, loc, cap, n_max=1 << 14, full=True):
        self.loc, self.n_max = loc, n_max
        self.b = Bufs(loc)
        self.d_in = [self.b(k * n_max) for k in (12, 8, 4, 4)]
        self.d_out = [self.b(k * n_max) for k in (12, 8, 4, 4)]
        self.d_n, self.d_m = self.b(8), self.b(8)
        (loc.lidar_reserve_full if full else loc.lidar_reserve)(cap)

    def push(self, xyz, t, inten=None, rg=None):
        n = len(t)
        arrs = (np.ascontiguousarray(xyz, f32), np.ascontiguousarray(t, np.float64), inten, rg)
        for d, a in zip(self.d_in, arrs):
            if a is not None and n:
                upload(self.loc, d, np.ascontiguousarray(a))
        put_count(self.loc, self.d_n, n)
        if inten is None:
            self.loc.lidar_push_async(self.d_in[0], self.d_in[1], self.d_n, max(n, 1))
        else:
            self.loc.lidar_push_full_async(*self.d_in, self.d_n, max(n, 1))

    def get(self, t1, t2):
        put_count(self.loc, self.d_m, -9)
        self.loc.lidar_get_points_full_async(t1, t2, *self.d_out, self.n_max, self.d_m)
        m = get_count(self.loc, self.d_m)
        return tuple(self.loc.download(d, np.empty((m, 3) if k == 0 else m, dt)) for k, (d, dt) in
                     enumerate(zip(self.d_out, (f32, np.float64, f32, f32))))

    def get_plain(self, t1, t2):
        put_count(self.loc, self.d_m, -9)
        self.loc.lidar_get_points_async(t1, t2, self.d_out[0], self.d_out[1], self.n_max, self.d_m)
        m = get_count(self.loc, self.d_m)
        return self.loc.download(self.d_out[0], np.empty((m, 3), f32)), self.loc.download(self.d_out[1], np.empty(m))

    def close(self):
        self.b.free()


def same_window(dev, ref, t1, t2, what):
    r = ref.get(t1, t2)
    same_full(dev.get(t1, t2), r, (what, t1, t2))
    gx, gt = dev.get_plain(t1, t2)                                    # the plain get of the same ring: the same window
    assert bits(gx) == bits(r[0]) and bits(gt) == bits(r[1]), (what, t1, t2)
    return len(r[1])


def test_full_windows_on_a_wrapping_ring_equal_the_restatement(lv, loc):
    rng = np.random.default_rng(8)
    cap = 3 * 24 * RINGS + 100
    dev, ref = FullBuffer(loc, cap), P.LidarBufferFull()
    clock, pushed = 0.0, 0
    seen = dict(tie_t2=0, late=0, overlap=0, plain=0, reserve=0, full=0, nonempty=0)
    for i in range(60):
        kind = rng.random()
        cols = int(rng.integers(8, 25))
        start = clock - 0.05 if kind < 0.1 else clock - 0.008 if kind < 0.2 else clock
        seen["late"] += kind < 0.1
        seen["overlap"] += 0.1 <= kind < 0.2
        xyz, t = velodyne_message(rng, start, cols)
        plain = rng.random() < 0.15
        inten = None if plain else rng.uniform(0, 255, len(t)).astype(f32)
        rg = None if plain else rng.uniform(0, 90, len(t)).astype(f32)
        seen["plain"] += plain
        if ref.size() + len(t) > cap:
            if not seen["full"] or rng.random() < 0.3:               # a push that does not fit: a deferred error, nothing changes
                dev.push(xyz, t, inten, rg)
                st, msg = loc.async_status()
                assert st == lv.ERR_ARG and "lidar push" in msg, msg
                seen["full"] += 1
            ref.clear(np.inf)
            loc.lidar_clear_async(np.inf)
        dev.push(xyz, t, inten, rg)
        ref.push_message(xyz, t, inten, rg)
        pushed += len(t)
        clock = max(clock, start + cols * 1e-3 + 2e-3)
        col_times = np.unique(ref.times())
        for _ in range(3):
            if len(col_times) and rng.random() < 0.8:
                t2 = float(rng.choice(col_times))
                t1 = t2 - 1e-3 * int(rng.integers(0, 12))
                seen["tie_t2"] += 1
            else:
                t1, t2 = sorted(rng.uniform(clock - 0.1, clock + 0.01, 2))
            seen["nonempty"] += same_window(dev, ref, t1, t2, i) > 0
        if i % 17 == 16:                                              # re-reserve: the live points keep their lanes, in order
            new_cap = cap + 64 if i % 2 else max(cap - 64, ref.size())
            if rng.random() < 0.5:
                loc.lidar_reserve(new_cap)                            # the plain reserve keeps the lanes
            else:
                loc.lidar_reserve_full(new_cap)
            cap = new_cap
            seen["reserve"] += 1
            same_window(dev, ref, -np.inf, np.inf, ("reserve", i))
        assert loc.lidar_info()["points"] == ref.size()
    assert pushed > 3 * cap, pushed
    assert all(v > 0 for v in seen.values()), seen
    assert loc.async_status() == (lv.OK, "")
    loc.lidar_clear_async(np.inf)
    dev.close()


def test_ties_and_a_plain_ring_that_gains_lanes(lv):
    L = lv.lib()
    loc = lv.Localizer(lv.default_params(max_points=1 << 14, max_map_points=1 << 12))
    rng = np.random.default_rng(3)
    dev, ref = FullBuffer(loc, 4096, n_max=4096, full=False), P.LidarBufferFull()
    # full calls on a ring without lanes are refused before any device work
    assert L.lv_lidar_push_full_device_async(loc.h, *dev.d_in, dev.d_n, 1) == lv.ERR_ARG
    assert b"lv_lidar_reserve_full first" in L.lv_last_error()
    assert L.lv_lidar_get_points_full_device_async(loc.h, 0.0, 1.0, *dev.d_out, 1, dev.d_m) == lv.ERR_ARG
    assert b"lv_lidar_reserve_full first" in L.lv_last_error()
    xyz, t = velodyne_message(rng, 5.0, 10)
    dev.push(xyz, t)                                                  # plain, on a plain ring
    ref.push_message(xyz, t)
    loc.lidar_reserve_full(4096)                                      # same capacity: the lanes are added, the live points get 0
    assert loc.lidar_info()["capacity"] == 4096
    xyz, t = velodyne_message(rng, 5.01, 10)
    inten, rg = rng.uniform(1, 255, len(t)).astype(f32), rng.uniform(1, 90, len(t)).astype(f32)
    dev.push(xyz, t, inten, rg)
    ref.push_message(xyz, t, inten, rg)
    t2 = 5.01 + 1e-3 * 6                                             # 64 points tied at t2: two come out, the next window the rest
    assert same_window(dev, ref, 5.01 + 1e-3 * 3, t2, "ties") == 3 * RINGS + 2
    assert same_window(dev, ref, t2, 5.01 + 1e-3 * 9, "next") == 3 * RINGS + 2
    assert same_window(dev, ref, 0.0, 6.0, "all") == 20 * RINGS
    w = dev.get(0.0, 6.0)
    assert (w[2][:10 * RINGS] == 0).all() and (w[3][:10 * RINGS] == 0).all()
    assert (w[2][10 * RINGS:] > 0).all() and (w[3][10 * RINGS:] > 0).all()
    loc.lidar_reserve(3000)                                           # the plain reserve of a ring with lanes keeps them
    assert same_window(dev, ref, 0.0, 6.0, "kept") == 20 * RINGS
    assert loc.async_status() == (lv.OK, "")
    dev.close()
    loc.close()


# ---- stamps ------------------------------------------------------------------------------------------------------------------------
def test_stamps_equal_the_restatement(lv, loc):
    rng = np.random.default_rng(4)
    b = Bufs(loc)
    base = 1.7e9
    cases = [np.zeros(0), np.zeros(17), np.array([0.0078125]), np.array([base + 0.0078125, base, base + 0.0234375, base + 0.001]),
             base + np.sort(rng.uniform(0, 0.1, 70000)), np.nextafter(np.full(3, 0.0078125), 0.0),
             rng.uniform(0, 100, 5000), np.arange(1 << 16) * 1e-6 + 10.0]
    d_s = b(8)
    for k, t in enumerate(cases):
        n_max = max(len(t), 1)
        d_t, d_n = b.upload(t) if len(t) else b(8), b(8)
        for cnt in sorted({len(t), len(t) // 2}):
            put_count(loc, d_n, cnt)
            upload(loc, d_s, np.array([12345], np.uint64))
            loc.cloud_stamp_async(d_t, d_n, n_max, d_s)
            got = int(loc.download(d_s, np.zeros(1, np.uint64))[0])
            assert got == P.stamp_us(t[:cnt]), (k, cnt, got)
    assert loc.async_status() == (lv.OK, "")
    assert loc.L.lv_cloud_stamp_device_async(loc.h, BASE, CNT, (1 << 17) + 1, d_s) == lv.ERR_ARG
    assert loc.L.lv_last_error() == b"cloud stamp: n_max above max_points"
    b.free()


# ---- windowed ticks from an empty map ------------------------------------------------------------------------------------------------
def lidar_messages(lv, sc, lidar, n_msgs=7, cut=3):
    """messages at 10 Hz, 64 rings x COLS columns ring-major (the rings of a column share its time); message `cut` keeps only 300
    points so its windows fall below MIN_POINTS.  Velodyne: float intensity and relative float time; Hesai: uint8 intensity and
    absolute float64 time; Ouster: uint16 reflectivity, uint32 range and relative uint32 ns"""
    rng = np.random.default_rng(31)
    msgs = []
    for i in range(n_msgs):
        x = sc.world.pose(8.0 + 0.1 * i, sc.prm)
        sw = sc.world.sweep(x, rings=RINGS, azimuths=COLS, seed=200 + i)
        xyz = sw.reshape(COLS, RINGS, 3).transpose(1, 0, 2).reshape(-1, 3)
        rel = np.tile(np.arange(COLS), RINGS) * (0.099 / (COLS - 1))
        pts = np.zeros(len(xyz), DTYPES[lidar])
        pts["x"], pts["y"], pts["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
        if lidar == "velodyne":
            pts["intensity"] = rng.uniform(0, 255, len(xyz)).astype(f32)
            pts["time"] = rel.astype(f32)
        elif lidar == "hesai":
            pts["intensity"] = rng.integers(0, 256, len(xyz))
            pts["timestamp"] = 10.0 + 0.1 * i + rel
        else:
            pts["t"] = (rel * 1e9).astype(np.uint32)
            pts["reflectivity"] = rng.integers(0, 65536, len(xyz))
            pts["range"] = (np.linalg.norm(xyz, axis=1) * 1000).astype(np.uint32)
        if i == cut:
            pts = pts[:300]
        msgs.append(dict(pts=pts, raw=np.frombuffer(pts.tobytes(), np.uint8).copy(), n=len(pts), stamp=10_000_000 + 100_000 * i,
                         layout=lv.cloud_layout(lidar, pts.dtype)))
    return msgs


class FullChain:
    """main.cpp:61-122 (mapping online, high_quality_publish) over one LiDAR type's messages.  `device`: every stage on the device
    with the attribute lanes, both clouds published with their stamps, nothing read back but what the test inspects.  Otherwise the
    deque of full points lives in the restatement (host decode), the tick runs the xyz-only synchronous calls, and the published
    points are built by the restatement from the downloaded compensated window"""

    def __init__(self, lv, sc, lidar, msgs, delta, device):
        prm = lv.params_from_yaml(lv.CONFIG_DIR + "/xaloc.yaml", max_map_points=1 << 19, max_points=1 << 16)
        self.lv, self.sc, self.lidar, self.delta, self.device = lv, sc, lidar, delta, device
        self.loc = lv.Localizer(prm)
        self.loc.set_state(sc.x_prop, sc.P0)
        b = self.b = Bufs(self.loc)
        self.nm = max(g["n"] for g in msgs)
        nx = self.n_max = 1 << 16
        self.d_msg = b(max(len(g["raw"]) for g in msgs))
        self.d_p = [b(k * self.nm) for k in (12, 8, 4, 4)]            # processed message: xyz, time, intensity, range
        self.d_w = [b(k * nx) for k in (12, 8, 4, 4)]                 # window (compensated in place)
        self.d_ds = [b(k * nx) for k in (12, 8, 4, 4)]                # downsampled window
        self.d_pub, self.d_full = b(12 * nx), b(12 * nx)              # global_ds_compensated, global_compensated (xyz)
        self.d_k, self.d_wn, self.d_m, self.d_pubn, self.d_fulln, self.d_stamps = b(8), b(8), b(8), b(8), b(8), b(16)
        if device:
            self.loc.lidar_reserve_full(3 * self.nm // RATE)
        self.ref = P.LidarBufferFull()
        self.t2 = np.finfo(np.float64).max
        self.ltu = -1.0
        self.published = None

    def receive(self, g):
        loc = self.loc
        if not self.device:
            xyz, t, inten, rg, _ = host_process(self.lv, self.lidar, g["pts"], g["stamp"], True, True, FRT, RATE, MD)
            self.ref.push_message(xyz, t, inten, rg)
            return t
        upload(loc, self.d_msg, g["raw"])
        loc.process_cloud_device_async(self.lidar, g["layout"], self.d_msg, len(g["raw"]), g["n"], g["stamp"], True, True, FRT, RATE, MD,
                                       self.d_p[0], self.d_p[1], self.d_k, self.d_p[2], self.d_p[3])
        loc.lidar_push_full_async(*self.d_p, self.d_k, g["n"])
        return None

    def tick(self, latest):
        loc, delta, nx = self.loc, self.delta, self.n_max
        self.t2 = min(self.t2 + delta, latest)
        t2 = self.t2
        t1 = max(t2 - delta, self.ltu)
        if t2 - t1 < delta - 1e-6:
            return "fov"
        loc.propagate_device(IMU_ACC, IMU_GYRO, np.full(4, delta / 4))
        path, x2 = window_path(self.lv, self.sc, t1, t2)
        if self.device:
            loc.lidar_get_points_full_async(t1, t2, *self.d_w, nx, self.d_wn)
            loc.compensate_device_async(path, x2, self.d_w[0], self.d_w[1], self.d_wn, nx, self.d_w[0])
            loc.voxelgrid_downsample_full_async(*self.d_w[:3], self.d_wn, nx, LEAF, *self.d_ds, self.d_m)
            loc.correct_device_async(self.d_ds[0], self.d_m, nx, MIN_POINTS, t2)
            loc.sweep_to_world_async(self.d_ds[0], self.d_m, nx, self.d_pub, self.d_pubn)      # main.cpp:92-94
            loc.sweep_to_world_async(self.d_w[0], self.d_wn, nx, self.d_full, self.d_fulln)    # main.cpp:91, high_quality_publish
            loc.cloud_stamp_async(self.d_ds[1], self.d_pubn, nx, self.d_stamps)
            loc.cloud_stamp_async(self.d_w[1], self.d_fulln, nx, self.d_stamps + 8)
            loc.map_add_last_sweep(True)
            loc.lidar_clear_async(t2 - EMPTY_LIDAR_TIME)
            loc.get_state()
            self.published = self.download_published()
            gated = self.published["ds"][0].shape[0] == 0
        else:
            xyz, t, inten, rg = self.ref.get(t1, t2)
            m = 0
            if len(t):
                upload(loc, self.d_w[0], xyz)
                upload(loc, self.d_w[1], t)
                loc.compensate_device(path, x2, self.d_w[0], self.d_w[1], len(t), self.d_w[0])
                comp = loc.download(self.d_w[0], np.empty((len(t), 3), f32))
                m = loc.voxelgrid_downsample_device(self.d_w[0], len(t), LEAF, self.d_ds[0])
            gated = m < MIN_POINTS                                    # main.cpp:81
            if not gated:
                loc.correct_device(self.d_ds[0], m, t2)
                loc.map_add_last_sweep(True)
                self.ref.clear(t2 - EMPTY_LIDAR_TIME)
                x, _ = loc.get_state()
                ds = P.voxelgrid_full(comp, t, inten, LEAF)
                assert bits(ds[0]) == bits(loc.download(self.d_ds[0], np.empty((m, 3), f32)))
                self.published = dict(ds=(g_world(loc, x, ds[0]),) + ds[1:], full=(g_world(loc, x, comp), t, inten, rg),
                                      stamps=(P.stamp_us(ds[1]), P.stamp_us(t)))
        self.ltu = loc.last_time_updated()
        return "gated" if gated else "tick"

    def download_published(self):
        loc = self.loc
        out = {}
        for key, d_xyz, d_n, lanes in (("ds", self.d_pub, self.d_pubn, self.d_ds), ("full", self.d_full, self.d_fulln, self.d_w)):
            k = get_count(loc, d_n)
            out[key] = (loc.download(d_xyz, np.empty((k, 3), f32)), loc.download(lanes[1], np.empty(k)),
                        loc.download(lanes[2], np.empty(k, f32)), loc.download(lanes[3], np.empty(k, f32)))
        out["stamps"] = tuple(int(v) for v in loc.download(self.d_stamps, np.zeros(2, np.uint64)))
        return out

    def result(self):
        st, logs = self.loc.last_logs()
        x, P_ = self.loc.get_state()
        return st, logs, x, P_, self.loc.last_time_updated()

    def close(self):
        self.b.free()
        self.loc.close()


@pytest.mark.parametrize("lidar", ["velodyne", "hesai", "ouster"])
def test_windowed_full_ticks_equal_the_host_chain(lv, scene_xaloc, lidar):
    sc = scene_xaloc
    msgs = lidar_messages(lv, sc, lidar)
    host, dev = FullChain(lv, sc, lidar, msgs, 0.02, False), FullChain(lv, sc, lidar, msgs, 0.02, True)
    seen = dict(ticks=0, gated=0, updates=0, ties=0, attrs=0)
    latest = -np.inf
    for i, g in enumerate(msgs):
        t_msg = host.receive(g)
        dev.receive(g)
        latest = max(latest, float(t_msg.max()))
        for _ in range(14):
            a, b = host.tick(latest), dev.tick(latest)
            assert a == b and host.t2 == dev.t2, (i, a, b, host.t2, dev.t2)
            if a == "fov":
                break
            seen["ticks"] += 1
            rh, rd = host.result(), dev.result()
            assert bits(rh[2]) == bits(rd[2]) and bits(rh[3]) == bits(rd[3]) and rh[4] == rd[4], (i, host.t2)
            assert bits(host.loc.map_points()) == bits(dev.loc.map_points()), (i, host.t2)
            pd = dev.published
            if a == "gated":
                seen["gated"] += 1
                assert len(pd["ds"][0]) == 0 and len(pd["full"][0]) == 0 and pd["stamps"] == (0, 0), (i, host.t2)
                continue
            seen["updates"] += rh[0] == lv.OK
            assert rh[0] == rd[0] and len(rh[1]) == len(rd[1]) and all(
                all(np.array_equal(p[k], q[k], equal_nan=True) for k in p) for p, q in zip(rh[1], rd[1])), (i, host.t2)
            ph = host.published
            for key in ("ds", "full"):
                same_full(pd[key], ph[key], (lidar, i, host.t2, key))
            assert pd["stamps"] == ph["stamps"] and ph["stamps"][0] == 0, (i, pd["stamps"], ph["stamps"])
            assert ph["stamps"][1] == P.stamp_us(ph["full"][1]) > 0
            seen["ties"] += int((ph["full"][1] == host.t2).sum()) == 2
            seen["attrs"] += bool((ph["full"][2] > 0).any() and (ph["ds"][2] > 0).any())
    assert dev.loc.async_status() == (lv.OK, "")
    assert seen["ticks"] >= 20 and seen["gated"] >= 1 and seen["updates"] >= 8 and seen["ties"] >= 1, seen
    assert seen["attrs"] >= seen["ticks"] - seen["gated"] - 1, seen
    assert len(dev.loc.map_points()) > 1000
    host.close()
    dev.close()
