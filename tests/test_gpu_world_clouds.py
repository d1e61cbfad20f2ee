"""The tick's output and mapping step on the device (main.cpp:88-117).

lv_sweep_to_world_device_async equals lv_match_all's g_world (the world points Mapper::match computes, pinned to the oracle
elsewhere) bit for bit at the same state: counts 0, 1, n_max and below, in place, far from the origin, a tick the MAX_POINTS2MATCH
gate stopped (count 0) and the first tick on an empty map (the propagated state).  lv_map_add_device_async equals lv_map_add_device
with the count on the host; applied to the published global_ds_compensated it leaves the map lv_map_add_last_sweep leaves, tick
after tick.  A windowed sequence with mapping_online false (main.cpp:106-117) run on the device equals the chain that downloads the
compensated full rotation, transforms it with the oracle and maps it through the host-buffer calls."""
import ctypes as C

import numpy as np
import pytest

from test_async_tick_args import BASE, CNT, OUT
from test_gpu_async_tick import Bufs, get_count, put_count
from test_gpu_cloud_frontend import FRT
from test_gpu_lidar_buffer import EMPTY_LIDAR_TIME, IMU_ACC, IMU_GYRO, LEAF, MIN_POINTS, RATE, MD, bits, sequence_messages, window_path
from test_world_clouds_args import RefMapper

pytestmark = pytest.mark.gpu
OFFSETS = [(0.0, 0.0, 0.0), (2e5, -3e5, 50.0)]
USAGE = ("points", "slots_used", "blocks_used", "arena_top", "error_flags", "capacity_points")


def upload(loc, d, arr):
    arr = np.ascontiguousarray(arr)
    assert loc.L.lv_memcpy_h2d(loc.h, C.c_void_p(d), arr.ctypes.data_as(C.c_void_p), arr.nbytes) == 0


def g_world(loc, x, xyz):
    """the world points of lv_match_all (x: the state; the handle's map must not be empty)"""
    out = loc.match_all(x, xyz)
    assert out["status"] == 0
    return out["g"]


def shifted(x, off):
    x = x.copy()
    x[0:3] += off
    return x


# ---- the transform ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("off", OFFSETS)
def test_transform_equals_match_all_g_world(lv, scene_xaloc, off):
    sc = scene_xaloc
    loc = lv.Localizer(sc.prm)
    b = Bufs(loc)
    loc.map_build(sc.map)
    x = shifted(sc.x_prop, off)
    loc.set_state(x, sc.P0)
    sw = sc.sweep
    n = len(sw)
    d_in, d_out, d_n, d_k = b.upload(sw), b(12 * n), b(8), b(8)
    sentinel = np.full((n, 3), 7.25, np.float32)
    for k, n_max, inplace, same_count in [(0, n, False, False), (1, n, False, False), (n, n, False, False), (n // 3, n, False, False),
                                          (n - 1, n - 1, False, False), (n, n, True, False), (n - 5, n, True, True)]:
        upload(loc, d_in, sw)
        upload(loc, d_out, sentinel)
        put_count(loc, d_n, k)
        put_count(loc, d_k, -3)
        dst, cnt = (d_in if inplace else d_out), (d_n if same_count else d_k)
        loc.sweep_to_world_async(d_in, d_n, n_max, dst, cnt)
        assert get_count(loc, cnt) == k, (k, n_max, inplace)
        got = loc.download(dst, np.empty((n, 3), np.float32))
        if k:
            assert bits(got[:k]) == bits(g_world(loc, x, sw[:k])), (k, n_max, inplace)
        rest = sw[k:] if inplace else sentinel[k:]
        assert bits(got[k:]) == bits(rest), (k, n_max, inplace)            # nothing past the count is written
    upload(loc, d_in, sw)                                            # the last case transformed it in place
    # a device count above n_max is clamped and reported
    put_count(loc, d_n, n + 3)
    loc.sweep_to_world_async(d_in, d_n, n - 10, d_out, d_k)
    assert get_count(loc, d_k) == n - 10
    st, msg = loc.async_status()
    assert st == lv.ERR_ARG and "outside [0, n_max]" in msg
    assert loc.L.lv_sweep_to_world_device_async(loc.h, BASE, CNT, sc.prm.max_points + 1, OUT, CNT + 8) == lv.ERR_ARG
    assert loc.L.lv_last_error() == b"sweep to world: n_max above max_points"
    # a tick the gate stopped publishes nothing; the next one publishes with the state its update left
    put_count(loc, d_n, MIN_POINTS - 1)
    loc.correct_device_async(d_in, d_n, n, MIN_POINTS, 1.0)
    put_count(loc, d_k, n)
    upload(loc, d_out, sentinel)
    loc.sweep_to_world_async(d_in, d_k, n, d_out, d_k)
    assert get_count(loc, d_k) == 0
    assert bits(loc.download(d_out, np.empty((n, 3), np.float32))) == bits(sentinel)
    assert loc.last_logs()[0] == lv.TOO_FEW_POINTS
    put_count(loc, d_n, n)
    loc.correct_device_async(d_in, d_n, n, MIN_POINTS, 2.0)
    loc.sweep_to_world_async(d_in, d_n, n, d_out, d_k)
    assert get_count(loc, d_k) == n
    got = loc.download(d_out, np.empty((n, 3), np.float32))
    x2, _ = loc.get_state()
    st = loc.last_logs()[0]
    if off == OFFSETS[0]:                                            # far from the map the update finds too few matches
        assert st == lv.OK and not np.array_equal(x2, x)
    assert st != lv.TOO_FEW_POINTS
    assert bits(got) == bits(g_world(loc, x2, sw))
    assert loc.async_status() == (lv.OK, "")
    b.free()
    loc.close()


@pytest.mark.parametrize("off", OFFSETS)
def test_transform_on_the_first_tick_uses_the_propagated_state(lv, scene_xaloc, off):
    sc = scene_xaloc
    loc = lv.Localizer(sc.prm)
    b = Bufs(loc)
    loc.set_state(shifted(sc.x_prop, off), sc.P0)
    loc.propagate_device(IMU_ACC, IMU_GYRO, np.full(4, 0.025))
    sw = sc.sweep
    n = len(sw)
    d_in, d_out, d_n, d_k = b.upload(sw), b(12 * n), b(8), b(8)
    put_count(loc, d_n, n)
    assert loc.correct_device_async(d_in, d_n, n, MIN_POINTS, 0.1) == lv.EMPTY_MAP
    loc.sweep_to_world_async(d_in, d_n, n, d_out, d_k)
    assert get_count(loc, d_k) == n
    got = loc.download(d_out, np.empty((n, 3), np.float32))
    loc.map_add_last_sweep(True)                                     # the first tick's build, with the same state
    x, _ = loc.get_state()
    assert not np.array_equal(x, shifted(sc.x_prop, off))           # propagated
    assert bits(got) == bits(g_world(loc, x, sw))
    b.free()
    loc.close()


# ---- the add with a device count ---------------------------------------------------------------------------------------------------
def map_state(loc):
    info = loc.map_info()
    return loc.map_points(), {k: info[k] for k in USAGE}


@pytest.mark.parametrize("growth", [False, True])
def test_async_add_equals_sync_add(lv, scene_xaloc, growth):
    sc = scene_xaloc
    prm = lv.params_from_yaml(lv.CONFIG_DIR + "/xaloc.yaml", max_map_points=1 << 13 if growth else 1 << 18, max_points=1 << 14)
    sync, asyn = lv.Localizer(prm), lv.Localizer(prm)
    if growth:
        sync.map_set_growth(1 << 18)
        asyn.map_set_growth(1 << 18)
    bs, ba = Bufs(sync), Bufs(asyn)
    rng = np.random.default_rng(11)
    n_max = 6000
    d_s, d_a, d_n = bs(12 * n_max), ba(12 * n_max), ba(8)
    # (points, downsample, device count); None: count above n_max (a deferred error; the add takes n_max points)
    steps = [(0, 1, 0), (4000, 1, 4000), (6000, 0, 6000), (3000, 1, 3000), (0, 1, 0), (6000, 1, 6000), (6000, 1, None), (2500, 0, 2500)]
    for i, (k, ds, dev) in enumerate(steps):
        pts = sc.map[rng.integers(0, len(sc.map), n_max)] + rng.normal(0, 0.05, (n_max, 3)).astype(np.float32)
        pts = np.ascontiguousarray(pts, np.float32)
        upload(sync, d_s, pts)
        upload(asyn, d_a, pts)
        put_count(asyn, d_n, n_max + 9 if dev is None else dev)
        sync.map_add_device(d_s, k if dev is not None else n_max, ds)
        asyn.map_add_device_async(d_a, d_n, n_max, ds)
        st, msg = asyn.async_status()
        assert (st == lv.ERR_ARG and "outside [0, n_max]" in msg) if dev is None else (st, msg) == (lv.OK, ""), (i, st, msg)
        (ps, us), (pa, ua) = map_state(sync), map_state(asyn)
        if us["capacity_points"] != ua["capacity_points"]:           # the growth bound is n_max: a re-hash recounts the slots
            for key in ("slots_used", "blocks_used", "capacity_points"):
                us.pop(key), ua.pop(key)
        assert us == ua, (i, us, ua)
        assert bits(ps) == bits(pa), i
    assert us["points"] > 10000
    if growth:
        assert asyn.map_info()["growths"] >= 1
    assert asyn.L.lv_map_add_device_async(asyn.h, BASE, CNT, prm.max_points + 1, 1) == lv.ERR_ARG
    assert asyn.L.lv_last_error() == b"map add async: n_max above max_points"
    bs.free()
    ba.free()
    sync.close()
    asyn.close()


def test_published_cloud_added_async_equals_add_last_sweep(lv, scene_xaloc):
    """main.cpp:91-105: map.add(global_ds_compensated) through the published cloud leaves the map lv_map_add_last_sweep leaves"""
    sc = scene_xaloc
    a, b = lv.Localizer(sc.prm), lv.Localizer(sc.prm)
    ba, bb = Bufs(a), Bufs(b)
    n_max = 1 << 14
    d_a, d_an = ba(12 * n_max), ba(8)
    d_b, d_bn, d_w, d_wn = bb(12 * n_max), bb(8), bb(12 * n_max), bb(8)
    for h in (a, b):
        h.set_state(sc.x_prop, sc.P0)
    seen = dict(gated=0, ok=0)
    for k in range(14):
        x = sc.world.pose(8.0 + 0.05 * k, sc.prm)
        sw = sc.world.sweep(x, rings=32, azimuths=256, seed=300 + k)[: (40 if k == 4 else None)]
        sw = lv_voxel(sw)
        m = len(sw)
        for h, d, dn in ((a, d_a, d_an), (b, d_b, d_bn)):
            upload(h, d, sw)
            put_count(h, dn, m)
            h.propagate_device(IMU_ACC, IMU_GYRO, np.full(4, 0.0125))
            h.correct_device_async(d, dn, n_max, MIN_POINTS, 0.05 * (k + 1))
        a.map_add_last_sweep(True)
        b.sweep_to_world_async(d_b, d_bn, n_max, d_w, d_wn)
        b.map_add_device_async(d_w, d_wn, n_max, True)
        ra, rb = a.last_logs(), b.last_logs()
        xa, Pa = a.get_state()
        xb, Pb = b.get_state()
        assert ra[0] == rb[0] and bits(xa) == bits(xb) and bits(Pa) == bits(Pb), k
        assert a.last_time_updated() == b.last_time_updated()
        assert bits(a.map_points()) == bits(b.map_points()), k
        seen["gated"] += get_count(b, d_wn) == 0
        seen["ok"] += ra[0] == lv.OK
    assert seen["gated"] >= 1 and seen["ok"] >= 6, seen
    assert a.async_status() == (lv.OK, "") and b.async_status() == (lv.OK, "")
    for bf, h in ((ba, a), (bb, b)):
        bf.free()
        h.close()


def lv_voxel(sw):
    """a coarse decimation that keeps the sweep well above MAX_POINTS2MATCH"""
    return np.ascontiguousarray(sw[::3], np.float32)


# ---- mapping offline: a windowed sequence -----------------------------------------------------------------------------------------
class OfflineChain:
    """main.cpp:61-122 with mapping_online false over Velodyne messages in the LiDAR buffer: `device` enqueues the tick's chain and
    the full-rotation map add with counts on the device; otherwise every count comes back to the host, the compensated full rotation
    is downloaded, transformed by the oracle and mapped through the host-buffer calls"""

    def __init__(self, lv, O, sc, msgs, delta, device):
        prm = lv.params_from_yaml(lv.CONFIG_DIR + "/xaloc.yaml", max_map_points=1 << 19, max_points=1 << 16)
        self.lv, self.O, self.sc, self.msgs, self.delta, self.device = lv, O, sc, msgs, delta, device
        self.loc = lv.Localizer(prm)
        self.loc.set_state(sc.x_prop, sc.P0)
        self.b = Bufs(self.loc)
        self.nm = max(g["n"] for g in msgs)
        self.n_max = 1 << 16
        self.d_msg = self.b(max(len(g["raw"]) for g in msgs))
        self.d_pxyz, self.d_pt, self.d_k = self.b(12 * self.nm), self.b(8 * self.nm), self.b(8)
        self.d_wxyz, self.d_wt, self.d_w = self.b(12 * self.n_max), self.b(8 * self.n_max), self.b(8)
        self.d_ds, self.d_m, self.d_pub, self.d_pubn = self.b(12 * self.n_max), self.b(8), self.b(12 * self.n_max), self.b(8)
        self.d_fxyz, self.d_ft, self.d_f, self.d_fds, self.d_fm = (self.b(12 * self.n_max), self.b(8 * self.n_max), self.b(8),
                                                                   self.b(12 * self.n_max), self.b(8))
        self.loc.lidar_reserve(3 * self.nm // RATE)
        self.mapper = RefMapper(FRT)
        self.oracle_map = O.Map()
        self.oracle_map.build(np.zeros((1, 3), np.float32))           # match_all needs a map; only its world points are used
        self.t2 = np.finfo(np.float64).max
        self.ltu = -1.0
        self.maps = 0

    def receive(self, g):
        loc = self.loc
        upload(loc, self.d_msg, g["raw"])
        args = ("velodyne", g["layout"], self.d_msg, len(g["raw"]), g["n"], g["stamp"], True, True, FRT, RATE, MD, self.d_pxyz, self.d_pt)
        loc.process_cloud_device_async(*args, self.d_k)
        loc.lidar_push_async(self.d_pxyz, self.d_pt, self.d_k, g["n"])
        return loc.download(self.d_pt, np.empty(get_count(loc, self.d_k)))

    def tick(self, latest):
        loc, delta = self.loc, self.delta
        self.t2 = min(self.t2 + delta, latest)
        t2 = self.t2
        t1 = max(t2 - delta, self.ltu)
        if t2 - t1 < delta - 1e-6:
            return "fov"
        loc.propagate_device(IMU_ACC, IMU_GYRO, np.full(4, delta / 4))
        path, x2 = window_path(self.lv, self.sc, t1, t2)
        if self.device:
            loc.lidar_get_points_async(t1, t2, self.d_wxyz, self.d_wt, self.n_max, self.d_w)
            loc.compensate_device_async(path, x2, self.d_wxyz, self.d_wt, self.d_w, self.n_max, self.d_wxyz)
            loc.voxelgrid_downsample_device_async(self.d_wxyz, self.d_w, self.n_max, LEAF, self.d_ds, self.d_m)
            loc.correct_device_async(self.d_ds, self.d_m, self.n_max, MIN_POINTS, t2)
            loc.sweep_to_world_async(self.d_ds, self.d_m, self.n_max, self.d_pub, self.d_pubn)   # publish global_ds_compensated
            st, _ = loc.last_logs()                                   # the tick's state read
            gated = get_count(loc, self.d_pubn) == 0                  # the publisher reads the count with the cloud
            if loc.L.lv_map_exists(loc.h) and self.ltu >= 0:
                assert gated == (st == self.lv.TOO_FEW_POINTS), (t2, st)
        else:
            k = loc.lidar_get_points(t1, t2, self.d_wxyz, self.d_wt, self.n_max)
            m = 0
            if k:
                loc.compensate_device(path, x2, self.d_wxyz, self.d_wt, k, self.d_wxyz)
                m = loc.voxelgrid_downsample_device(self.d_wxyz, k, LEAF, self.d_ds)
            gated = m < MIN_POINTS                                    # main.cpp:81
            if not gated:
                loc.correct_device(self.d_ds, m, t2)
        if gated:
            return "gated"
        if self.mapper.hasToMap(t2):                                  # main.cpp:106-117
            fpath, fx2 = window_path(self.lv, self.sc, t2 - FRT, t2)
            if self.device:
                loc.lidar_get_points_async(t2 - FRT, t2, self.d_fxyz, self.d_ft, self.n_max, self.d_f)
                loc.compensate_device_async(fpath, fx2, self.d_fxyz, self.d_ft, self.d_f, self.n_max, self.d_fxyz)
                loc.sweep_to_world_async(self.d_fxyz, self.d_f, self.n_max, self.d_fxyz, self.d_f)
                loc.voxelgrid_downsample_device_async(self.d_fxyz, self.d_f, self.n_max, LEAF, self.d_fds, self.d_fm)
                loc.map_add_device_async(self.d_fds, self.d_fm, self.n_max, True)
            else:
                kf = loc.lidar_get_points(t2 - FRT, t2, self.d_fxyz, self.d_ft, self.n_max)
                loc.compensate_device(fpath, fx2, self.d_fxyz, self.d_ft, kf, self.d_fxyz)
                full = loc.download(self.d_fxyz, np.empty((kf, 3), np.float32))
                x, _ = loc.get_state()
                g = self.oracle_map.match_all(x, self.sc.oprm, full)["g"]
                loc.map_add(loc.voxelgrid_downsample(g, LEAF), True)
            self.mapper.add(t2)
            self.maps += 1
        loc.lidar_clear_async(t2 - EMPTY_LIDAR_TIME)                  # main.cpp:122
        loc.get_state()
        self.ltu = loc.last_time_updated()
        return "tick"

    def result(self):
        st, logs = self.loc.last_logs()
        x, P = self.loc.get_state()
        return st, logs, x, P, self.loc.last_time_updated()

    def close(self):
        self.b.free()
        self.loc.close()


def test_offline_mapping_sequence_equals_the_host_round_trip_chain(lv, O, scene_xaloc):
    sc = scene_xaloc
    msgs = sequence_messages(lv, sc)
    host, dev = OfflineChain(lv, O, sc, msgs, 0.02, False), OfflineChain(lv, O, sc, msgs, 0.02, True)
    seen = dict(ticks=0, gated=0, updates=0)
    latest = -np.inf
    for i, g in enumerate(msgs):
        t_msg = host.receive(g)
        dev.receive(g)
        latest = max(latest, float(t_msg.max()))
        for _ in range(14):
            a, b = host.tick(latest), dev.tick(latest)
            assert a == b and host.t2 == dev.t2, (i, a, b)
            if a == "fov":
                break
            seen["ticks"] += 1
            seen["gated"] += a == "gated"
            rh, rd = host.result(), dev.result()
            seen["updates"] += a == "tick" and rh[0] == lv.OK
            assert (a == "gated" or rh[0] == rd[0]) and rh[4] == rd[4], (i, host.t2, rh[0], rd[0], rh[4], rd[4])
            assert bits(rh[2]) == bits(rd[2]) and bits(rh[3]) == bits(rd[3]), (i, host.t2)
            if a != "gated":                                          # a gated async update leaves an empty log
                assert len(rh[1]) == len(rd[1]) and all(
                    all(np.array_equal(p[k], q[k], equal_nan=True) for k in p) for p, q in zip(rh[1], rd[1])), (i, host.t2)
            assert bits(host.loc.map_points()) == bits(dev.loc.map_points()), (i, host.t2)
            assert host.mapper.last_map_time == dev.mapper.last_map_time
    assert dev.loc.async_status() == (lv.OK, "")
    assert seen["ticks"] >= 20 and seen["gated"] >= 1 and seen["updates"] >= 8, seen
    assert dev.maps == host.maps >= 3, (dev.maps, host.maps)
    assert len(dev.loc.map_points()) > 1000
    host.close()
    dev.close()
