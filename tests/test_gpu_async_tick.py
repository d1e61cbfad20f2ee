"""The stream-ordered tick (lv_*_async): every stage equals its synchronous form bit for bit, a sequence of ticks from an empty
map with windows below MAX_POINTS2MATCH equals the synchronous chain in which the host applies main.cpp:81, enqueuing a whole
tick never waits for the GPU, deferred errors are reported by lv_async_status and leave the handle usable, and map growth gives
the same results."""
import ctypes as C
import time

import numpy as np
import pytest

import bagwriter as W
from test_bag_reader import BagMessage, PC2View, VELO as BAG_VELO
from test_gpu_cloud_frontend import FRT, LIDARS, STAMP_US, assert_same, edge_clouds, u32
from test_wire_format import make_cloud

pytestmark = pytest.mark.gpu


def put_count(loc, d, v):
    a = np.array([v], np.int64)
    assert loc.L.lv_memcpy_h2d(loc.h, C.c_void_p(d), a.ctypes.data_as(C.c_void_p), 8) == 0


def get_count(loc, d):
    return int(loc.download(d, np.zeros(1, np.int64))[0])


class Bufs:
    """device buffers of one handle, freed together"""

    def __init__(self, loc):
        self.loc, self.ptrs = loc, []

    def __call__(self, nbytes):
        p = self.loc.device_alloc(max(int(nbytes), 8))
        self.ptrs.append(p)
        return p

    def upload(self, arr):
        arr = np.ascontiguousarray(arr)
        p = self(arr.nbytes)
        if arr.nbytes:
            assert self.loc.L.lv_memcpy_h2d(self.loc.h, C.c_void_p(p), arr.ctypes.data_as(C.c_void_p), arr.nbytes) == 0
        return p

    def free(self):
        for p in self.ptrs:
            self.loc.device_free(p)
        self.ptrs = []


@pytest.fixture(scope="module")
def loc(lv):
    h = lv.Localizer(lv.default_params(max_points=1 << 16, max_map_points=1 << 16))
    yield h
    h.close()


# ---- each stage against its synchronous form ---------------------------------------------------------------------------------
@pytest.mark.parametrize("lidar", LIDARS)
@pytest.mark.parametrize("rate,md", [(1, 0.0), (4, 3.0)])
def test_process_cloud_async_equals_sync(lv, loc, lidar, rate, md):
    clouds = dict(edge_clouds(lidar, rate))
    clouds["random"] = make_cloud(lidar, 3001, np.random.default_rng(5))
    for name, pts in clouds.items():
        b = Bufs(loc)
        n, nb = len(pts), pts.nbytes
        d_msg = b.upload(pts) if nb else b(8)
        lay = lv.cloud_layout(lidar, pts.dtype)
        sync = [b(k * n) for k in (12, 8, 4, 4, 4)]
        asyn = [b(k * n) for k in (12, 8, 4, 4, 4)]
        d_m = b(8)
        put_count(loc, d_m, -7)
        m = loc.process_cloud_device(lidar, lay, d_msg, nb, n, STAMP_US, True, True, FRT, rate, md, *sync)
        loc.process_cloud_device_async(lidar, lay, d_msg, nb, n, STAMP_US, True, True, FRT, rate, md, asyn[0], asyn[1], d_m, *asyn[2:])
        assert get_count(loc, d_m) == m, (lidar, name)
        host = lambda: (np.empty((m, 3), np.float32), np.empty(m), np.empty(m, np.float32), np.empty(m, np.float32),
                        np.empty(m, np.int32))
        got = tuple(loc.download(d, a) for d, a in zip(asyn, host()))
        ref = tuple(loc.download(d, a) for d, a in zip(sync, host()))
        assert_same(got, ref, (lidar, name))
        assert loc.async_status() == (lv.OK, "")
        b.free()


def voxel_cases():
    rng = np.random.default_rng(11)
    pts = (rng.normal(0, 15, (5000, 3))).astype(np.float32)
    wide = (rng.uniform(-1000, 1000, (3000, 3))).astype(np.float32)
    return [("n0", pts, 0, 0.5), ("n1", pts, 1, 0.5), ("n17", pts, 17, 0.5), ("n<n_max", pts, 3210, 0.5),
            ("n=n_max", pts, 5000, 0.5), ("fine", pts, 5000, 0.05), ("2^31 cells: pass-through", wide, 3000, 0.01),
            ("2^31 cells, n<n_max", wide, 2000, 0.01)]


def test_voxelgrid_async_equals_sync(lv, loc):
    for name, pts, k, leaf in voxel_cases():
        b = Bufs(loc)
        n_max = len(pts)
        d_in = b.upload(pts)
        d_sync, d_async, d_n, d_m = b(12 * n_max), b(12 * n_max), b(8), b(8)
        put_count(loc, d_n, k)
        put_count(loc, d_m, -3)
        m = loc.voxelgrid_downsample_device(d_in, k, leaf, d_sync) if k else 0
        loc.voxelgrid_downsample_device_async(d_in, d_n, n_max, leaf, d_async, d_m)
        assert get_count(loc, d_m) == m, name
        if "pass-through" in name or "2^31" in name:
            assert m == k and k > 0, name
        a = loc.download(d_async, np.empty((m, 3), np.float32))
        r = loc.download(d_sync, np.empty((m, 3), np.float32))
        assert (u32(a) == u32(r)).all(), name
        assert loc.async_status() == (lv.OK, "")
        b.free()


def make_path(lv, sc, t1=10.0, t2=10.1, seed=9):
    """the deskew path and Xt2 of a sweep between t1 and t2 (Compensator::upsample / get_t2 on the host)"""
    rng = np.random.default_rng(seed)
    st_t = np.linspace(t1 - 0.012, t2 - 0.004, 4)
    imu_t = np.arange(st_t[0] + 0.5e-3, t2 + 4e-3, 2.5e-3)
    imu_a = (np.array([0.3, -0.2, 9.8]) + rng.normal(0, 0.05, (len(imu_t), 3))).astype(np.float32)
    imu_w = (np.array([0.0, 0.0, 0.5]) + rng.normal(0, 0.01, (len(imu_t), 3))).astype(np.float32)
    states = []
    for ts in st_t:
        x = sc.world.pose(8.0 + 15.0 * (ts - t1), sc.prm).copy()
        x[14:17] = [15.0, 0.0, 0.0]
        j = int(np.searchsorted(imu_t, ts))
        states.append(lv.state_from_ikfom(sc.prm, x, ts, imu_a[j], imu_w[j]))
    path = lv.compensator_upsample(states, imu_a, imu_w, imu_t)
    return path, lv.compensator_get_t2(path, t2)


def test_compensate_async_equals_sync(lv, loc, scene_xaloc):
    path, x2 = make_path(lv, scene_xaloc)
    rng = np.random.default_rng(3)
    n_max = 4000
    xyz = rng.normal(0, 20, (n_max, 3)).astype(np.float32)
    t = np.sort(rng.uniform(10.0, 10.099, n_max))
    for k in (1, 2500, n_max):
        b = Bufs(loc)
        d_xyz, d_t, d_n = b.upload(xyz), b.upload(t), b(8)
        d_sync, d_async = b(12 * n_max), b(12 * n_max)
        put_count(loc, d_n, k)
        loc.compensate_device(path, x2, d_xyz, d_t, k, d_sync)
        loc.compensate_device_async(path, x2, d_xyz, d_t, d_n, n_max, d_async)
        loc.compensate_device_async(path, x2, d_xyz, d_t, d_n, n_max, d_xyz)     # in place
        r = loc.download(d_sync, np.empty((k, 3), np.float32))
        assert (u32(loc.download(d_async, np.empty((k, 3), np.float32))) == u32(r)).all(), k
        assert (u32(loc.download(d_xyz, np.empty((k, 3), np.float32))) == u32(r)).all(), k
        assert loc.async_status() == (lv.OK, "")
        b.free()


def test_max_points_bound(lv, loc):
    b = Bufs(loc)
    d, d_n = b(12 * 70000), b(8)
    L = lv.lib()
    assert L.lv_voxelgrid_downsample_device_async(loc.h, d, d_n, (1 << 16) + 1, C.c_float(0.5), d + 12 * 65537, d_n) == lv.ERR_ARG
    assert b"max_points" in L.lv_last_error()
    assert L.lv_correct_device_async(loc.h, d, d_n, (1 << 16) + 1, 10, 1.0) == lv.ERR_ARG
    assert b"max_points" in L.lv_last_error()
    b.free()


# ---- ticks from an empty map -------------------------------------------------------------------------------------------------
def tick_messages(lv, sc, tmp_path, n_ticks=18):
    """ring-major Velodyne messages of the synthetic scene in a bag, parsed back; every 4th one (the first included) cut to 300
    points, so its downsampled window falls below MIN_POINTS"""
    rings, cols = 32, 256
    W_msgs = []
    for i in range(n_ticks):
        x = sc.world.pose(8.0 + 0.02 * i, sc.prm)
        sw = sc.world.sweep(x, rings=rings, azimuths=cols, seed=100 + i)
        xyz = sw.reshape(cols, rings, 3).transpose(1, 0, 2).reshape(-1, 3)
        col = np.tile(np.arange(cols), rings)
        velo = np.zeros(len(xyz), BAG_VELO)
        velo["x"], velo["y"], velo["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
        velo["time"] = (col * (0.099 / (cols - 1))).astype(np.float32)
        if i % 4 == 0:
            velo = velo[:300]
        W_msgs.append((1, 10, 0, W.pointcloud2(velo, 10, 0)))
    bag = str(tmp_path / "ticks.bag")
    W.write_bag(bag, {1: ("/velodyne_points", "sensor_msgs/PointCloud2")}, W_msgs)
    L = lv.lib()
    L.lv_bag_next.argtypes = [C.c_void_p, C.POINTER(BagMessage)]
    L.lv_bag_parse_pointcloud2.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.POINTER(PC2View)]
    L.lv_bag_close.argtypes = [C.c_void_p]
    handle = C.c_void_p()
    assert L.lv_bag_open(bag.encode(), C.byref(handle)) == lv.OK
    msgs, m = [], BagMessage()
    while L.lv_bag_next(handle, C.byref(m)) == 1:
        v = PC2View()
        assert L.lv_bag_parse_pointcloud2(C.cast(m.data, C.c_void_p), m.size, 0, C.byref(v)) == lv.OK
        msgs.append(dict(n=v.n_points, stamp=v.stamp_sec * 1_000_000 + v.stamp_nsec // 1000, layout=lv.CloudLayout.from_buffer_copy(v.layout),
                         raw=np.ctypeslib.as_array(v.data, shape=(v.data_bytes,)).copy()))
    L.lv_bag_close(handle)
    assert len(msgs) == n_ticks
    return msgs


RATE, MD, LEAF, MIN_POINTS = 2, 3.0, 0.5, 200
IMU_ACC, IMU_GYRO = np.array([[0.05, 0.0, 9.81]] * 4), np.array([[0.0, 0.0, 0.01]] * 4)


class Chain:
    """one handle running the tick: sync (the host reads every count and applies main.cpp:81) or async (counts on the device)"""

    def __init__(self, lv, sc, msgs, path, x2, growth=0, max_map_points=1 << 19, stream=None):
        prm = lv.params_from_yaml(lv.CONFIG_DIR + "/xaloc.yaml", max_map_points=max_map_points, max_points=1 << 16)
        if stream is not None:
            prm.stream = stream
        self.lv, self.msgs, self.path, self.x2 = lv, msgs, path, x2
        self.loc = lv.Localizer(prm)
        if growth:
            self.loc.map_set_growth(growth)
        self.loc.set_state(sc.x_prop, sc.P0)
        self.b = Bufs(self.loc)
        nm = max(g["n"] for g in msgs)
        self.d_msg = self.b(max(len(g["raw"]) for g in msgs))
        self.d_xyz, self.d_t, self.d_ds = self.b(12 * nm), self.b(8 * nm), self.b(12 * nm)
        self.d_k, self.d_m = self.b(8), self.b(8)
        self.statuses = []

    def upload(self, g):
        raw = g["raw"]
        assert self.loc.L.lv_memcpy_h2d(self.loc.h, C.c_void_p(self.d_msg), raw.ctypes.data_as(C.c_void_p), len(raw)) == 0

    def tick_sync(self, i, t):
        g, loc = self.msgs[i], self.loc
        self.upload(g)
        loc.propagate_device(IMU_ACC, IMU_GYRO, np.full(4, 0.025))
        k = loc.process_cloud_device("velodyne", g["layout"], self.d_msg, len(g["raw"]), g["n"], g["stamp"], True, True, FRT, RATE, MD,
                                     self.d_xyz, self.d_t)
        loc.compensate_device(self.path, self.x2, self.d_xyz, self.d_t, k, self.d_xyz)
        m = loc.voxelgrid_downsample_device(self.d_xyz, k, LEAF, self.d_ds)
        if m < MIN_POINTS:                                        # main.cpp:81
            self.statuses.append(self.lv.TOO_FEW_POINTS)
            return
        st = loc.correct_device(self.d_ds, m, t)
        loc.map_add_last_sweep(True)
        self.statuses.append(st)

    def tick_async(self, i, t):
        g, loc = self.msgs[i], self.loc
        self.upload(g)
        self.enqueue(g, t)

    def enqueue(self, g, t):
        loc, nm = self.loc, g["n"]
        loc.propagate_device(IMU_ACC, IMU_GYRO, np.full(4, 0.025))
        loc.process_cloud_device_async("velodyne", g["layout"], self.d_msg, len(g["raw"]), nm, g["stamp"], True, True, FRT, RATE, MD,
                                       self.d_xyz, self.d_t, self.d_k)
        loc.compensate_device_async(self.path, self.x2, self.d_xyz, self.d_t, self.d_k, nm, self.d_xyz)
        loc.voxelgrid_downsample_device_async(self.d_xyz, self.d_k, nm, LEAF, self.d_ds, self.d_m)
        st = loc.correct_device_async(self.d_ds, self.d_m, nm, MIN_POINTS, t)
        loc.map_add_last_sweep(True)
        self.statuses.append(st)

    def result(self):
        st, logs = self.loc.last_logs()
        x, P = self.loc.get_state()
        return st, logs, x, P, self.loc.last_time_updated()

    def close(self):
        self.b.free()
        self.loc.close()


def same_result(a, b, what):
    (sa, la, xa, Pa, ta), (sb, lb, xb, Pb, tb) = a, b
    assert sa == sb and ta == tb, (what, sa, sb, ta, tb)
    assert (xa == xb).all() and (Pa == Pb).all(), what
    assert len(la) == len(lb), what
    for p, q in zip(la, lb):
        assert all(np.array_equal(p[key], q[key]) for key in p), what


def run_chains(lv, sc, msgs, path, x2, **kw):
    sync, per_tick, at_end = Chain(lv, sc, msgs, path, x2, **kw), Chain(lv, sc, msgs, path, x2, **kw), Chain(lv, sc, msgs, path, x2, **kw)
    gated = 0
    for i in range(len(msgs)):
        t = 10.1 + 0.1 * i
        sync.tick_sync(i, t)
        per_tick.tick_async(i, t)
        at_end.tick_async(i, t)
        rs = sync.result()
        ra = per_tick.result()
        if sync.statuses[-1] == lv.TOO_FEW_POINTS:
            gated += 1
            if i > 0:                                             # the update did not run: the fetched status says so
                assert ra[0] == lv.TOO_FEW_POINTS, i
            assert (rs[2] == ra[2]).all() and (rs[3] == ra[3]).all() and rs[4] == ra[4], i
        else:
            same_result(rs, ra, i)
        assert (sync.loc.map_points() == per_tick.loc.map_points()).all(), i
    assert gated >= 4 and sync.statuses[0] == lv.TOO_FEW_POINTS and sync.statuses[1] == lv.EMPTY_MAP
    same_result(sync.result(), at_end.result(), "end")
    ms = sync.loc.map_points()
    assert len(ms) > 1000 and (ms == at_end.loc.map_points()).all()
    assert per_tick.loc.async_status() == (lv.OK, "") and at_end.loc.async_status() == (lv.OK, "")
    info = [c.loc.map_info() for c in (sync, per_tick, at_end)]
    for c in (sync, per_tick, at_end):
        c.close()
    return info


def test_ticks_from_an_empty_map_equal_the_sync_chain(lv, scene_xaloc, tmp_path):
    sc = scene_xaloc
    msgs = tick_messages(lv, sc, tmp_path)
    path, x2 = make_path(lv, sc)
    run_chains(lv, sc, msgs, path, x2)


def test_ticks_with_map_growth_equal_the_sync_chain(lv, scene_xaloc, tmp_path):
    sc = scene_xaloc
    msgs = tick_messages(lv, sc, tmp_path, n_ticks=16)
    path, x2 = make_path(lv, sc)
    info = run_chains(lv, sc, msgs, path, x2, growth=1 << 20, max_map_points=4096)
    assert all(i["growths"] > 0 for i in info), info
    assert info[0]["points"] == info[1]["points"] == info[2]["points"]


# ---- no host wait ------------------------------------------------------------------------------------------------------------
def test_enqueuing_a_tick_does_not_wait_for_the_gpu(lv, scene_xaloc, tmp_path):
    import torch
    sc = scene_xaloc
    msgs = tick_messages(lv, sc, tmp_path, n_ticks=8)
    path, x2 = make_path(lv, sc)
    stream = torch.cuda.Stream()
    busy = Chain(lv, sc, msgs, path, x2, stream=stream.cuda_stream)
    eager = Chain(lv, sc, msgs, path, x2)
    for c in (busy, eager):                                       # warm-up: graphs, scratch, the map
        for i in range(3):
            c.tick_async(i, 10.1 + 0.1 * i)
        c.result()
    enqueue_ms = []
    for i in (5, 6):                                              # full-size windows: their update graph exists
        g = msgs[i]
        busy.upload(g)                                            # synchronous copy: before the GPU is busy
        with torch.cuda.stream(stream):
            torch.cuda._sleep(100_000_000)                        # ~50 ms at the H100's clock: the stream is busy
        t0 = time.perf_counter()
        busy.enqueue(g, 10.1 + 0.1 * i)
        enqueue_ms.append(1e3 * (time.perf_counter() - t0))
        stream.synchronize()
        eager.tick_async(i, 10.1 + 0.1 * i)
        same_result(busy.result(), eager.result(), i)
    assert max(enqueue_ms) < 10.0, enqueue_ms
    assert (busy.loc.map_points() == eager.loc.map_points()).all()
    busy.close()
    eager.close()


# ---- deferred errors ---------------------------------------------------------------------------------------------------------
def test_deferred_errors_name_the_stage_and_leave_the_handle_usable(lv, loc, scene_xaloc):
    path, x2 = make_path(lv, scene_xaloc)
    rng = np.random.default_rng(31)
    pts = make_cloud("velodyne", 2000, rng)
    pts["time"] = np.linspace(0.0, 0.09, 2000, dtype=np.float32)
    bad = pts.copy()
    bad["time"][999] = np.nan                                     # a kept point (rate 1)
    b = Bufs(loc)
    n = len(pts)
    lay = lv.cloud_layout("velodyne", pts.dtype)
    d_good, d_bad = b.upload(pts), b.upload(bad)
    d_xyz, d_t, d_k, d_ref = b(12 * n), b(8 * n), b(8), b(12 * n)
    stamp = 10_000_000                                            # 10 s: inside the path
    loc.process_cloud_device_async("velodyne", lay, d_bad, pts.nbytes, n, stamp, True, True, FRT, 1, 0.0, d_xyz, d_t, d_k)
    st, msg = loc.async_status()
    assert st == lv.ERR_ARG and "process cloud" in msg and "NaN" in msg, msg
    assert loc.async_status() == (lv.OK, "")                      # reported once
    # a stamp outside the path: the message 1 s late
    loc.process_cloud_device_async("velodyne", lay, d_good, pts.nbytes, n, stamp + 1_000_000, True, True, FRT, 1, 0.0, d_xyz, d_t, d_k)
    loc.compensate_device_async(path, x2, d_xyz, d_t, d_k, n, d_xyz)
    st, msg = loc.async_status()
    assert st == lv.ERR_ARG and "compensate" in msg and "process cloud" not in msg, msg
    # the next tick on the same handle is right
    loc.process_cloud_device_async("velodyne", lay, d_good, pts.nbytes, n, stamp, True, True, FRT, 1, 0.0, d_xyz, d_t, d_k)
    loc.compensate_device_async(path, x2, d_xyz, d_t, d_k, n, d_xyz)
    assert loc.async_status() == (lv.OK, "")
    k = loc.process_cloud_device("velodyne", lay, d_good, pts.nbytes, n, stamp, True, True, FRT, 1, 0.0, d_ref, d_t)
    assert k == get_count(loc, d_k) == n
    loc.compensate_device(path, x2, d_ref, d_t, k, d_ref)
    assert (u32(loc.download(d_xyz, np.empty((k, 3), np.float32))) == u32(loc.download(d_ref, np.empty((k, 3), np.float32)))).all()
    # a device count outside [0, n_max] is clamped and flagged
    put_count(loc, d_k, n + 5)
    loc.voxelgrid_downsample_device_async(d_xyz, d_k, n, LEAF, d_ref, d_k)
    st, msg = loc.async_status()
    assert st == lv.ERR_ARG and "outside [0, n_max]" in msg, msg
    b.free()
