"""The LiDAR buffer in HBM (lv_lidar_*) against tests/lidar_buffer_ref.py, the literal restatement of Buffer / Accumulator::get,
bit for bit: every window's xyz, time and count through the synchronous and the stream-ordered get, on a ring of about three
messages that wraps several times, with 64-point ties at t2 and at t1, late and overlapping messages, empty windows, messages with
nothing kept and clears of everything; a push that does not fit and a window above n_max are deferred errors that leave the
buffer unchanged and the handle usable.  Then whole sequences of windowed ticks from an empty map (main.cpp:61-122, t1 / t2 / the
field-of-view check on the host) equal the chain that keeps the deque in the restatement and runs the synchronous device calls."""
import ctypes as C

import numpy as np
import pytest

import lidar_buffer_ref as R
from test_bag_reader import VELO
from test_gpu_async_tick import Bufs, get_count, put_count
from test_gpu_cloud_frontend import FRT

pytestmark = pytest.mark.gpu
RINGS = 64


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8).tobytes()


@pytest.fixture(scope="module")
def loc(lv):
    h = lv.Localizer(lv.default_params(max_points=1 << 16, max_map_points=1 << 16))
    yield h
    h.close()


class DeviceBuffer:
    """the handle's buffer with staging for messages and windows"""

    def __init__(self, loc, cap, n_max=1 << 14):
        self.loc, self.n_max = loc, n_max
        self.b = Bufs(loc)
        self.d_xyz, self.d_t, self.d_n = self.b(12 * n_max), self.b(8 * n_max), self.b(8)
        self.w_xyz, self.w_t, self.d_m = self.b(12 * n_max), self.b(8 * n_max), self.b(8)
        loc.lidar_reserve(cap)

    def push(self, xyz, t):
        n = len(t)
        if n:
            self.b.loc.L.lv_memcpy_h2d(self.loc.h, C.c_void_p(self.d_xyz), np.ascontiguousarray(xyz, np.float32).ctypes.data_as(C.c_void_p), 12 * n)
            self.b.loc.L.lv_memcpy_h2d(self.loc.h, C.c_void_p(self.d_t), np.ascontiguousarray(t, np.float64).ctypes.data_as(C.c_void_p), 8 * n)
        put_count(self.loc, self.d_n, n)
        self.loc.lidar_push_async(self.d_xyz, self.d_t, self.d_n, max(n, 1))

    def get(self, t1, t2, sync, n_max=None):
        n_max = n_max or self.n_max
        if sync:
            m = self.loc.lidar_get_points(t1, t2, self.w_xyz, self.w_t, n_max)
        else:
            put_count(self.loc, self.d_m, -9)
            self.loc.lidar_get_points_async(t1, t2, self.w_xyz, self.w_t, n_max, self.d_m)
            m = get_count(self.loc, self.d_m)
        return self.loc.download(self.w_xyz, np.empty((m, 3), np.float32)), self.loc.download(self.w_t, np.empty(m))

    def close(self):
        self.b.free()


def velodyne_message(rng, start, cols, dt=1e-3):
    """RINGS points per firing column, the column's points sharing one time (ring-major within a column)"""
    t = np.repeat(start + dt * np.arange(cols), RINGS)
    return rng.normal(0, 20, (len(t), 3)).astype(np.float32), t


def same_window(lv, dev, ref, t1, t2, what):
    rx, rt = ref.get(t1, t2)
    for sync in (True, False):
        gx, gt = dev.get(t1, t2, sync)
        assert len(gt) == len(rt), (what, sync, t1, t2, len(gt), len(rt))
        assert bits(gx) == bits(rx) and bits(gt) == bits(rt), (what, sync, t1, t2)
    return len(rt)


def same_content(lv, dev, ref, what):
    info = dev.loc.lidar_info()
    assert info["points"] == ref.size(), (what, info, ref.size())
    if ref.size():
        assert bits(np.float64(info["newest_time"])) == bits(np.float64(ref.content[0][0])), what
        assert bits(np.float64(info["oldest_time"])) == bits(np.float64(ref.content[-1][0])), what
    assert dev.loc.async_status() == (lv.OK, "")


def test_windows_on_a_wrapping_ring_equal_the_restatement(lv, loc):
    rng = np.random.default_rng(7)
    cap = 3 * 24 * RINGS + 100                                    # about three messages
    dev, ref = DeviceBuffer(loc, cap), R.LidarBuffer()
    clock, pushed, seen = 0.0, 0, dict(tie_t2=0, tie_t1=0, empty=0, late=0, overlap=0, cleared_all=0, nothing_kept=0, nonempty=0)
    for i in range(60):
        kind = rng.random()
        cols = int(rng.integers(8, 25))
        if kind < 0.1:
            start = clock - 0.05                                   # late: older than what the buffer holds
            seen["late"] += 1
        elif kind < 0.2:
            start = clock - 0.008                                 # overlaps the previous message
            seen["overlap"] += 1
        else:
            start = clock
        if rng.random() < 0.08:
            cols = 0
            seen["nothing_kept"] += 1
        xyz, t = velodyne_message(rng, start, cols)
        if ref.size() + len(t) > cap:
            ref.clear(np.inf)
            loc.lidar_clear_async(np.inf)
            seen["cleared_all"] += 1
        dev.push(xyz, t)
        ref.push_message(xyz, t)
        pushed += len(t)
        clock = max(clock, start + cols * 1e-3 + 2e-3)
        same_content(lv, dev, ref, i)
        col_times = np.unique(ref.times())
        for _ in range(4):
            if len(col_times) and rng.random() < 0.8:
                t2 = float(rng.choice(col_times))
                t1 = t2 - 1e-3 * int(rng.integers(0, 12))          # on a column time too, when there is one
                seen["tie_t2"] += 1
                seen["tie_t1"] += t1 in col_times
            else:
                t1, t2 = sorted(rng.uniform(clock - 0.1, clock + 0.01, 2))
            m = same_window(lv, dev, ref, t1, t2, i)
            seen["empty"] += m == 0
            seen["nonempty"] += m > 0
        if rng.random() < 0.3:
            tc = float(rng.choice(col_times)) if len(col_times) else clock
            ref.clear(tc)
            loc.lidar_clear_async(tc)
            same_content(lv, dev, ref, ("clear", i))
    assert pushed > 3 * cap, pushed                                # wrapped several times
    assert all(v > 0 for v in seen.values()), seen
    ref.clear(np.inf)
    loc.lidar_clear_async(np.inf)
    same_content(lv, dev, ref, "end")
    assert same_window(lv, dev, ref, -np.inf, np.inf, "empty") == 0
    dev.close()


def test_ties_at_t2_return_two_and_the_next_window_the_rest(lv, loc):
    rng = np.random.default_rng(3)
    dev, ref = DeviceBuffer(loc, 4096), R.LidarBuffer()
    xyz, t = velodyne_message(rng, 5.0, 10)
    dev.push(xyz, t)
    ref.push_message(xyz, t)
    t2 = 5.0 + 1e-3 * 6
    assert same_window(lv, dev, ref, 5.0 + 1e-3 * 3, t2, "ties") == 3 * RINGS + 2
    assert same_window(lv, dev, ref, t2, 5.0 + 1e-3 * 9, "next") == 3 * RINGS + 2
    loc.lidar_clear_async(np.inf)
    assert loc.lidar_info()["points"] == 0
    dev.close()


def test_a_push_that_does_not_fit_is_a_deferred_error_and_changes_nothing(lv, loc):
    rng = np.random.default_rng(4)
    dev, ref = DeviceBuffer(loc, 1000), R.LidarBuffer()
    for k in range(3):
        xyz, t = velodyne_message(rng, 1.0 + 0.01 * k, 5)          # 320 points each
        dev.push(xyz, t)
        ref.push_message(xyz, t)
    xyz, t = velodyne_message(rng, 1.05, 2)                       # 960 + 128 > 1000
    dev.push(xyz, t)
    st, msg = loc.async_status()
    assert st == lv.ERR_ARG and "lidar push" in msg, msg
    same_content(lv, dev, ref, "full")
    same_window(lv, dev, ref, 0.0, 2.0, "full")
    ref.clear(1.015)
    loc.lidar_clear_async(1.015)
    dev.push(xyz, t)                                              # fits now
    ref.push_message(xyz, t)
    same_content(lv, dev, ref, "after")
    same_window(lv, dev, ref, 1.0, 1.06, "after")
    loc.lidar_clear_async(np.inf)
    dev.close()


def test_a_window_above_n_max_is_count_zero_and_a_deferred_error(lv, loc):
    rng = np.random.default_rng(5)
    dev, ref = DeviceBuffer(loc, 4096), R.LidarBuffer()
    xyz, t = velodyne_message(rng, 2.0, 20)
    dev.push(xyz, t)
    ref.push_message(xyz, t)
    t2 = float(t[-1])
    rx, rt = ref.get(2.0, t2)
    assert len(rt) == 19 * RINGS + 2                              # two of the last column's 64
    gx, gt = dev.get(2.0, t2, sync=False, n_max=len(rt) - 1)
    assert len(gt) == 0
    st, msg = loc.async_status()
    assert st == lv.ERR_ARG and "lidar get points" in msg and "n_max" in msg, msg
    with pytest.raises(RuntimeError, match="holds %d points" % len(rt)):
        dev.get(2.0, t2, sync=True, n_max=len(rt) - 1)
    assert loc.async_status() == (lv.OK, "")                      # the synchronous form reports it itself
    gx, gt = dev.get(2.0, t2, sync=False, n_max=len(rt))       # exactly n_max: fits
    assert bits(gx) == bits(rx) and bits(gt) == bits(rt)
    same_window(lv, dev, ref, 2.005, 2.010, "usable")
    loc.lidar_clear_async(np.inf)
    dev.close()


def test_reserve_keeps_the_live_points_in_order(lv, loc):
    rng = np.random.default_rng(6)
    dev, ref = DeviceBuffer(loc, 700), R.LidarBuffer()
    for k in range(5):                                            # wraps the 700-slot ring
        xyz, t = velodyne_message(rng, 3.0 + 0.004 * k, 4)
        if ref.size() + len(t) > 700:
            ref.clear(3.0 + 0.004 * k - 0.006)
            loc.lidar_clear_async(3.0 + 0.004 * k - 0.006)
        dev.push(xyz, t)
        ref.push_message(xyz, t)
    for cap in (5000, ref.size(), 3000):
        loc.lidar_reserve(cap)
        assert loc.lidar_info()["capacity"] == cap
        same_content(lv, dev, ref, cap)
        same_window(lv, dev, ref, 3.0, 4.0, cap)
        same_window(lv, dev, ref, 3.009, 3.013, cap)
    L = lv.lib()
    assert L.lv_lidar_reserve(loc.h, ref.size() - 1) == lv.ERR_CAPACITY and b"live" in L.lv_last_error()
    same_content(lv, dev, ref, "refused")
    loc.lidar_clear_async(np.inf)
    dev.close()


def test_argument_refusals_that_need_a_handle(lv):
    L = lv.lib()
    loc = lv.Localizer(lv.default_params(max_points=1 << 12, max_map_points=1 << 12))
    b = Bufs(loc)
    d, d_n = b(12 * 100), b(8)
    for call in (lambda: L.lv_lidar_push_device_async(loc.h, d, d + 1200, d_n, 1),
                 lambda: L.lv_lidar_get_points_device_async(loc.h, 0.0, 1.0, d, d + 1200, 1, d_n),
                 lambda: L.lv_lidar_get_points_device(loc.h, 0.0, 1.0, d, d + 1200, 1, C.byref(C.c_int64())),
                 lambda: L.lv_lidar_clear_async(loc.h, 1.0)):
        assert call() == lv.ERR_ARG and b"lv_lidar_reserve first" in L.lv_last_error()
    info = loc.lidar_info()
    assert info["points"] == 0 and info["capacity"] == 0 and np.isnan(info["oldest_time"])
    loc.lidar_reserve(1)
    info = loc.lidar_info()
    assert info["points"] == 0 and info["capacity"] == 1 and np.isnan(info["newest_time"])
    assert loc.async_status() == (lv.OK, "")
    b.free()
    loc.close()


# ---- windowed ticks from an empty map ----------------------------------------------------------------------------------------------
COLS, RATE, MD, LEAF, MIN_POINTS = 256, 2, 3.0, 0.5, 100
EMPTY_LIDAR_TIME = 0.15                                          # main.cpp:122's empty_lidar_time, short so that clears bite
IMU_ACC, IMU_GYRO = np.array([[0.05, 0.0, 9.81]] * 4), np.array([[0.0, 0.0, 0.01]] * 4)


def sequence_messages(lv, sc, n_msgs=7, cut=3):
    """Velodyne messages at 10 Hz, 64 rings x COLS columns (the rings of a column share its time), ring-major; message `cut` keeps
    only 300 points, so its windows fall below MIN_POINTS"""
    msgs = []
    for i in range(n_msgs):
        x = sc.world.pose(8.0 + 0.1 * i, sc.prm)
        sw = sc.world.sweep(x, rings=RINGS, azimuths=COLS, seed=200 + i)
        xyz = sw.reshape(COLS, RINGS, 3).transpose(1, 0, 2).reshape(-1, 3)
        velo = np.zeros(len(xyz), VELO)
        velo["x"], velo["y"], velo["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
        velo["time"] = (np.tile(np.arange(COLS), RINGS) * (0.099 / (COLS - 1))).astype(np.float32)
        if i == cut:
            velo = velo[:300]
        msgs.append(dict(raw=np.frombuffer(velo.tobytes(), np.uint8).copy(), n=len(velo), stamp=10_000_000 + 100_000 * i,
                         layout=lv.cloud_layout("velodyne", VELO)))
    return msgs


def window_path(lv, sc, t1, t2):
    """Compensator::path(t1, t2) stand-in (upsample of host states and IMUs around the window) and Compensator::get_t2"""
    rng = np.random.default_rng(int(t2 * 1e4))
    st_t = np.linspace(t1 - 0.012, t2 + 0.004, 4)
    imu_t = np.arange(st_t[0] + 0.5e-3, t2 + 8e-3, 2.5e-3)
    imu_a = (np.array([0.3, -0.2, 9.8]) + rng.normal(0, 0.05, (len(imu_t), 3))).astype(np.float32)
    imu_w = (np.array([0.0, 0.0, 0.5]) + rng.normal(0, 0.01, (len(imu_t), 3))).astype(np.float32)
    states = []
    for ts in st_t:
        x = sc.world.pose(8.0 + (ts - 10.0), sc.prm).copy()
        x[14:17] = [1.0, 0.0, 0.0]
        j = int(np.searchsorted(imu_t, ts))
        states.append(lv.state_from_ikfom(sc.prm, x, ts, imu_a[j], imu_w[j]))
    path = lv.compensator_upsample(states, imu_a, imu_w, imu_t)
    assert path[0].time <= t1 and path[-1].time >= t2
    return path, lv.compensator_get_t2(path, t2)


class WindowChain:
    """one handle running main.cpp:61-122 over the messages: `device` keeps the buffer in HBM and enqueues the tick; otherwise the
    deque lives in the restatement and every window is uploaded to the synchronous calls"""

    def __init__(self, lv, sc, msgs, delta, device):
        prm = lv.params_from_yaml(lv.CONFIG_DIR + "/xaloc.yaml", max_map_points=1 << 19, max_points=1 << 16)
        self.lv, self.sc, self.msgs, self.delta, self.device = lv, sc, msgs, delta, device
        self.loc = lv.Localizer(prm)
        self.loc.set_state(sc.x_prop, sc.P0)
        self.b = Bufs(self.loc)
        self.nm = max(g["n"] for g in msgs)
        self.n_max = 1 << 16
        self.d_msg = self.b(max(len(g["raw"]) for g in msgs))
        self.d_pxyz, self.d_pt, self.d_k = self.b(12 * self.nm), self.b(8 * self.nm), self.b(8)
        self.d_wxyz, self.d_wt, self.d_w = self.b(12 * self.n_max), self.b(8 * self.n_max), self.b(8)
        self.d_ds, self.d_m = self.b(12 * self.n_max), self.b(8)
        if device:
            self.loc.lidar_reserve(3 * self.nm // RATE)           # about three messages: wraps
        self.ref = R.LidarBuffer()
        self.t2 = np.finfo(np.float64).max
        self.ltu = -1.0
        self.window = None

    def receive(self, g):
        """Accumulator::receive_lidar: returns the processed message's times (the host chain reads them)"""
        loc = self.loc
        assert loc.L.lv_memcpy_h2d(loc.h, C.c_void_p(self.d_msg), g["raw"].ctypes.data_as(C.c_void_p), len(g["raw"])) == 0
        args = ("velodyne", g["layout"], self.d_msg, len(g["raw"]), g["n"], g["stamp"], True, True, FRT, RATE, MD, self.d_pxyz, self.d_pt)
        if self.device:
            loc.process_cloud_device_async(*args, self.d_k)
            loc.lidar_push_async(self.d_pxyz, self.d_pt, self.d_k, g["n"])
            return None
        k = loc.process_cloud_device(*args)
        xyz, t = loc.download(self.d_pxyz, np.empty((k, 3), np.float32)), loc.download(self.d_pt, np.empty(k))
        self.ref.push_message(xyz, t)
        return t

    def tick(self, latest):
        """main.cpp:61-122; returns 'fov', 'gated' (the host chain only: the device chain cannot tell) or the update status"""
        loc, delta = self.loc, self.delta
        self.t2 = min(self.t2 + delta, latest)                    # not real_time: t2 advances by delta, no further than latest
        t2 = self.t2
        t1 = max(t2 - delta, self.ltu)
        if t2 - t1 < delta - 1e-6:
            return "fov", t1, t2
        loc.propagate_device(IMU_ACC, IMU_GYRO, np.full(4, delta / 4))
        path, x2 = window_path(self.lv, self.sc, t1, t2)
        if self.device:
            loc.lidar_get_points_async(t1, t2, self.d_wxyz, self.d_wt, self.n_max, self.d_w)
            k = get_count(loc, self.d_w)                          # the test reads the window; the tick itself does not
            self.window = (loc.download(self.d_wxyz, np.empty((k, 3), np.float32)), loc.download(self.d_wt, np.empty(k)))
            loc.compensate_device_async(path, x2, self.d_wxyz, self.d_wt, self.d_w, self.n_max, self.d_wxyz)
            loc.voxelgrid_downsample_device_async(self.d_wxyz, self.d_w, self.n_max, LEAF, self.d_ds, self.d_m)
            st = loc.correct_device_async(self.d_ds, self.d_m, self.n_max, MIN_POINTS, t2)
            loc.map_add_last_sweep(True)
            loc.lidar_clear_async(t2 - EMPTY_LIDAR_TIME)
            loc.get_state()                                       # publish: resolves last_time_updated
        else:
            xyz, t = self.window = self.ref.get(t1, t2)
            m = 0
            if len(t):
                assert loc.L.lv_memcpy_h2d(loc.h, C.c_void_p(self.d_wxyz), xyz.ctypes.data_as(C.c_void_p), xyz.nbytes) == 0
                assert loc.L.lv_memcpy_h2d(loc.h, C.c_void_p(self.d_wt), t.ctypes.data_as(C.c_void_p), t.nbytes) == 0
                loc.compensate_device(path, x2, self.d_wxyz, self.d_wt, len(t), self.d_wxyz)
                m = loc.voxelgrid_downsample_device(self.d_wxyz, len(t), LEAF, self.d_ds)
            if m < MIN_POINTS:                                    # main.cpp:81
                return "gated", t1, t2
            st = loc.correct_device(self.d_ds, m, t2)
            loc.map_add_last_sweep(True)
            self.ref.clear(t2 - EMPTY_LIDAR_TIME)                 # main.cpp:122
        self.ltu = loc.last_time_updated()
        return st, t1, t2

    def result(self):
        st, logs = self.loc.last_logs()
        x, P = self.loc.get_state()
        return st, logs, x, P, self.loc.last_time_updated()

    def close(self):
        self.b.free()
        self.loc.close()


@pytest.mark.parametrize("delta", [0.01, 0.02])
def test_windowed_ticks_equal_the_restatement_chain(lv, scene_xaloc, delta):
    sc = scene_xaloc
    msgs = sequence_messages(lv, sc)
    host, dev = WindowChain(lv, sc, msgs, delta, False), WindowChain(lv, sc, msgs, delta, True)
    seen = dict(ticks=0, fov=0, gated=0, updates=0, two_messages=0, t2_on_column=0)
    latest, spans = -np.inf, []
    for i, g in enumerate(msgs):
        t_msg = host.receive(g)
        dev.receive(g)
        latest = max(latest, float(t_msg.max()))                  # Accumulator::latest_time: the newest point received
        spans.append((float(t_msg.min()), float(t_msg.max())))
        for _ in range(14):                                       # the driver loop spins until the field of view runs out
            a, t1, t2 = host.tick(latest)
            b, t1b, t2b = dev.tick(latest)
            assert (t1, t2) == (t1b, t2b), (i, t1, t2, t1b, t2b)
            if a == "fov":
                assert b == "fov"
                seen["fov"] += 1
                break
            seen["ticks"] += 1
            (hx, ht), (gx, gt) = host.window, dev.window
            assert bits(gx) == bits(hx) and bits(gt) == bits(ht), (i, t1, t2)
            seen["two_messages"] += sum(bool(((ht >= lo) & (ht <= hi)).any()) for lo, hi in spans) == 2
            seen["t2_on_column"] += int((ht == t2).sum()) == 2 and int((host.ref.times() == t2).sum()) > 2
            rh, rd = host.result(), dev.result()
            if a == "gated":
                seen["gated"] += 1
                if rh[4] >= 0:                                    # an update ran before: the device's fetched status says the gate
                    assert rd[0] == lv.TOO_FEW_POINTS, (i, t2)
                assert bits(rh[2]) == bits(rd[2]) and bits(rh[3]) == bits(rd[3]) and rh[4] == rd[4], (i, t2)
            else:
                seen["updates"] += a == lv.OK
                assert rh[0] == rd[0] and rh[4] == rd[4], (i, t2, rh[0], rd[0], rh[4], rd[4])
                assert bits(rh[2]) == bits(rd[2]) and bits(rh[3]) == bits(rd[3]), (i, t2)
                assert len(rh[1]) == len(rd[1]) and all(
                    all(np.array_equal(p[k], q[k], equal_nan=True) for k in p) for p, q in zip(rh[1], rd[1])), (i, t2)
            assert (host.loc.map_points() == dev.loc.map_points()).all(), (i, t2)
    info = dev.loc.lidar_info()
    assert info["points"] == host.ref.size(), (info, host.ref.size())
    assert dev.loc.async_status() == (lv.OK, "")
    assert seen["ticks"] >= 30 and seen["fov"] >= 1 and seen["gated"] >= 1 and seen["updates"] >= 10, seen
    assert seen["two_messages"] >= 1 and seen["t2_on_column"] >= 1, seen
    assert len(host.loc.map_points()) > 1000
    host.close()
    dev.close()
