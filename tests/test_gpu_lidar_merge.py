"""The time-ordered merge of the LiDAR buffer in HBM (lv_lidar_merge(_full)_device_async) against tests/lidar_merge_ref.py, bit for
bit: messages that do not reach back into the buffer give exactly what the push gives; interleaved messages of two and three
sensors with random overlaps and equal-time ties, 0 to 240 000 points at odd addresses, with and without transforms and lanes, give
the restatement's windows and content after every merge; the refusals and the unsorted case leave the handle usable, and a merge
costs the same launches whatever its overlap.  Then two synthetic spinning LiDARs, each seen from its own extrinsic, run through the
windowed device tick (process, merge with L0_T_L1, get, compensate, voxel grid, correct, map add, clear) and equal the chain that
keeps the buffer in the restatement and runs the synchronous device calls."""
import ctypes as C

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import lidar_merge_ref as M
from test_gpu_async_tick import Bufs, get_count, put_count
from test_gpu_cloud_frontend import FRT
from test_gpu_lidar_buffer import EMPTY_LIDAR_TIME, MD, RATE, WindowChain, bits, sequence_messages

pytestmark = pytest.mark.gpu
f32 = np.float32
INF = float("inf")


def upload(loc, d, a):
    a = np.ascontiguousarray(a)
    if a.nbytes:
        assert loc.L.lv_memcpy_h2d(loc.h, C.c_void_p(d), a.ctypes.data_as(C.c_void_p), a.nbytes) == 0


class Ring:
    """one handle's buffer with staging: messages at odd addresses (one element past an allocation's start), windows back"""

    def __init__(self, lv, cap, reserve, n_max, lanes, window_max=None):
        self.lv, self.lanes, self.n_max = lv, lanes, n_max
        self.loc = lv.Localizer(lv.default_params(max_points=1 << 12, max_map_points=1 << 12))
        self.b = Bufs(self.loc)
        self.d_xyz, self.d_t = self.b(12 * n_max + 16) + 4, self.b(8 * n_max + 16) + 8
        self.d_i, self.d_r, self.d_n = self.b(4 * n_max + 8) + 4, self.b(4 * n_max + 8) + 4, self.b(16) + 8
        self.w_max = window_max or cap
        self.w = [self.b(k * self.w_max) for k in (12, 8, 4, 4)] + [self.b(8)]
        (self.loc.lidar_reserve_full if lanes else self.loc.lidar_reserve)(cap)
        if reserve:
            self.loc.lidar_reserve_merge(reserve)

    def _stage(self, xyz, t, inten, rng):
        n = len(t)
        upload(self.loc, self.d_xyz, np.asarray(xyz, f32))
        upload(self.loc, self.d_t, np.asarray(t, np.float64))
        if inten is not None:
            upload(self.loc, self.d_i, np.asarray(inten, f32))
            upload(self.loc, self.d_r, np.asarray(rng, f32))
        put_count(self.loc, self.d_n, n)
        return max(n, 1)

    def merge(self, xyz, t, T=None, inten=None, rng=None):
        n_max = self._stage(xyz, t, inten, rng)
        if inten is not None:
            self.loc.lidar_merge_full_async(self.d_xyz, self.d_t, self.d_i, self.d_r, self.d_n, n_max, T)
        else:
            self.loc.lidar_merge_async(self.d_xyz, self.d_t, self.d_n, n_max, T)

    def push(self, xyz, t, inten=None, rng=None):
        n_max = self._stage(xyz, t, inten, rng)
        if inten is not None:
            self.loc.lidar_push_full_async(self.d_xyz, self.d_t, self.d_i, self.d_r, self.d_n, n_max)
        else:
            self.loc.lidar_push_async(self.d_xyz, self.d_t, self.d_n, n_max)

    def window(self, t1, t2):
        """the get's window: (xyz, time[, intensity, range])"""
        loc, (wx, wt, wi, wr, wn) = self.loc, self.w
        put_count(loc, wn, -3)
        if self.lanes:
            loc.lidar_get_points_full_async(t1, t2, wx, wt, wi, wr, self.w_max, wn)
        else:
            loc.lidar_get_points_async(t1, t2, wx, wt, self.w_max, wn)
        m = get_count(loc, wn)
        out = [loc.download(wx, np.empty((m, 3), f32)), loc.download(wt, np.empty(m))]
        if self.lanes:
            out += [loc.download(wi, np.empty(m, f32)), loc.download(wr, np.empty(m, f32))]
        return out

    def close(self):
        self.b.free()
        self.loc.close()


def same_windows(a, b, what):
    assert len(a) == len(b) and all(x.shape == y.shape and bits(x) == bits(y) for x, y in zip(a, b)), what


def ref_window(ref, t1, t2, lanes):
    return list(ref.get(t1, t2)) if lanes else list(ref.get(t1, t2))[:2]


def same_info(ring, ref, what):
    info = ring.loc.lidar_info()
    assert info["points"] == ref.size(), (what, info, ref.size())
    if ref.size():
        assert bits(np.float64(info["newest_time"])) == bits(np.float64(ref.content[0][0])), what
        assert bits(np.float64(info["oldest_time"])) == bits(np.float64(ref.content[-1][0])), what


def column_message(rng, start_tick, n, span_ticks, tick=1e-5):
    """n points whose times lie on a shared grid of ticks (equal times inside a message and across sensors), sorted"""
    t = (start_tick + np.sort(rng.integers(0, span_ticks, n))) * tick
    xyz = rng.normal(0, 20, (n, 3)).astype(f32)
    return xyz, t, rng.uniform(0, 255, n).astype(f32), rng.uniform(1, 90, n).astype(f32)


# ---- 4: merges that do not reach back are the push -----------------------------------------------------------------------------
@pytest.mark.parametrize("lanes", [False, True])
def test_non_overlapping_merges_equal_the_push(lv, lanes):
    rng = np.random.default_rng(11 + lanes)
    cap = 30_000
    merged, pushed = Ring(lv, cap, 1000, 8000, lanes), Ring(lv, cap, 0, 8000, lanes)
    ref = M.MergeBufferFull() if lanes else M.MergeBuffer()
    tick, total = 0, 0
    for step in range(70):
        n = int(rng.choice([0, 1, 7, 500, 4000, 8000]))
        xyz, t, inten, rg = column_message(rng, tick, n, 400)
        if not lanes or rng.random() < 0.3:
            inten = rg = None
        if ref.size() + n > cap:
            tc = float(ref.content[0][0]) - 2e-3
            ref.clear(tc)
            merged.loc.lidar_clear_async(tc)
            pushed.loc.lidar_clear_async(tc)
        T = M.random_extrinsic(rng) if step % 3 == 0 else None
        merged.merge(xyz, t, T, inten, rg)
        pushed.push(M.rt_apply(T, xyz) if T is not None else xyz, t, inten, rg)
        if lanes:
            ref.merge_message(xyz, t, T, inten, rg)
        else:
            ref.merge_message(xyz, t, T)
        total += n
        tick = int(round(t[-1] / 1e-5)) if n else tick            # the next message may start on the newest time
        a, b = merged.loc.lidar_info(), pushed.loc.lidar_info()
        assert bits(np.array(list(a.values()), np.float64)) == bits(np.array(list(b.values()), np.float64)), (step, a, b)
        same_info(merged, ref, step)
        for t1, t2 in [(-INF, INF)] + [tuple(sorted(rng.uniform(t[0] - 0.01, t[-1] + 1e-3, 2))) for _ in range(2) if n]:
            w = merged.window(t1, t2)
            same_windows(w, pushed.window(t1, t2), (step, t1, t2))
            same_windows(w, ref_window(ref, t1, t2, lanes), (step, t1, t2, "ref"))
    assert total > 3 * cap                                        # wrapped
    for r in (merged, pushed):
        assert r.loc.async_status() == (lv.OK, "")
        r.close()


# ---- 5: interleaved sensors --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sensors,lanes,transform", [(2, False, False), (2, True, True), (3, False, True), (3, True, False)])
def test_interleaved_sensors_equal_the_restatement(lv, sensors, lanes, transform):
    rng = np.random.default_rng(100 * sensors + 10 * lanes + transform)
    cap, n_big = 1_200_000, 240_000
    reserve = cap                                                  # every merge goes through: the refusals are test 6's
    ring = Ring(lv, cap, reserve, n_big, lanes, window_max=cap)
    ref = M.MergeBufferFull(cap, reserve) if lanes else M.MergeBuffer(cap, reserve)
    Ts = [None] + [M.random_extrinsic(rng) if transform else None for _ in range(sensors - 1)]
    sizes = [0, 1, 7] + [24_000] * 5 + [240_000]
    clock, seen = 0, dict(merged_back=0, ties=0, big=0, empty=0)
    for step in range(20):
        k = step % sensors
        n = sizes[int(rng.integers(0, len(sizes)))] if step != 3 else n_big
        span = 10_000                                              # 0.1 s of ticks
        back = int(rng.choice([0, span // 4, span // 2, span]))
        xyz, t, inten, rg = column_message(rng, clock - back, n, span)
        if not lanes or rng.random() < 0.2:
            inten = rg = None
        if ref.size() + n > cap:
            tc = float(np.sort(ref.times())[ref.size() // 2])
            ref.clear(tc)
            ring.loc.lidar_clear_async(tc)
        L_ = list(reversed(ref.content))
        split = M.split_of(L_, t[0]) if n else len(L_)
        ring.merge(xyz, t, Ts[k], inten, rg)
        mode = ref.merge_message(xyz, t, Ts[k], inten, rg) if lanes else ref.merge_message(xyz, t, Ts[k])
        assert mode == "write", (step, mode)
        seen["merged_back"] += split < len(L_) and n > 0
        seen["ties"] += n > 0 and bool(np.isin(t, [p[0] for p in L_[split:]]).any())
        seen["big"] += n == n_big
        seen["empty"] += n == 0
        clock = max(clock, int(round(t[-1] / 1e-5)) if n else clock)
        same_info(ring, ref, step)
        for _ in range(3):
            t1 = float(rng.uniform(clock - 3 * span, clock)) * 1e-5
            t2 = t1 + float(rng.choice([0.005, 0.02, 0.1]))
            same_windows(ring.window(t1, t2), ref_window(ref, t1, t2, lanes), (step, t1, t2))
    same_windows(ring.window(-INF, INF), ref_window(ref, -INF, INF, lanes), "content")
    assert ring.loc.async_status() == (lv.OK, "")
    assert seen["merged_back"] >= 8 and seen["ties"] >= 4 and seen["big"] >= 1, seen
    ring.close()


# ---- 6: refusals, the unsorted case and the launch count ---------------------------------------------------------------------------
def test_refusals_unsorted_and_launches(lv):
    rng = np.random.default_rng(6)
    ring = Ring(lv, 3000, 500, 2000, False)
    ref = M.MergeBuffer(3000, 500)
    loc = ring.loc

    def do(xyz, t, T=None):
        ring.merge(xyz, t, T)
        return ref.merge_message(xyz, t, T)

    def check(what):
        same_info(ring, ref, what)
        same_windows(ring.window(-INF, INF), ref_window(ref, -INF, INF, False), what)

    xyz, t, _, _ = column_message(rng, 0, 2000, 1000)
    assert do(xyz, t) == "write"
    check("first")
    # reaches back over more than 500 buffered points: refused, nothing changes
    xyz2, t2, _, _ = column_message(rng, 200, 300, 100)
    assert do(xyz2, t2) == "overlap"
    st, msg = loc.async_status()
    assert st == lv.ERR_ARG and "lidar merge" in msg and "merge reserve" in msg, msg
    check("overlap")
    # does not fit: refused, nothing changes
    xyz3, t3, _, _ = column_message(rng, 990, 1500, 20)
    assert do(xyz3, t3) == "full"
    st, msg = loc.async_status()
    assert st == lv.ERR_ARG and "do not fit" in msg and "merge" in msg, msg
    check("full")
    # unsorted input: appended as the push does, reported
    t4 = t3[:400][::-1].copy()
    assert do(xyz3[:400], t4) == "append"
    st, msg = loc.async_status()
    assert st == lv.ERR_ARG and "not time-ordered" in msg, msg
    check("unsorted")
    # a NaN time: appended too
    t5 = np.array([0.02, np.nan, 0.03])
    assert do(xyz3[:3], t5) == "append"
    assert "not time-ordered" in loc.async_status()[1]
    info = loc.lidar_info()
    assert info["points"] == ref.size()
    # usable afterwards: clear everything, merge again
    loc.lidar_clear_async(INF)
    ref.clear(INF)                                              # a NaN stops the clear in both
    check("cleared")
    loc.lidar_clear_async(INF)
    assert loc.lidar_info()["points"] == ref.size()
    ring2 = Ring(lv, 3000, 500, 2000, False)
    ref2 = M.MergeBuffer(3000, 500)
    launches = []
    for back in (0, 100, 490):                                   # no overlap, some, nearly the reserve
        xa, ta, _, _ = column_message(rng, 10_000, 500, 500)
        xb, tb, _, _ = column_message(rng, 10_500 - back, 500, 500)
        ring2.loc.lidar_clear_async(INF)
        ref2.clear(INF)
        ring2.merge(xa, ta)
        assert ref2.merge_message(xa, ta) == "write"
        ring2.loc.profile()                                       # reset the counters
        ring2.merge(xb, tb)
        assert ref2.merge_message(xb, tb) == "write"
        launches.append(ring2.loc.profile()["total_launches"])
        same_windows(ring2.window(-INF, INF), ref_window(ref2, -INF, INF, False), back)
    assert launches == [3, 3, 3], launches
    assert ring2.loc.async_status() == (lv.OK, "")
    ring2.close()
    ring.close()


def test_argument_refusals_that_need_a_handle(lv):
    L = lv.lib()
    loc = lv.Localizer(lv.default_params(max_points=1 << 12, max_map_points=1 << 12))
    b = Bufs(loc)
    d, d_n = b(4096), b(8)
    T = lv._transform12(np.eye(3, 4, dtype=f32).ravel())
    assert L.lv_lidar_merge_device_async(loc.h, d, d + 1200, d_n, 1, T) == lv.ERR_ARG and b"lv_lidar_reserve first" in L.lv_last_error()
    loc.lidar_reserve(100)
    assert L.lv_lidar_merge_device_async(loc.h, d, d + 1200, d_n, 1, None) == lv.ERR_ARG
    assert b"lv_lidar_reserve_merge first" in L.lv_last_error()
    loc.lidar_reserve_merge(10)
    assert L.lv_lidar_merge_full_device_async(loc.h, d, d + 1200, d + 2000, d + 2400, d_n, 1, None) == lv.ERR_ARG
    assert b"lv_lidar_reserve_full first" in L.lv_last_error()
    # the scratch gains lanes with the ring
    loc.lidar_reserve_full(100)
    put_count(loc, d_n, 0)
    assert L.lv_lidar_merge_full_device_async(loc.h, d, d + 1200, d + 2000, d + 2400, d_n, 1, None) == lv.OK
    assert loc.async_status() == (lv.OK, "") and loc.lidar_info()["points"] == 0
    b.free()
    loc.close()


# ---- 7: two spinning LiDARs through the windowed device tick -------------------------------------------------------------------------
def quat_rot(q):
    return Rotation.from_quat(q).as_matrix()                       # (x, y, z, w), the state's order


def second_sensor(x0):
    """the state seen by a second LiDAR: its own IMU-frame extrinsic, and L0_T_L1 = inv(I_T_L0) * I_T_L1"""
    R0, t0 = quat_rot(x0[7:11]), x0[11:14]
    q1 = (Rotation.from_quat(x0[7:11]) * Rotation.from_euler("zyx", [100.0, 4.0, -3.0], degrees=True)).as_quat()
    t1 = t0 + np.array([0.35, -0.6, 0.12])
    x1 = x0.copy()
    x1[7:11], x1[11:14] = q1, t1
    R1 = quat_rot(q1)
    T = np.concatenate([(R0.T @ R1).ravel(), R0.T @ (t1 - t0)]).astype(f32)
    return x1, T


class MergeChain(WindowChain):
    """WindowChain whose messages come from two sensors: the second one's merged through L0_T_L1"""

    def __init__(self, lv, sc, msgs, delta, device):
        super().__init__(lv, sc, msgs, delta, device)
        self.ref = M.MergeBuffer()
        if device:
            self.loc.lidar_reserve(6 * self.nm // RATE)
            self.loc.lidar_reserve_merge(2 * self.nm // RATE)

    def receive(self, g):
        loc = self.loc
        assert loc.L.lv_memcpy_h2d(loc.h, C.c_void_p(self.d_msg), g["raw"].ctypes.data_as(C.c_void_p), len(g["raw"])) == 0
        args = ("velodyne", g["layout"], self.d_msg, len(g["raw"]), g["n"], g["stamp"], True, True, FRT, RATE, MD, self.d_pxyz,
                self.d_pt)
        if self.device:
            loc.process_cloud_device_async(*args, self.d_k)
            loc.lidar_merge_async(self.d_pxyz, self.d_pt, self.d_k, g["n"], g["T"])
            return None
        k = loc.process_cloud_device(*args)
        xyz, t = loc.download(self.d_pxyz, np.empty((k, 3), f32)), loc.download(self.d_pt, np.empty(k))
        assert self.ref.merge_message(xyz, t, g["T"]) == "write"
        return t


class TwoSensorWorld:
    """sc.world with every pose carrying the second sensor's extrinsic (lv_synth_sweep reads it from the state)"""

    def __init__(self, world):
        self.world = world

    def pose(self, s, prm):
        return second_sensor(self.world.pose(s, prm))[0]

    def sweep(self, *a, **k):
        return self.world.sweep(*a, **k)


class _Scene:
    def __init__(self, sc, world):
        self.world, self.prm = world, sc.prm


@pytest.mark.parametrize("delta", [0.01, 0.02])
def test_two_sensor_ticks_equal_the_restatement_chain(lv, scene_xaloc, delta):
    sc = scene_xaloc
    m0 = sequence_messages(lv, sc, n_msgs=7, cut=3)
    m1 = sequence_messages(lv, _Scene(sc, TwoSensorWorld(sc.world)), n_msgs=7, cut=5)
    _, T = second_sensor(sc.world.pose(8.0, sc.prm))
    msgs = []
    for a, b in zip(m0, m1):
        a["T"], b["T"] = None, T
        b["stamp"] += 47_000                                       # half a sweep later: the spans overlap, the column times differ
        msgs += [a, b]
    host, dev = MergeChain(lv, sc, msgs, delta, False), MergeChain(lv, sc, msgs, delta, True)
    seen = dict(ticks=0, fov=0, updates=0, both_sensors=0, merged_back=0)
    newest, times, log = [-np.inf, -np.inf], [[], []], []
    for i, g in enumerate(msgs):
        k = i % 2
        before = host.ref.times()
        t_msg = host.receive(g)
        dev.receive(g)
        if len(t_msg) and len(before):
            seen["merged_back"] += float(t_msg.min()) < float(np.nanmax(before))
        newest[k] = max(newest[k], float(t_msg.max()))
        times[k].append(t_msg)
        latest = min(newest)                                       # t2 never passes what every sensor has delivered
        if latest == -np.inf:
            continue                                               # a sensor has delivered nothing yet
        for _ in range(30):
            a, t1, t2 = host.tick(latest)
            b, t1b, t2b = dev.tick(latest)
            log.append((i, str(a), round(t1, 4), round(t2, 4), host.ref.size()))
            assert (t1, t2) == (t1b, t2b), (i, t1, t2, t1b, t2b)
            if a == "fov":
                assert b == "fov"
                seen["fov"] += 1
                break
            seen["ticks"] += 1
            (hx, ht), (gx, gt) = host.window, dev.window
            assert bits(gx) == bits(hx) and bits(gt) == bits(ht), (i, t1, t2)
            s0, s1 = np.concatenate(times[0]), np.concatenate(times[1])
            seen["both_sensors"] += bool(np.isin(ht, s0).any() and np.isin(ht, s1).any())
            rh, rd = host.result(), dev.result()
            if a == "gated":
                if rh[4] >= 0:
                    assert rd[0] == lv.TOO_FEW_POINTS, (i, t2)
                assert bits(rh[2]) == bits(rd[2]) and bits(rh[3]) == bits(rd[3]) and rh[4] == rd[4], (i, t2)
            else:
                seen["updates"] += a == lv.OK
                assert rh[0] == rd[0] and rh[4] == rd[4], (i, t2, rh[0], rd[0], rh[4], rd[4])
                assert bits(rh[2]) == bits(rd[2]) and bits(rh[3]) == bits(rd[3]), (i, t2)
                assert len(rh[1]) == len(rd[1]) and all(
                    all(np.array_equal(p[q], r[q], equal_nan=True) for q in p) for p, r in zip(rh[1], rd[1])), (i, t2)
            assert (host.loc.map_points() == dev.loc.map_points()).all(), (i, t2)
    assert dev.loc.async_status() == (lv.OK, "")
    assert seen["ticks"] >= 20 and seen["updates"] >= 10 and seen["both_sensors"] >= 10 and seen["merged_back"] >= 5, (seen, log)
    tc = t2 - EMPTY_LIDAR_TIME                                     # the device chain also clears after gated ticks (INTEGRATION B5b)
    host.ref.clear(tc)
    dev.loc.lidar_clear_async(tc)
    assert dev.loc.lidar_info()["points"] == host.ref.size()
    assert len(host.loc.map_points()) > 1000
    host.close()
    dev.close()

