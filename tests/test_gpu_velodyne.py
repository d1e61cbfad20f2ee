"""lv_process_velodyne_device(_async) — Accumulator::process on a VelodyneScan's packets in HBM — against the host chain, bit for bit:
lv_velodyne_to_points, lv_temporal_downsample on its output (the rank among the msg2points points), lv_time_sort_indices, then the
gathers.  The uploaded rotation tables read back entry for entry.  Then the deferred flags (a dual-return packet, a stamp that does not convert), the launch count, the async count into the
LiDAR buffer with lanes, a stream of synthetic VLP-16 scans through the windowed device tick against the host decode plus push, and
two VLP-16 streams merged through their extrinsics against the restated merge."""
import ctypes as C

import numpy as np
import pytest
from scipy.spatial import cKDTree

import frontend_ref as F
import lidar_merge_ref as M
import velodyne_cases as VC
from test_gpu_async_tick import Bufs, get_count, put_count
from test_gpu_full_points import FullBuffer, FullChain, same_full
from test_gpu_lidar_buffer import EMPTY_LIDAR_TIME, MD, RATE, WindowChain, bits
from test_gpu_lidar_merge import TwoSensorWorld, _Scene, second_sensor
from test_gpu_world_clouds import upload

pytestmark = pytest.mark.gpu
f32 = np.float32


@pytest.fixture(scope="module")
def loc(lv):
    h = lv.Localizer(lv.default_params(max_points=1 << 18, max_map_points=1 << 16))
    yield h
    h.close()


def host_chain(lv, loc, pk, cal, rate, md):
    """lv_velodyne_to_points -> lv_temporal_downsample (device, on the point list) -> lv_time_sort_indices"""
    xyz, t, inten, rg, idx = lv.velodyne_to_points(pk.tobytes(), cal)
    _, keep = loc.temporal_downsample(xyz, rate, md) if len(xyz) else (None, np.zeros(0, np.int32))
    order = keep[lv.time_sort_indices(t[keep])] if len(keep) else keep
    return xyz[order], t[order], inten[order], rg[order], idx[order]


def same(got, ref, what, fields=5):
    for name, a, b in list(zip(("xyz", "time", "intensity", "range", "idx"), got, ref))[:fields]:
        assert a.shape == b.shape and bits(a) == bits(b), (what, name, a.shape, b.shape)


def device_run(loc, d_msg, shift, pk, cal, rate, md, outs, d_n=None, optional=True):
    """the packets at d_msg + shift; the synchronous form, or the async one with its count at d_n.  optional=False passes NULL for
    intensity, range and idx"""
    raw = np.frombuffer(pk.tobytes(), np.uint8)
    if len(raw):
        upload(loc, d_msg + shift, raw)
    o = outs if optional else outs[:2] + [None] * 3
    if d_n is None:
        m = loc.process_velodyne_device(d_msg + shift, len(raw), len(pk), cal, rate, md, *o)
    else:
        put_count(loc, d_n, -5)
        loc.process_velodyne_device_async(d_msg + shift, len(raw), len(pk), cal, rate, md, o[0], o[1], d_n, *o[2:])
        m = get_count(loc, d_n)
    host = (np.empty((m, 3), f32), np.empty(m), np.empty(m, f32), np.empty(m, f32), np.empty(m, np.int32))
    return tuple(loc.download(d, a) for d, a in zip(outs, host))


# ---- sizes x rates, both forms, at odd addresses, every output optional -------------------------------------------------------------
@pytest.mark.parametrize("n_packets", [0, 1, 76, 754])
def test_process_velodyne_equals_the_host_chain(lv, loc, n_packets):
    rng = np.random.default_rng(100 + n_packets)
    pk = VC.packets(rng, n_packets, sec=1_712_345_678, nsec=999_900_000)     # the ns -> s carry inside the scan
    cals = [VC.calibration(lv), VC.random_calibration(lv, rng)]
    n = 384 * n_packets
    b = Bufs(loc)
    d_msg = b(1214 * n_packets + 16)
    outs = [b(k * max(n, 1)) for k in (12, 8, 4, 4, 4)]
    d_n = b(8)
    seen = 0
    for c, cal in enumerate(cals):
        for rate in (1, 2, 4, 7):
            md = 3.0 if rate % 2 else 0.0
            ref = host_chain(lv, loc, pk, cal, rate, md)
            same(ref, VC.process(pk, cal, rate, md), ("restatement", n_packets, c, rate))
            for shift, asyn, optional in ((1, False, True), (3, True, True), (5, False, False), (7, True, False)):
                got = device_run(loc, d_msg, shift, pk, cal, rate, md, outs, d_n if asyn else None, optional)
                same(got, ref, (n_packets, c, rate, shift, asyn), 5 if optional else 2)
            seen += len(ref[0]) > 0
    assert loc.async_status() == (lv.OK, "")
    if n_packets:
        assert seen == 8
    b.free()


def test_edge_packets_and_launches(lv):
    loc = lv.Localizer(lv.default_params(max_points=1 << 14, max_map_points=1 << 12))
    rng = np.random.default_rng(3)
    cal = VC.calibration(lv)
    b = Bufs(loc)
    d_msg = b(1214 * 16)
    outs = [b(k * 384 * 16) for k in (12, 8, 4, 4, 4)]
    d_n = b(8)
    for name, pk in VC.edge_packets(rng).items():
        for rate, md in ((1, 0.0), (3, 0.9), (8, 3.0)):
            ref = VC.process(pk, cal, rate, md)
            same(host_chain(lv, loc, pk, cal, rate, md), ref, (name, rate))
            same(device_run(loc, d_msg, 1, pk, cal, rate, md, outs), ref, (name, rate))
            same(device_run(loc, d_msg, 2, pk, cal, rate, md, outs, d_n), ref, (name, rate, "async"))
    assert loc.async_status() == (lv.OK, "")
    loc.profile()                                                     # reset the counters
    device_run(loc, d_msg, 0, VC.packets(rng, 10), cal, 4, 3.0, outs)
    assert loc.profile()["total_launches"] == 9
    device_run(loc, d_msg, 0, VC.packets(rng, 10), cal, 4, 3.0, outs, d_n)
    assert loc.profile()["total_launches"] == 9
    assert loc.async_status() == (lv.OK, "")
    b.free()
    loc.close()


def test_device_rotation_tables_are_float64_rounded(lv):
    """the tables the first call uploads, read back through the device decoder entry for entry (velodyne_cases.table_packets)"""
    loc = lv.Localizer(lv.default_params(max_points=1 << 14, max_map_points=1 << 12))
    pk = VC.table_packets()
    raw = np.frombuffer(pk.tobytes(), np.uint8)
    n = 384 * len(pk)
    b = Bufs(loc)
    d_msg = b.upload(raw)
    d_xyz, d_t, d_idx = b(12 * n), b(8 * n), b(4 * n)
    m = loc.process_velodyne_device(d_msg, len(raw), len(pk), lv.VelodyneCalibration(), 1, 0.0, d_xyz, d_t, None, None, d_idx)
    assert m == n
    c, s = VC.tables_from_points(loc.download(d_xyz, np.empty((n, 3), f32)), loc.download(d_idx, np.empty(n, np.int32)))
    want_c, want_s = VC.tables()
    assert bits(c) == bits(want_c) and bits(s) == bits(want_s)
    assert loc.async_status() == (lv.OK, "")
    b.free()
    loc.close()


# ---- the deferred flags ---------------------------------------------------------------------------------------------------------------
def test_dual_return_and_stamp_flags(lv):
    loc = lv.Localizer(lv.default_params(max_points=1 << 14, max_map_points=1 << 12))
    rng = np.random.default_rng(4)
    cal = VC.calibration(lv)
    b = Bufs(loc)
    d_msg = b(1214 * 8)
    outs = [b(k * 384 * 8) for k in (12, 8, 4, 4, 4)]
    d_n = b(8)
    L = loc.L
    for name, pk in (("dual", VC.dual_packets(rng)), ("stamp", VC.bad_stamp_packets(rng))):
        ref = VC.process(pk, cal, 2, 0.0)                             # the other packets' points, the times as the rule computes them
        assert len(ref[0]) > 500
        if name == "dual":
            same(host_chain(lv, loc, pk, cal, 2, 0.0), ref, name)       # the host decoder skips the packet
        else:
            with pytest.raises(RuntimeError):
                lv.velodyne_to_points(pk.tobytes(), cal)              # the host decoder refuses the stamp
        raw = np.frombuffer(pk.tobytes(), np.uint8)
        upload(loc, d_msg + 1, raw)
        m = C.c_int64(-1)
        st = L.lv_process_velodyne_device(loc.h, d_msg + 1, len(raw), len(pk), C.byref(cal), 2, 0.0, *outs, C.byref(m))
        assert st == lv.ERR_ARG and m.value == 0, name
        assert b"process velodyne: a packet is a dual-return one" in L.lv_last_error()
        got = tuple(loc.download(d, np.empty_like(a)) for d, a in zip(outs, ref))
        same(got, ref, (name, "sync outputs"))
        assert loc.async_status() == (lv.OK, "")                      # the synchronous form raises no deferred flag
        got = device_run(loc, d_msg, 3, pk, cal, 2, 0.0, outs, d_n)
        same(got, ref, (name, "async"))
        st, msg = loc.async_status()
        assert st == lv.ERR_ARG and "process velodyne: a packet is a dual-return one" in msg, (name, msg)
        assert loc.async_status() == (lv.OK, "")                      # read and cleared
        good = VC.packets(rng, 5)                                     # the next call starts clean
        same(device_run(loc, d_msg, 0, good, cal, 2, 0.0, outs, d_n), VC.process(good, cal, 2, 0.0), (name, "after"))
        same(device_run(loc, d_msg, 0, good, cal, 2, 0.0, outs), VC.process(good, cal, 2, 0.0), (name, "after sync"))
        assert loc.async_status() == (lv.OK, "")
    b.free()
    loc.close()


def test_refusals_leave_the_handle_untouched(lv):
    loc = lv.Localizer(lv.default_params(max_points=1 << 14, max_map_points=1 << 12))
    rng = np.random.default_rng(12)
    cal = VC.calibration(lv)
    pk = VC.packets(rng, 10)
    raw = np.frombuffer(pk.tobytes(), np.uint8)
    b = Bufs(loc)
    d_msg = b.upload(raw)
    outs = [b(k * 3840) for k in (12, 8, 4, 4, 4)]
    d_n = b(8)
    ref = VC.process(pk, cal, 4, 3.0)
    bad = VC.calibration(lv)
    bad.dist_correction[3] = float("nan")
    L = loc.L
    loc.profile()
    m = C.c_int64(-1)
    for kw in (dict(k=11), dict(cal=bad), dict(out0=d_msg + 100), dict(k=-1)):
        k, c = kw.get("k", 10), kw.get("cal", cal)
        o = [kw.get("out0", outs[0])] + outs[1:]
        assert L.lv_process_velodyne_device(loc.h, d_msg, len(raw), k, C.byref(c), 4, 3.0, *o, C.byref(m)) == lv.ERR_ARG, kw
        assert m.value == 0
        put_count(loc, d_n, 123)
        assert L.lv_process_velodyne_device_async(loc.h, d_msg, len(raw), k, C.byref(c), 4, 3.0, *o, d_n) == lv.ERR_ARG, kw
        assert get_count(loc, d_n) == 123                               # the count was not written
    assert loc.profile()["total_launches"] == 0
    assert loc.process_velodyne_device(d_msg, len(raw), 10, cal, 4, 3.0, *outs) == len(ref[0])
    got = tuple(loc.download(d, np.empty_like(a)) for d, a in zip(outs, ref))
    same(got, ref, "after the refusals")
    assert loc.async_status() == (lv.OK, "")
    b.free()
    loc.close()


# ---- the async count into the LiDAR buffer with lanes ------------------------------------------------------------------------------
def test_async_count_feeds_the_full_buffer(lv, loc):
    rng = np.random.default_rng(9)
    cal = VC.calibration(lv)
    dev, ref = FullBuffer(loc, 1 << 17, 1 << 17), FullBuffer(loc, 1 << 17, 1 << 17)   # one ring per handle: ref is replayed after dev
    b = Bufs(loc)
    d_msg = b(1214 * 76 + 8)
    msgs = []
    for i in range(5):
        k = int(rng.integers(20, 76))
        msgs.append((VC.packets(rng, k, sec=20, nsec=i * 100_000_000), 1 + i % 4))
    windows = [(20.0, 20.05), (20.1, 20.25), (-np.inf, np.inf), (20.2, 20.2 + 1e-6), (20.3, 20.6)]
    for pk, rate in msgs:
        raw = np.frombuffer(pk.tobytes(), np.uint8)
        upload(loc, d_msg + 1, raw)
        put_count(loc, dev.d_n, -1)
        loc.process_velodyne_device_async(d_msg + 1, len(raw), len(pk), cal, rate, MD, dev.d_in[0], dev.d_in[1], dev.d_n, dev.d_in[2],
                                          dev.d_in[3])
        loc.lidar_push_full_async(*dev.d_in, dev.d_n, 384 * len(pk))
    got = [dev.get(t1, t2) for t1, t2 in windows]
    loc.lidar_clear_async(np.inf)
    loc.lidar_reserve_full(1 << 17)
    for pk, rate in msgs:                                              # the host-decoded points, pushed
        xyz, t, inten, rg, _ = host_chain(lv, loc, pk, cal, rate, MD)
        ref.push(xyz, t, inten, rg)
    for (t1, t2), g in zip(windows, got):
        same_full(g, ref.get(t1, t2), (t1, t2))
    assert sum(len(g[1]) for g in got) > 10000
    assert loc.async_status() == (lv.OK, "")
    loc.lidar_clear_async(np.inf)
    dev.close()
    ref.close()
    b.free()


# ---- synthetic VLP-16 scans through the windowed device tick --------------------------------------------------------------------------
SCAN_PACKETS = 75                                                     # 75 x 12 blocks x 0.4 deg: one turn in 99.5 ms


def vlp16_scans(lv, sc, n_msgs=6, cut=3, stamp0=10 * 10**9, world=None):
    """10 Hz VelodyneScans of the synthetic world: each slot's return is the world point nearest to the slot's beam (its laser's
    elevation, its firing's azimuth clockwise from +x), its range in 2 mm units; message `cut` keeps one packet (a gated window)"""
    world = world or sc.world
    rng = np.random.default_rng(51)
    el = np.array(VC.VLP16_DEG, np.float64)
    msgs = []
    for i in range(n_msgs):
        sw = world.sweep(world.pose(8.0 + 0.1 * i, sc.prm), rings=61, azimuths=3600, elev=(-15.0, 15.0), seed=400 + i).astype(np.float64)
        r = np.linalg.norm(sw, axis=1)
        ang = np.stack([np.mod(np.degrees(np.arctan2(-sw[:, 1], sw[:, 0])), 360.0), np.degrees(np.arcsin(sw[:, 2] / r))], 1)
        tree = cKDTree(ang)
        pk = VC.packets(rng, SCAN_PACKETS, az0=int(rng.integers(0, 36000)), step=40, sec=stamp0 // 10**9 + i // 10,
                        nsec=stamp0 % 10**9 + (i % 10) * 100_000_000, zero=0.0)
        slot = np.arange(384 * SCAN_PACKETS)
        k, s = slot // 384, slot % 384
        bl, f, l = s // 32, (s % 32) // 16, s % 16
        az = np.mod(pk["data"]["blocks"]["azimuth"][k, bl] * 0.01 + 0.4 * (l * 2.304 + f * 55.296) / 110.592, 360.0)
        dist, j = tree.query(np.stack([az, el[l]], 1))
        raw = np.where((dist < 0.3) & (r[j] < 130.0), np.round(r[j] / 0.002), 0).astype(np.uint16)
        pk["data"]["blocks"]["ch"]["dist"] = raw.reshape(SCAN_PACKETS, 12, 32)
        if i == cut:
            pk = pk[:1]
        raw_bytes = np.frombuffer(pk.tobytes(), np.uint8).copy()
        msgs.append(dict(pk=pk, raw=raw_bytes, n=384 * len(pk), n_packets=len(pk)))
    return msgs


class VelodyneChain(FullChain):
    """FullChain with VelodyneScans: on the device lv_process_velodyne_device_async -> lv_lidar_push_full_device_async; otherwise the
    host decode (lv_velodyne_to_points, the decimator on the rank, lv_time_sort_indices) pushed onto the restated deque"""

    def receive(self, g):
        cal = self.lv.velodyne_calibration()
        if not self.device:
            xyz, t, inten, rg, _ = self.lv.velodyne_to_points(g["raw"], cal)
            keep = F.temporal(xyz, RATE, MD)
            order = keep[self.lv.time_sort_indices(t[keep])]
            self.ref.push_message(xyz[order], t[order], inten[order], rg[order])
            return t[order]
        upload(self.loc, self.d_msg, g["raw"])
        self.loc.process_velodyne_device_async(self.d_msg, len(g["raw"]), g["n_packets"], cal, RATE, MD, self.d_p[0], self.d_p[1], self.d_k,
                                               self.d_p[2], self.d_p[3])
        self.loc.lidar_push_full_async(*self.d_p, self.d_k, g["n"])
        return None


def test_vlp16_stream_through_the_device_tick_equals_the_host_chain(lv, scene_xaloc):
    sc = scene_xaloc
    msgs = vlp16_scans(lv, sc)
    host, dev = VelodyneChain(lv, sc, "velodyne", msgs, 0.02, False), VelodyneChain(lv, sc, "velodyne", msgs, 0.02, True)
    seen = dict(ticks=0, gated=0, updates=0)
    latest = -np.inf
    for i, g in enumerate(msgs):
        latest = max(latest, float(host.receive(g).max()))
        dev.receive(g)
        for _ in range(14):
            a, b = host.tick(latest), dev.tick(latest)
            assert a == b and host.t2 == dev.t2, (i, a, b)
            if a == "fov":
                break
            seen["ticks"] += 1
            rh, rd = host.result(), dev.result()
            assert bits(rh[2]) == bits(rd[2]) and bits(rh[3]) == bits(rd[3]) and rh[4] == rd[4], (i, host.t2)
            assert bits(host.loc.map_points()) == bits(dev.loc.map_points()), (i, host.t2)
            if a == "gated":                                          # the host chain runs no update, so it keeps the last status
                seen["gated"] += 1
                continue
            assert rh[0] == rd[0] and len(rh[1]) == len(rd[1]) and all(
                all(np.array_equal(p[k], q[k], equal_nan=True) for k in p) for p, q in zip(rh[1], rd[1])), (i, host.t2)
            seen["updates"] += rh[0] == lv.OK
            for key in ("ds", "full"):
                same_full(dev.published[key], host.published[key], (i, host.t2, key))
            assert dev.published["stamps"] == host.published["stamps"]
    assert dev.loc.async_status() == (lv.OK, "")
    assert seen["ticks"] >= 15 and seen["gated"] >= 1 and seen["updates"] >= 5, seen
    host.close()
    dev.close()


# ---- two VLP-16 streams merged through their extrinsics -------------------------------------------------------------------------------
class VelodyneMergeChain(WindowChain):
    """WindowChain over two VLP-16 streams, the second one's scans merged through L0_T_L1: the device chain runs
    lv_process_velodyne_device_async -> lv_lidar_merge_device_async; the host chain processes synchronously and merges on the restated
    buffer"""

    def __init__(self, lv, sc, msgs, delta, device):
        super().__init__(lv, sc, msgs, delta, device)
        self.ref = M.MergeBuffer()
        if device:
            self.loc.lidar_reserve(6 * self.nm // RATE)
            self.loc.lidar_reserve_merge(2 * self.nm // RATE)

    def receive(self, g):
        loc, cal = self.loc, self.lv.velodyne_calibration()
        upload(loc, self.d_msg, g["raw"])
        args = (self.d_msg, len(g["raw"]), g["n_packets"], cal, RATE, MD, self.d_pxyz, self.d_pt)
        if self.device:
            loc.process_velodyne_device_async(*args, self.d_k)
            loc.lidar_merge_async(self.d_pxyz, self.d_pt, self.d_k, g["n"], g["T"])
            return None
        k = loc.process_velodyne_device(*args)
        xyz, t = loc.download(self.d_pxyz, np.empty((k, 3), f32)), loc.download(self.d_pt, np.empty(k))
        assert self.ref.merge_message(xyz, t, g["T"]) == "write"
        return t


def test_two_vlp16_streams_merged_equal_the_restatement_chain(lv, scene_xaloc):
    sc = scene_xaloc
    m0 = vlp16_scans(lv, sc, n_msgs=6, cut=3)
    m1 = vlp16_scans(lv, _Scene(sc, TwoSensorWorld(sc.world)), n_msgs=6, cut=4, stamp0=10 * 10**9 + 47_000_000,
                     world=TwoSensorWorld(sc.world))
    _, T = second_sensor(sc.world.pose(8.0, sc.prm))
    msgs = []
    for a, b in zip(m0, m1):
        a["T"], b["T"] = None, T
        msgs += [a, b]
    host, dev = VelodyneMergeChain(lv, sc, msgs, 0.02, False), VelodyneMergeChain(lv, sc, msgs, 0.02, True)
    seen = dict(ticks=0, updates=0, merged_back=0)
    newest = [-np.inf, -np.inf]
    for i, g in enumerate(msgs):
        before = host.ref.times()
        t_msg = host.receive(g)
        dev.receive(g)
        if len(t_msg) and len(before):
            seen["merged_back"] += float(t_msg.min()) < float(np.nanmax(before))
        newest[i % 2] = max(newest[i % 2], float(t_msg.max()))
        latest = min(newest)                                          # t2 never passes what every sensor has delivered
        if latest == -np.inf:
            continue
        for _ in range(30):
            a, t1, t2 = host.tick(latest)
            b, t1b, t2b = dev.tick(latest)
            assert (t1, t2) == (t1b, t2b), (i, t1, t2, t1b, t2b)
            if a == "fov":
                assert b == "fov"
                break
            seen["ticks"] += 1
            (hx, ht), (gx, gt) = host.window, dev.window
            assert bits(gx) == bits(hx) and bits(gt) == bits(ht), (i, t1, t2)
            rh, rd = host.result(), dev.result()
            if a == "gated":
                if rh[4] >= 0:
                    assert rd[0] == lv.TOO_FEW_POINTS, (i, t2)
                assert bits(rh[2]) == bits(rd[2]) and bits(rh[3]) == bits(rd[3]) and rh[4] == rd[4], (i, t2)
            else:
                seen["updates"] += a == lv.OK
                assert rh[0] == rd[0] and rh[4] == rd[4], (i, t2, rh[0], rd[0], rh[4], rd[4])
                assert bits(rh[2]) == bits(rd[2]) and bits(rh[3]) == bits(rd[3]), (i, t2)
            assert (host.loc.map_points() == dev.loc.map_points()).all(), (i, t2)
    assert dev.loc.async_status() == (lv.OK, "")
    assert seen["ticks"] >= 15 and seen["updates"] >= 5 and seen["merged_back"] >= 3, seen
    tc = t2 - EMPTY_LIDAR_TIME
    host.ref.clear(tc)
    dev.loc.lidar_clear_async(tc)
    assert dev.loc.lidar_info()["points"] == host.ref.size()
    host.close()
    dev.close()
