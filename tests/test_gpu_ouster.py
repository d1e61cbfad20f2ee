"""lv_process_ouster_device(_async) — Accumulator::process on Ouster LEGACY packets in HBM — against the host chain, bit for bit:
lv_ouster_to_points, lv_temporal_downsample on its output (the rank among the msg2points points), lv_time_sort_indices, then the
gathers.  The uploaded column table reads back entry for entry.  Then the launch count, refusals that leave the handle usable, the
async count into the LiDAR buffer with lanes, and a stream of synthetic OS1-64 frames through the windowed device tick against the
host decode plus push, with the IMU samples of both chains passed through encoded IMU packets."""
import ctypes as C

import numpy as np
import pytest
from scipy.spatial import cKDTree

import frontend_ref as F
import ouster_cases as OC
from test_gpu_async_tick import Bufs, get_count, put_count
from test_gpu_full_points import FullBuffer, FullChain, same_full
from test_gpu_lidar_buffer import MD, RATE, bits
from test_gpu_world_clouds import upload

pytestmark = pytest.mark.gpu
f32 = np.float32


@pytest.fixture(scope="module")
def loc(lv):
    h = lv.Localizer(lv.default_params(max_points=1 << 18, max_map_points=1 << 16))
    yield h
    h.close()


def host_chain(lv, loc, pk, cal, rate, md):
    """lv_ouster_to_points -> lv_temporal_downsample (device, on the point list) -> lv_time_sort_indices"""
    xyz, t, inten, rg, idx = lv.ouster_to_points(pk.tobytes(), cal)
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
        m = loc.process_ouster_device(d_msg + shift, len(raw), len(pk), cal, rate, md, *o)
    else:
        put_count(loc, d_n, -5)
        loc.process_ouster_device_async(d_msg + shift, len(raw), len(pk), cal, rate, md, o[0], o[1], d_n, *o[2:])
        m = get_count(loc, d_n)
    host = (np.empty((m, 3), f32), np.empty(m), np.empty(m, f32), np.empty(m, f32), np.empty(m, np.int32))
    return tuple(loc.download(d, a) for d, a in zip(outs, host))


# ---- sizes x rates, both forms, at odd addresses, every output optional -------------------------------------------------------------
@pytest.mark.parametrize("n_packets,Wc,H", [(0, 1024, 64), (1, 1024, 64), (64, 1024, 64), (128, 2048, 128)])
def test_process_ouster_equals_the_host_chain(lv, loc, n_packets, Wc, H):
    rng = np.random.default_rng(100 + n_packets)
    pk = OC.packets(rng, n_packets, Wc, H, m0=Wc - 100, ts0=1_712_345_678 * 10**9 + 999_900_000)   # frame wrap and ns -> s carry
    cals = [OC.calibration(lv, Wc, H), OC.calibration(lv, Wc, H, OC.ORIGIN_MM, rng)]
    n = 16 * H * n_packets
    b = Bufs(loc)
    d_msg = b(OC.packet_bytes(H) * n_packets + 16)
    outs = [b(k * max(n, 1)) for k in (12, 8, 4, 4, 4)]
    d_n = b(8)
    seen = 0
    for c, cal in enumerate(cals):
        for rate in (1, 2, 4, 7):
            md = 3.0 if rate % 2 else 0.0
            ref = host_chain(lv, loc, pk, cal, rate, md)
            same(ref, OC.process(pk, cal, rate, md), ("restatement", n_packets, c, rate))
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
    cal = OC.calibration(lv, 512, 32)
    b = Bufs(loc)
    d_msg = b(OC.packet_bytes(32) * 8 + 8)
    outs = [b(k * 16 * 32 * 8) for k in (12, 8, 4, 4, 4)]
    d_n = b(8)
    edges = {"invalid": OC.packets(rng, 4, 512, 32, invalid=1.0), "bad_m": OC.packets(rng, 4, 512, 32, bad_m=1.0),
             "no_return": OC.packets(rng, 4, 512, 32, zero=1.0), "mixed": OC.packets(rng, 8, 512, 32, invalid=0.3, bad_m=0.3, zero=0.5),
             "equal_stamps": OC.packets(rng, 3, 512, 32), "near": OC.packets(rng, 3, 512, 32, max_mm=2000)}
    edges["equal_stamps"].reshape(-1)["ts"] = 5 * 10**9                  # equal times keep slot order
    for name, pk in edges.items():
        for rate, md in ((1, 0.0), (3, 0.9), (8, 3.0)):
            ref = OC.process(pk, cal, rate, md)
            same(host_chain(lv, loc, pk, cal, rate, md), ref, (name, rate))
            same(device_run(loc, d_msg, 1, pk, cal, rate, md, outs), ref, (name, rate))
            same(device_run(loc, d_msg, 2, pk, cal, rate, md, outs, d_n), ref, (name, rate, "async"))
    assert loc.async_status() == (lv.OK, "")
    loc.profile()                                                     # reset the counters
    device_run(loc, d_msg, 0, OC.packets(rng, 4, 512, 32), cal, 4, 3.0, outs)
    assert loc.profile()["total_launches"] == 9
    device_run(loc, d_msg, 0, OC.packets(rng, 4, 512, 32), cal, 4, 3.0, outs, d_n)
    assert loc.profile()["total_launches"] == 9
    assert loc.async_status() == (lv.OK, "")
    b.free()
    loc.close()


def test_device_column_table_is_float64_rounded(lv):
    """the table the first call uploads, read back through the device decoder entry for entry (ouster_cases.table_packets)"""
    loc = lv.Localizer(lv.default_params(max_points=1 << 14, max_map_points=1 << 12))
    pk = OC.table_packets()
    raw = np.frombuffer(pk.tobytes(), np.uint8)
    n = 16 * 16 * len(pk)
    b = Bufs(loc)
    d_msg = b.upload(raw)
    d_xyz, d_t, d_idx = b(12 * n), b(8 * n), b(4 * n)
    m = loc.process_ouster_device(d_msg, len(raw), len(pk), OC.table_calibration(lv), 1, 0.0, d_xyz, d_t, None, None, d_idx)
    assert m == n
    c, s = OC.tables_from_points(loc.download(d_xyz, np.empty((n, 3), f32)), loc.download(d_idx, np.empty(n, np.int32)))
    want_c, want_s = OC.table()
    assert bits(c) == bits(want_c) and bits(s) == bits(want_s)
    assert loc.async_status() == (lv.OK, "")
    b.free()
    loc.close()


def test_refusals_leave_the_handle_untouched(lv):
    loc = lv.Localizer(lv.default_params(max_points=1 << 14, max_map_points=1 << 12))
    rng = np.random.default_rng(12)
    cal = OC.calibration(lv, 1024, 16)
    pk = OC.packets(rng, 10, 1024, 16)
    raw = np.frombuffer(pk.tobytes(), np.uint8)
    b = Bufs(loc)
    d_msg = b.upload(raw)
    outs = [b(k * 2560) for k in (12, 8, 4, 4, 4)]
    d_n = b(8)
    ref = OC.process(pk, cal, 4, 3.0)
    nan, wide = OC.calibration(lv, 1024, 16), OC.calibration(lv, 1024, 16)
    nan.beam_azimuth_angles[3] = float("nan")
    wide.columns_per_frame = 4096
    L = loc.L
    loc.profile()
    m = C.c_int64(-1)
    for kw in (dict(k=11), dict(cal=nan), dict(cal=wide), dict(out0=d_msg + 100), dict(k=-1)):
        k, c = kw.get("k", 10), kw.get("cal", cal)
        o = [kw.get("out0", outs[0])] + outs[1:]
        assert L.lv_process_ouster_device(loc.h, d_msg, len(raw), k, C.byref(c), 4, 3.0, *o, C.byref(m)) == lv.ERR_ARG, kw
        assert m.value == 0
        put_count(loc, d_n, 123)
        assert L.lv_process_ouster_device_async(loc.h, d_msg, len(raw), k, C.byref(c), 4, 3.0, *o, d_n) == lv.ERR_ARG, kw
        assert get_count(loc, d_n) == 123                               # the count was not written
    assert loc.profile()["total_launches"] == 0
    assert loc.process_ouster_device(d_msg, len(raw), 10, cal, 4, 3.0, *outs) == len(ref[0])
    got = tuple(loc.download(d, np.empty_like(a)) for d, a in zip(outs, ref))
    same(got, ref, "after the refusals")
    assert loc.async_status() == (lv.OK, "")
    b.free()
    loc.close()


# ---- the async count into the LiDAR buffer with lanes ------------------------------------------------------------------------------
def test_async_count_feeds_the_full_buffer(lv, loc):
    rng = np.random.default_rng(9)
    cal = OC.calibration(lv, 1024, 32, OC.ORIGIN_MM, rng)
    dev, ref = FullBuffer(loc, 1 << 17, 1 << 17), FullBuffer(loc, 1 << 17, 1 << 17)   # one ring per handle: ref is replayed after dev
    b = Bufs(loc)
    d_msg = b(OC.packet_bytes(32) * 64 + 8)
    msgs = []
    for i in range(5):
        k = int(rng.integers(20, 64))
        msgs.append((OC.packets(rng, k, 1024, 32, m0=16 * int(rng.integers(0, 64)), ts0=20 * 10**9 + i * 100_000_000), 1 + i % 4))
    windows = [(20.0, 20.05), (20.1, 20.25), (-np.inf, np.inf), (20.2, 20.2 + 1e-6), (20.3, 20.6)]
    for pk, rate in msgs:
        raw = np.frombuffer(pk.tobytes(), np.uint8)
        upload(loc, d_msg + 1, raw)
        put_count(loc, dev.d_n, -1)
        loc.process_ouster_device_async(d_msg + 1, len(raw), len(pk), cal, rate, MD, dev.d_in[0], dev.d_in[1], dev.d_n, dev.d_in[2],
                                        dev.d_in[3])
        loc.lidar_push_full_async(*dev.d_in, dev.d_n, 16 * 32 * len(pk))
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


# ---- synthetic OS1-64 frames through the windowed device tick --------------------------------------------------------------------------
OS1_W, OS1_H = 1024, 64


def os1_frames(lv, sc, cal, n_msgs=6, cut=3, stamp0=10 * 10**9):
    """10 Hz frames of the synthetic world, 64 LEGACY packets each: each slot's return is the world point nearest to the slot's beam
    (column angle plus the beam's azimuth, clockwise from +x; the beam's altitude), its range in mm; message `cut` keeps one packet
    (a gated window)"""
    world = sc.world
    rng = np.random.default_rng(52)
    alt = np.array(cal.beam_altitude_angles[:OS1_H])
    az = np.array(cal.beam_azimuth_angles[:OS1_H])
    msgs = []
    for i in range(n_msgs):
        sw = world.sweep(world.pose(8.0 + 0.1 * i, sc.prm), rings=64, azimuths=2048, elev=(-17.0, 17.0), seed=500 + i).astype(np.float64)
        r = np.linalg.norm(sw, axis=1)
        ang = np.stack([np.mod(np.degrees(np.arctan2(-sw[:, 1], sw[:, 0])), 360.0), np.degrees(np.arcsin(sw[:, 2] / r))], 1)
        tree = cKDTree(ang)
        pk = OC.packets(rng, OS1_W // 16, OS1_W, OS1_H, m0=0, ts0=stamp0 + i * 100_000_000, invalid=0.0, bad_m=0.0, zero=0.0)
        col = pk.reshape(-1)
        slot = np.arange(OS1_W * OS1_H)
        g, p = slot // OS1_H, slot % OS1_H
        beam_az = np.mod(360.0 * col["m"][g] / OS1_W + az[p], 360.0)
        dist, j = tree.query(np.stack([beam_az, alt[p]], 1))
        mm = np.where((dist < 0.3) & (r[j] < 120.0), np.round(r[j] * 1000.0), 0).astype(np.uint32)
        col["px"]["range"] = (mm | (col["px"]["range"].reshape(-1) & ~np.uint32(OC.RANGE_MASK))).reshape(-1, OS1_H)
        if i == cut:
            pk = pk[:1]
        msgs.append(dict(pk=pk, raw=np.frombuffer(pk.tobytes(), np.uint8).copy(), n=16 * OS1_H * len(pk), n_packets=len(pk)))
    return msgs


class OusterChain(FullChain):
    """FullChain with Ouster LEGACY packets: on the device lv_process_ouster_device_async -> lv_lidar_push_full_device_async; otherwise
    the host decode (lv_ouster_to_points, the decimator on the rank, lv_time_sort_indices) pushed onto the restated deque.  Both chains
    propagate on IMU samples that went through encoded IMU packets and lv_ouster_imu_packet"""

    def __init__(self, lv, sc, cal, msgs, delta, device):
        super().__init__(lv, sc, "ouster", msgs, delta, device)
        self.cal, self.imu_stamps = cal, []
        propagate = self.loc.propagate_device

        def propagate_from_packets(acc, gyro, dt):
            t0 = int(round(self.t2 * 1e9))
            a, w = np.empty_like(acc), np.empty_like(gyro)
            for k in range(len(acc)):
                pkt = OC.imu_packet(t0 + k, np.asarray(acc[k]) / 9.80665, np.degrees(gyro[k]))
                s = lv.ouster_imu_packet(pkt)
                self.imu_stamps.append((s.stamp_sec, s.stamp_nsec))
                a[k], w[k] = s.linear_acceleration[:], s.angular_velocity[:]
            return propagate(a, w, dt)
        self.loc.propagate_device = propagate_from_packets

    def receive(self, g):
        if not self.device:
            xyz, t, inten, rg, _ = self.lv.ouster_to_points(g["raw"], self.cal)
            keep = F.temporal(xyz, RATE, MD)
            order = keep[self.lv.time_sort_indices(t[keep])]
            self.ref.push_message(xyz[order], t[order], inten[order], rg[order])
            return t[order]
        upload(self.loc, self.d_msg, g["raw"])
        self.loc.process_ouster_device_async(self.d_msg, len(g["raw"]), g["n_packets"], self.cal, RATE, MD, self.d_p[0], self.d_p[1],
                                             self.d_k, self.d_p[2], self.d_p[3])
        self.loc.lidar_push_full_async(*self.d_p, self.d_k, g["n"])
        return None


def test_os1_stream_through_the_device_tick_equals_the_host_chain(lv, scene_xaloc):
    sc = scene_xaloc
    rng = np.random.default_rng(53)
    cal = OC.calibration(lv, OS1_W, OS1_H, OC.ORIGIN_MM, rng)
    msgs = os1_frames(lv, sc, cal)
    host, dev = OusterChain(lv, sc, cal, msgs, 0.02, False), OusterChain(lv, sc, cal, msgs, 0.02, True)
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
    assert host.imu_stamps == dev.imu_stamps and len(dev.imu_stamps) == 4 * (seen["ticks"])
    host.close()
    dev.close()
