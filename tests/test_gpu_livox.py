"""lv_process_livox_device(_async) — Accumulator::process on a Livox CustomMsg's records in HBM — against the host chain, bit for bit:
lv_livox_to_points (tag filter), lv_temporal_downsample on its output (the rank among the tag-kept points), lv_time_sort_indices, then
the gathers.  Then the async count into the LiDAR buffer with lanes, a stream of rosette-ordered messages of the synthetic world through
the windowed device tick against the host decode plus push, and the refusals before any device work."""
import ctypes as C

import numpy as np
import pytest
from scipy.spatial import cKDTree

import livox_cases as LC
from test_gpu_async_tick import Bufs, get_count, put_count
from test_gpu_full_points import FullBuffer, FullChain, same_full
from test_gpu_lidar_buffer import MD, RATE, bits
from test_gpu_world_clouds import upload

pytestmark = pytest.mark.gpu
f32 = np.float32
TB = 1_712_345_678 * 10**9 + 999_999_500                          # the ns -> s carry inside the message


@pytest.fixture(scope="module")
def loc(lv):
    h = lv.Localizer(lv.default_params(max_points=1 << 18, max_map_points=1 << 16))
    yield h
    h.close()


def host_chain(lv, loc, recs, tb, mask, rate, md):
    """lv_livox_to_points -> lv_temporal_downsample (device, on the kept list) -> lv_time_sort_indices"""
    xyz, t, inten, rg, idx = lv.livox_to_points(recs, tb, mask)
    _, keep = loc.temporal_downsample(xyz, rate, md) if len(xyz) else (None, np.zeros(0, np.int32))
    order = keep[lv.time_sort_indices(t[keep])] if len(keep) else keep
    return xyz[order], t[order], inten[order], rg[order], idx[order]


def same(got, ref, what):
    for name, a, b in zip(("xyz", "time", "intensity", "range", "idx"), got, ref):
        assert a.shape == b.shape and bits(a) == bits(b), (what, name, a.shape, b.shape)


def device_run(loc, d_msg, shift, recs, tb, mask, rate, md, outs, d_n=None):
    """the records at d_msg + shift; the synchronous form, or the async one with its count at d_n"""
    raw = np.frombuffer(recs.tobytes(), np.uint8)
    n = len(recs)
    if len(raw):
        upload(loc, d_msg + shift, raw)
    if d_n is None:
        m = loc.process_livox_device(d_msg + shift, len(raw), n, tb, mask, rate, md, *outs)
    else:
        put_count(loc, d_n, -5)
        loc.process_livox_device_async(d_msg + shift, len(raw), n, tb, mask, rate, md, outs[0], outs[1], d_n, *outs[2:])
        m = get_count(loc, d_n)
    host = (np.empty((m, 3), f32), np.empty(m), np.empty(m, f32), np.empty(m, f32), np.empty(m, np.int32))
    return tuple(loc.download(d, a) for d, a in zip(outs, host))


# ---- every size x rate x mask, both forms, at odd addresses ------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 7, 240_000])
def test_process_livox_equals_the_host_chain(lv, loc, n):
    rng = np.random.default_rng(100 + n)
    recs = LC.records(rng, n)
    if n > 7:
        near = rng.choice(n, n // 10, replace=False)
        for k in "xyz":
            recs[k][near] *= f32(0.02)                                # inside min_dist
        recs["offset_time"][rng.choice(n, n // 4, replace=False)] = 777   # equal times
    b = Bufs(loc)
    d_msg = b(19 * n + 16)
    outs = [b(k * max(n, 1)) for k in (12, 8, 4, 4, 4)]
    d_n = b(8)
    seen = 0
    for mask in LC.MASKS:
        for rate in range(1, 9):
            md = 3.0 if rate % 2 else 0.0
            ref = host_chain(lv, loc, recs, TB, mask, rate, md)
            same(ref, LC.process(recs, TB, mask, rate, md), ("restatement", n, mask, rate))
            for shift, asyn in ((1, False), (3, True)):
                got = device_run(loc, d_msg, shift, recs, TB, mask, rate, md, outs, d_n if asyn else None)
                same(got, ref, (n, mask, rate, shift, asyn))
            seen += len(ref[0]) > 0
    assert loc.async_status() == (lv.OK, "")
    if n > 7:
        assert seen == 32
    b.free()


def test_edge_records_and_launches(lv):
    loc = lv.Localizer(lv.default_params(max_points=1 << 14, max_map_points=1 << 12))
    rng = np.random.default_rng(3)
    b = Bufs(loc)
    d_msg = b(19 * 2000)
    outs = [b(k * 2000) for k in (12, 8, 4, 4, 4)]
    d_n = b(8)
    for name, (recs, tb) in LC.edge_records(rng).items():
        for mask in LC.MASKS + [0x10, 0x30]:
            for rate, md in ((1, 0.0), (3, 3.0), (8, 3.0)):
                ref = LC.process(recs, tb, mask, rate, md)
                same(host_chain(lv, loc, recs, tb, mask, rate, md), ref, (name, mask, rate))
                same(device_run(loc, d_msg, 1, recs, tb, mask, rate, md, outs), ref, (name, mask, rate))
                same(device_run(loc, d_msg, 2, recs, tb, mask, rate, md, outs, d_n), ref, (name, mask, rate, "async"))
    loc.profile()                                                     # reset the counters
    recs = LC.records(rng, 1000)
    device_run(loc, d_msg, 0, recs, TB, 0x20, 4, 3.0, outs)
    assert loc.profile()["total_launches"] == 9
    assert loc.async_status() == (lv.OK, "")
    b.free()
    loc.close()


# ---- the async count into the LiDAR buffer with lanes ------------------------------------------------------------------------------
def test_async_count_feeds_the_full_buffer(lv, loc):
    rng = np.random.default_rng(9)
    dev, ref = FullBuffer(loc, 1 << 15, 1 << 15), FullBuffer(loc, 1 << 15, 1 << 15)   # one ring per handle: ref is replayed after dev
    b = Bufs(loc)
    d_msg = b(19 * 4000 + 8)
    msgs = []
    for i in range(6):
        n = int(rng.integers(1000, 4000))
        recs = LC.records(rng, n, t_span=100_000_000)
        msgs.append((recs, 20 * 10**9 + i * 100_000_000, [0, 0x20, 0x0F][i % 3], 1 + i % 4))
    windows = [(20.0, 20.15), (20.1, 20.35), (-np.inf, np.inf), (20.25, 20.25 + 1e-9), (20.3, 20.6)]
    got = []
    for recs, tb, mask, rate in msgs:
        raw = np.frombuffer(recs.tobytes(), np.uint8)
        upload(loc, d_msg + 1, raw)
        put_count(loc, dev.d_n, -1)
        loc.process_livox_device_async(d_msg + 1, len(raw), len(recs), tb, mask, rate, MD, dev.d_in[0], dev.d_in[1], dev.d_n, dev.d_in[2],
                                       dev.d_in[3])
        loc.lidar_push_full_async(*dev.d_in, dev.d_n, len(recs))
    got = [dev.get(t1, t2) for t1, t2 in windows]
    loc.lidar_clear_async(np.inf)
    loc.lidar_reserve_full(1 << 15)
    for recs, tb, mask, rate in msgs:                                  # the host-decoded points, pushed
        xyz, t, inten, rg, _ = host_chain(lv, loc, recs, tb, mask, rate, MD)
        ref.push(xyz, t, inten, rg)
    for (t1, t2), g in zip(windows, got):
        same_full(g, ref.get(t1, t2), (t1, t2))
    assert sum(len(g[1]) for g in got) > 5000
    assert loc.async_status() == (lv.OK, "")
    loc.lidar_clear_async(np.inf)
    dev.close()
    ref.close()
    b.free()


# ---- rosette-ordered messages through the windowed device tick -------------------------------------------------------------------------
def rosette_messages(lv, sc, n_msgs=6, cut=3):
    """10 Hz messages of the synthetic world inside a 70-degree cone around x: each point gets the time of the nearest sample of a
    rosette (r = sin(w1 t), angle w2 t) over 0.1 s, and the message is in firing (time) order, as a Livox driver publishes it.  Most
    tags are 0, some mark second returns (0x10) or third (0x20) and noise (0x01); message `cut` keeps 300 points (a gated window)"""
    rng = np.random.default_rng(41)
    ts = np.linspace(0.0, 0.1, 40_000, endpoint=False)
    half = np.deg2rad(35.0)
    curve = np.stack([half * np.sin(2 * np.pi * 180 * ts) * np.cos(2 * np.pi * 23 * ts),
                      half * np.sin(2 * np.pi * 180 * ts) * np.sin(2 * np.pi * 23 * ts)], 1)
    tree = cKDTree(curve)
    msgs = []
    for i in range(n_msgs):
        sw = sc.world.sweep(sc.world.pose(8.0 + 0.1 * i, sc.prm), rings=64, azimuths=2048, elev=(-35.0, 35.0), seed=300 + i)
        d = sw / np.linalg.norm(sw, axis=1, keepdims=True)
        ang = np.stack([np.arctan2(d[:, 1], d[:, 0]), np.arcsin(np.clip(d[:, 2], -1, 1))], 1)
        inside = (d[:, 0] > 0) & (np.hypot(ang[:, 0], ang[:, 1]) < half)
        pts, ang = sw[inside], ang[inside]
        _, k = tree.query(ang)
        off = (ts[k] * 1e9).astype(np.uint32)
        order = np.argsort(off, kind="stable")
        recs = np.zeros(len(order), LC.RECORD)
        recs["x"], recs["y"], recs["z"] = pts[order, 0], pts[order, 1], pts[order, 2]
        recs["offset_time"] = off[order]
        recs["reflectivity"] = rng.integers(0, 256, len(order))
        recs["tag"] = rng.choice([0x00, 0x10, 0x20, 0x01], len(order), p=[0.8, 0.1, 0.05, 0.05])
        recs["line"] = rng.integers(0, 6, len(order))
        if i == cut:
            recs = recs[:300]
        raw = np.frombuffer(recs.tobytes(), np.uint8).copy()
        msgs.append(dict(recs=recs, raw=raw, n=len(recs), tb=10 * 10**9 + i * 100_000_000))
    return msgs


class LivoxChain(FullChain):
    """FullChain with Livox messages: on the device lv_process_livox_device_async -> lv_lidar_push_full_device_async; otherwise the host
    decode (lv_livox_to_points, the decimator on the rank, lv_time_sort_indices) pushed onto the restated deque"""
    MASK = 0x20

    def receive(self, g):
        if not self.device:
            import frontend_ref as F
            xyz, t, inten, rg, _ = self.lv.livox_to_points(g["recs"], g["tb"], self.MASK)
            keep = F.temporal(xyz, RATE, MD)
            order = keep[self.lv.time_sort_indices(t[keep])]
            self.ref.push_message(xyz[order], t[order], inten[order], rg[order])
            return t[order]
        upload(self.loc, self.d_msg, g["raw"])
        self.loc.process_livox_device_async(self.d_msg, len(g["raw"]), g["n"], g["tb"], self.MASK, RATE, MD, self.d_p[0], self.d_p[1], self.d_k,
                                            self.d_p[2], self.d_p[3])
        self.loc.lidar_push_full_async(*self.d_p, self.d_k, g["n"])
        return None


def test_rosette_stream_through_the_device_tick_equals_the_host_chain(lv, scene_xaloc):
    sc = scene_xaloc
    msgs = rosette_messages(lv, sc)
    assert min(g["n"] for g in msgs if g["n"] > 300) > 10000
    host, dev = LivoxChain(lv, sc, "livox", msgs, 0.02, False), LivoxChain(lv, sc, "livox", msgs, 0.02, True)
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


# ---- refusals before any device work -------------------------------------------------------------------------------------------------
def test_refusals_leave_the_handle_untouched(lv):
    loc = lv.Localizer(lv.default_params(max_points=1 << 14, max_map_points=1 << 12))
    rng = np.random.default_rng(12)
    recs = LC.records(rng, 1000)
    raw = np.frombuffer(recs.tobytes(), np.uint8)
    b = Bufs(loc)
    d_msg = b.upload(raw)
    outs = [b(k * 1000) for k in (12, 8, 4, 4, 4)]
    d_n = b(8)
    ref = LC.process(recs, TB, 0x20, 4, 3.0)
    L = loc.L
    loc.profile()
    m = C.c_int64(-1)
    for kw in (dict(n=1001), dict(tb=LC.TIMEBASE_MAX + 1), dict(out0=d_msg + 100), dict(n=-1)):
        n, tb = kw.get("n", 1000), kw.get("tb", TB)
        o = [kw.get("out0", outs[0])] + outs[1:]
        assert L.lv_process_livox_device(loc.h, d_msg, len(raw), n, tb, 0x20, 4, 3.0, *o, C.byref(m)) == lv.ERR_ARG, kw
        assert m.value == 0
        put_count(loc, d_n, 123)
        assert L.lv_process_livox_device_async(loc.h, d_msg, len(raw), n, tb, 0x20, 4, 3.0, *o, d_n) == lv.ERR_ARG, kw
        assert get_count(loc, d_n) == 123                               # the count was not written
    assert loc.profile()["total_launches"] == 0
    assert loc.process_livox_device(d_msg, len(raw), 1000, TB, 0x20, 4, 3.0, *outs) == len(ref[0])
    got = tuple(loc.download(d, np.empty_like(a)) for d, a in zip(outs, ref))
    same(got, ref, "after the refusals")
    assert loc.async_status() == (lv.OK, "")
    b.free()
    loc.close()
