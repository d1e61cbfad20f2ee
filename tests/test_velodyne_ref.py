"""The Velodyne packet front end without a GPU.

lv_velodyne_to_points (the host build of lv_wire.h's decoder) then the decimator on the rank and lv_time_sort_indices equal the NumPy
restatement of tests/velodyne_cases.py bit for bit, for the nominal VLP-16 and Puck Hi-Res calibrations and a factory-like one, every
rate 1-8 and several min_dist values.  The library's rotation tables, read back through the host decoder, are float64 cos / sin
rounded, entry for entry.  lv_bag_parse_velodyne_scan reads packets at every address mod 4 and refuses truncations and trailing bytes.
Every argument refusal of lv_process_velodyne_device(_async) happens before any device call (the device pointers below are never
dereferenced).  An independent geometric check encodes points placed in the ROS frame into packets by the manual's definitions of
range, elevation, azimuth and firing time, and decodes them back."""
import ctypes as C
import math

import numpy as np
import pytest

import bagwriter as W
import frontend_ref as F
import velodyne_cases as VC
from test_bag_reader import BagMessage

BASE = 1 << 40                       # a device address that is never touched
f32 = np.float32


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64 if a.dtype.itemsize == 8 else np.uint32).tobytes()


def same(got, ref, what):
    assert len(got) == len(ref) == 5, what
    for name, a, b in zip(("xyz", "time", "intensity", "range", "idx"), got, ref):
        assert a.shape == b.shape and bits(a) == bits(b), (what, name)


def host_chain(lv, pk, cal, rate, md):
    """lv_velodyne_to_points -> the decimator on the rank (frontend_ref.temporal) -> lv_time_sort_indices"""
    xyz, t, inten, rg, idx = lv.velodyne_to_points(pk.tobytes(), cal)
    keep = F.temporal(xyz, rate, md)
    order = keep[lv.time_sort_indices(t[keep])] if len(keep) else keep
    return xyz[order], t[order], inten[order], rg[order], idx[order]


# ---- the tables and the calibrations ----------------------------------------------------------------------------------------------
def test_rotation_tables_are_float64_rounded(lv):
    assert f32(500) * f32(0.002) == 1                                   # d of table_packets
    pk = VC.table_packets()
    xyz, _, _, _, idx = lv.velodyne_to_points(pk.tobytes(), lv.VelodyneCalibration())
    c, s = VC.tables_from_points(xyz, idx)
    want_c = np.array([f32(math.cos(q * 0.01 * math.pi / 180.0)) for q in range(36000)], f32)
    want_s = np.array([f32(math.sin(q * 0.01 * math.pi / 180.0)) for q in range(36000)], f32)
    assert bits(c) == bits(want_c) and bits(s) == bits(want_s)
    assert bits(c) == bits(VC.tables()[0]) and bits(s) == bits(VC.tables()[1])
    assert c[0] == 1 and s[0] == 0 and c[9000] == f32(math.cos(math.pi / 2)) and s[9000] == 1


def test_default_calibrations(lv):
    for model, deg in (("vlp16", VC.VLP16_DEG), ("puck_hires", VC.HIRES_DEG)):
        cal = lv.velodyne_calibration(model)
        assert list(cal.vert_correction) == [d * math.pi / 180.0 for d in deg]
        for name in ("rot_correction", "dist_correction", "vert_offset_correction", "horiz_offset_correction"):
            assert list(getattr(cal, name)) == [0.0] * 16, (model, name)
    L = lv.lib()
    cal = lv.VelodyneCalibration()
    assert L.lv_velodyne_default_calibration(2, C.byref(cal)) == lv.ERR_ARG
    assert L.lv_velodyne_default_calibration(0, None) == lv.ERR_ARG


# ---- the host decoder against the restatement ------------------------------------------------------------------------------------
def cases(lv, rng):
    pk = VC.packets(rng, 76)
    out = [(name, p, VC.calibration(lv)) for name, p in VC.edge_packets(rng).items()]
    out += [("rotation", pk, VC.calibration(lv)), ("rotation_hires", pk, VC.calibration(lv, "puck_hires")),
            ("rotation_factory", pk, VC.random_calibration(lv, rng))]
    return out


def test_velodyne_to_points_equals_the_restatement(lv):
    rng = np.random.default_rng(11)
    seen = 0
    for name, pk, cal in cases(lv, rng):
        ref = VC.to_points(pk, cal)
        same(lv.velodyne_to_points(pk.tobytes(), cal), ref, name)
        seen += len(ref[0])
        for rate in range(1, 9):
            for md in (0.0, 0.9, 3.0):
                same(host_chain(lv, pk, cal, rate, md), VC.process(pk, cal, rate, md), (name, rate, md))
    assert seen > 30000


def test_msg2points_rule(lv):
    rng = np.random.default_rng(12)
    cal = VC.calibration(lv)
    p = VC.edge_packets(rng)["bad_flags"]
    idx = lv.velodyne_to_points(p.tobytes(), cal)[4]
    k, b = idx // 384, (idx % 384) // 32
    assert not ((k == 1) & (b >= 7)).any() and ((k == 1) & (b == 6)).any()
    assert not (k == 3).any() and not ((k == 4) & (b == 11)).any() and ((k == 4) & (b == 10)).any()
    p = VC.dual_packets(rng)
    idx = lv.velodyne_to_points(p.tobytes(), cal)[4]
    assert not (idx // 384 == 2).any() and (idx // 384 == 3).any()              # a dual-return packet contributes no points
    raw = p["data"]["blocks"]["ch"]["dist"].reshape(len(p), 384).ravel()
    assert set(idx.tolist()) == set(np.nonzero((raw != 0) & (np.arange(len(raw)) // 384 != 2))[0].tolist())


def test_velodyne_time_rule(lv):
    rng = np.random.default_rng(13)
    cal = VC.calibration(lv)
    p = VC.packets(rng, 2, sec=1_700_000_000, nsec=999_999_999 - 24 * 55296 + 1, zero=0.0)
    _, t, _, _, idx = lv.velodyne_to_points(p.tobytes(), cal)
    r = idx % 384
    total = [int(p["sec"][i // 384]) * 10**9 + int(p["nsec"][i // 384]) + (2 * (s // 32) + (s % 32) // 16) * 55296 + (s % 16) * 2304
             for i, s in zip(idx.tolist(), r.tolist())]
    assert t.tolist() == [float(np.float64(v // 10**9) + np.float64(v % 10**9) * 1e-9) for v in total]
    assert t[0] == 1_700_000_000.0 + np.float64(999_999_999 - 24 * 55296 + 1) * 1e-9
    assert (np.diff(t) > 0).all()
    p = VC.packets(rng, 1, sec=2**32 - 1, nsec=999_999_999 - 24 * 55296, zero=0.0)   # the largest stamp: no wrap
    _, t, *_ = lv.velodyne_to_points(p.tobytes(), cal)
    assert t[-1] == np.float64(2**32 - 1) + np.float64(999_999_999 - 24 * 55296 + 23 * 55296 + 15 * 2304) * 1e-9


# ---- an independent geometric check ------------------------------------------------------------------------------------------------
def test_decoded_positions_and_times_match_the_manual(lv):
    """points placed in the ROS frame (x forward, y left, z up), encoded by the manual: range |p| in 2 mm units, the laser whose
    elevation asin(z / |p|) is the point's, azimuth clockwise from +x seen from above; the sensor turns D = 0.48 deg per block, laser l
    of firing f fires (l 2.304 + f 55.296) us into its block, which is 110.592 us long, so it points D (l 2.304 + f 55.296) / 110.592 =
    (l + 24 f) 0.01 deg past the block's azimuth"""
    rng = np.random.default_rng(14)
    for az0 in (35_500, 9000 - 3 * 48, 27000 - 5 * 48):                # across the wrap, through 90 and 270 deg
        quarter = manual_round_trip(lv, rng, az0)
        assert quarter[9000 if az0 < 20000 else 27000] if az0 != 35_500 else True


def manual_round_trip(lv, rng, az0):
    cal = VC.calibration(lv)
    n = 3
    pk = VC.packets(rng, n, az0=az0, step=48, sec=100, nsec=5_000, zero=0.0)
    slot = np.arange(384 * n)
    k, r = slot // 384, slot % 384
    b, f, l = r // 32, (r % 32) // 16, r % 16
    az = (pk["data"]["blocks"]["azimuth"][k, b].astype(np.int64) + l + 24 * f) % 36000
    alpha = np.deg2rad(az * 0.01)
    elev = np.deg2rad(np.array(VC.VLP16_DEG, np.float64))[l]
    d = rng.uniform(0.5, 110.0, len(slot))
    p = d[:, None] * np.stack([np.cos(elev) * np.cos(alpha), -np.cos(elev) * np.sin(alpha), np.sin(elev)], 1)
    # encode each point from its position
    rng_ = np.linalg.norm(p, axis=1)
    assert np.allclose(np.arcsin(p[:, 2] / rng_), elev, atol=1e-12)
    assert np.allclose(np.mod(np.degrees(np.arctan2(-p[:, 1], p[:, 0])) * 100, 36000), az, atol=1e-6)
    raw = np.round(rng_ / 0.002).astype(np.uint16)
    pk["data"]["blocks"]["ch"]["dist"] = raw.reshape(n, 12, 32)
    xyz, t, inten, rg, idx = lv.velodyne_to_points(pk.tobytes(), cal)
    assert (idx == slot).all()
    tol = 0.001 + 64 * 2.0**-24 * rng_                                  # half a distance step + the fp32 chain
    err = np.linalg.norm(xyz.astype(np.float64) - p, axis=1)
    assert (err <= tol).all(), err.max()
    assert (np.abs(rg - rng_) <= tol).all()
    # the quarter turns: azimuth 90 deg is to the right (-y), 270 deg to the left
    quarter = {}
    for q, sign in ((9000, -1), (27000, 1)):
        hit = az == q
        quarter[q] = bool(hit.any())
        assert (np.sign(xyz[hit, 1]) == sign).all() and (np.abs(xyz[hit, 0]) < 1e-4).all()
    # firing times: (2b + f) 55.296 us + l 2.304 us after the packet stamp
    stamp = pk["sec"][k].astype(np.float64) + pk["nsec"][k] * 1e-9
    assert np.allclose(t - stamp, (2 * b + f) * 55.296e-6 + l * 2.304e-6, rtol=0, atol=1e-12)
    assert np.allclose(np.diff(stamp[::384]), 24 * 55.296e-6, rtol=0, atol=1e-12)
    return quarter


# ---- the host decoder's refusals ------------------------------------------------------------------------------------------------
def test_velodyne_to_points_refusals(lv):
    L = lv.lib()
    cal = VC.calibration(lv)
    pk = VC.packets(np.random.default_rng(15), 3)
    raw = np.frombuffer(pk.tobytes(), np.uint8)
    n = 384 * 3
    out = [np.empty(3 * n, np.float32), np.empty(n), np.empty(n, np.float32), np.empty(n, np.float32), np.empty(n, np.int32)]
    ptr = [a.ctypes.data_as(C.c_void_p) for a in out]
    m = C.c_int64(7)

    def call(data=raw.ctypes.data_as(C.c_void_p), nb=len(raw), k=3, c=cal, outs=ptr, n_out=True):
        m.value = 7
        st = L.lv_velodyne_to_points(data, nb, k, C.byref(c) if c is not None else None, *outs, C.byref(m) if n_out else None)
        return st, m.value
    good = len(VC.to_points(pk, cal)[0])
    assert call() == (lv.OK, good)
    assert call(outs=ptr[:2] + [None] * 3) == (lv.OK, good)             # intensity, range and idx are optional
    assert call(k=0, nb=0) == (lv.OK, 0)
    bad_cal = VC.calibration(lv)
    bad_cal.horiz_offset_correction[5] = float("nan")
    inf_cal = VC.calibration(lv)
    inf_cal.vert_correction[0] = float("inf")
    for kw in (dict(data=None), dict(nb=len(raw) - 1), dict(k=-1), dict(k=VC.MAX_PACKETS + 1, nb=1 << 40), dict(c=None),
               dict(c=bad_cal), dict(c=inf_cal), dict(outs=[None] + ptr[1:]), dict(outs=ptr[:1] + [None] + ptr[2:])):
        assert call(**kw) == (lv.ERR_ARG, 0), kw
    assert call(n_out=False)[0] == lv.ERR_ARG
    for nsec in (1_000_000_000, 0xFFFFFFFF):                            # a stamp that cannot be converted
        bad = pk.copy()
        bad["nsec"][2] = nsec
        b = np.frombuffer(bad.tobytes(), np.uint8)
        assert call(data=b.ctypes.data_as(C.c_void_p)) == (lv.ERR_ARG, 0), nsec
    bad = pk.copy()
    bad["nsec"][2] = 999_999_999
    b = np.frombuffer(bad.tobytes(), np.uint8)
    assert call(data=b.ctypes.data_as(C.c_void_p))[0] == lv.OK


# ---- the bag reader ---------------------------------------------------------------------------------------------------------------
def read_bag(lv, path):
    L = lv.lib()
    L.lv_bag_next.argtypes = [C.c_void_p, C.POINTER(BagMessage)]
    L.lv_bag_close.argtypes = [C.c_void_p]
    bag = C.c_void_p()
    assert L.lv_bag_open(path.encode(), C.byref(bag)) == lv.OK
    out, m = [], BagMessage()
    while L.lv_bag_next(bag, C.byref(m)) == 1:
        v = lv.VelodyneView()
        st = L.lv_bag_parse_velodyne_scan(C.cast(m.data, C.c_void_p), m.size, C.byref(v)) \
            if m.type == b"velodyne_msgs/VelodyneScan" else None
        pk = np.frombuffer(C.string_at(v.packets, v.data_bytes), VC.PACKET).copy() if st == lv.OK and v.n_packets else None
        out.append((m.type.decode(), st, v, pk, (v.packets or 0) % 4))
    L.lv_bag_close(bag)
    return out


def test_bag_parse_velodyne_round_trip(lv, tmp_path):
    rng = np.random.default_rng(16)
    sets = [VC.packets(rng, n) for n in (76, 0, 1, 5)]
    frames = ["velodyne", "", "a", "abc"]
    conns = {0: ("/imu", "sensor_msgs/Imu"), 1: ("/velodyne_packets", "velodyne_msgs/VelodyneScan")}
    msgs = []
    for k, (pk, frame) in enumerate(zip(sets, frames)):
        msgs.append((0, 100, k, W.imu(100, k, (0, 0, 0, 1), (0.1, 0.2, 0.3), (0.0, 0.1, 9.8))))
        msgs.append((1, 100, 1000 + k, VC.scan_msg(pk, 100 + k, 7_000 * k, frame, k)))
    path = str(tmp_path / "velodyne.bag")
    W.write_bag(path, conns, msgs)
    got = read_bag(lv, path)
    assert [g[0] for g in got] == ["sensor_msgs/Imu", "velodyne_msgs/VelodyneScan"] * len(sets)
    for k, (g, pk) in enumerate(zip([g for g in got if g[1] is not None], sets)):
        _, st, v, got_pk, _ = g
        assert st == lv.OK and (v.stamp_sec, v.stamp_nsec, v.n_packets, v.data_bytes) == (100 + k, 7_000 * k, len(pk), 1214 * len(pk))
        if len(pk):
            assert got_pk.tobytes() == pk.tobytes()
    v, raw = lv.bag_parse_velodyne_scan(msgs[1][3])
    assert v.n_packets == 76 and raw.tobytes() == sets[0].tobytes()
    seen = set()
    for k in range(4):                                                 # frame_id lengths 0 .. 3: the packets at every address mod 4
        path = str(tmp_path / ("align%d.bag" % k))
        W.write_bag(path, {1: conns[1]}, [(1, 100, 0, VC.scan_msg(sets[3], 9, 9, "f" * k))])
        (_, st, v, got_pk, mod4), = read_bag(lv, path)
        assert st == lv.OK and got_pk.tobytes() == sets[3].tobytes()
        seen.add(mod4)
    assert seen == {0, 1, 2, 3}
    cal = VC.calibration(lv)                                           # the decoder reads packets at any address
    ref = VC.to_points(sets[3], cal)
    nb, n = sets[3].nbytes, 384 * len(sets[3])
    for shift in range(4):
        buf = np.zeros(nb + 8, np.uint8)
        buf[shift:shift + nb] = np.frombuffer(sets[3].tobytes(), np.uint8)
        out = (np.empty((n, 3), f32), np.empty(n), np.empty(n, f32), np.empty(n, f32), np.empty(n, np.int32))
        m = C.c_int64(0)
        assert lv.lib().lv_velodyne_to_points(buf.ctypes.data + shift, nb, len(sets[3]), C.byref(cal),
                                              *(a.ctypes.data for a in out), C.byref(m)) == lv.OK
        same(tuple(a[:m.value] for a in out), ref, shift)


def test_bag_parse_velodyne_refusals(lv):
    L = lv.lib()
    good = VC.scan_msg(VC.packets(np.random.default_rng(17), 3))
    v = lv.VelodyneView()
    assert L.lv_bag_parse_velodyne_scan(good, len(good), C.byref(v)) == lv.OK and v.n_packets == 3
    for cut in (1, 7, 1214, 1215, len(good) - 12):                      # truncated anywhere
        assert L.lv_bag_parse_velodyne_scan(good, len(good) - cut, C.byref(v)) == lv.ERR_ARG, cut
    assert L.lv_bag_parse_velodyne_scan(good + b"\x00", len(good) + 1, C.byref(v)) == lv.ERR_ARG
    empty = VC.scan_msg(VC.packets(np.random.default_rng(17), 0))
    assert L.lv_bag_parse_velodyne_scan(empty, len(empty), C.byref(v)) == lv.OK and v.n_packets == 0 and v.data_bytes == 0
    huge = good[:-(3 * 1214 + 4)] + (0xFFFFFFFF).to_bytes(4, "little") + good[-3 * 1214:]   # a count the bytes cannot hold
    assert L.lv_bag_parse_velodyne_scan(huge, len(huge), C.byref(v)) == lv.ERR_ARG
    assert L.lv_bag_parse_velodyne_scan(None, len(good), C.byref(v)) == lv.ERR_ARG
    assert L.lv_bag_parse_velodyne_scan(good, len(good), None) == lv.ERR_ARG


# ---- the device calls' argument checks (before any device work) --------------------------------------------------------------------
N = 10
NB = 1214 * N
NS = 384 * N


@pytest.fixture
def dcall(lv):
    L = lv.lib()
    good = lv.velodyne_calibration()

    def run(h=None, data=BASE, data_bytes=NB, k=N, cal=good, outs=None, n_out=True, asynch=False):
        outs = outs if outs is not None else [BASE + (1 << 30) + j * (1 << 24) for j in range(5)]
        c = C.byref(cal) if cal is not None else None
        if asynch:
            st = L.lv_process_velodyne_device_async(h, data, data_bytes, k, c, 4, 3.0, *outs, BASE + (1 << 35) if n_out else None)
        else:
            m = C.c_int64(7)
            st = L.lv_process_velodyne_device(h, data, data_bytes, k, c, 4, 3.0, *outs, C.byref(m) if n_out else None)
            if n_out:
                assert m.value == 0
        return st, L.lv_last_error()
    return run


@pytest.mark.parametrize("asynch", [False, True])
def test_process_velodyne_refusals_before_device_work(lv, dcall, asynch):
    handle = (lv.ERR_ARG, b"process velodyne: null handle")
    assert dcall(asynch=asynch) == handle
    for kw in (dict(data=None), dict(n_out=False), dict(cal=None)):
        st, msg = dcall(asynch=asynch, **kw)
        assert st == lv.ERR_ARG and b"null packets" in msg, kw
    for j in (0, 1):
        outs = [BASE + (1 << 30) + i * (1 << 24) for i in range(5)]
        outs[j] = None
        st, msg = dcall(asynch=asynch, outs=outs)
        assert st == lv.ERR_ARG and b"null packets" in msg, j
    outs = [BASE + (1 << 30) + i * (1 << 24) for i in range(5)]
    outs[2:] = [None] * 3
    assert dcall(asynch=asynch, outs=outs) == handle
    for k in (-1, VC.MAX_PACKETS + 1, 1 << 62):
        st, msg = dcall(asynch=asynch, k=k, data_bytes=1 << 45)
        assert st == lv.ERR_ARG and (b"n_packets" in msg or b"negative" in msg), k
    assert dcall(asynch=asynch, k=0, data_bytes=0) == handle
    st, msg = dcall(asynch=asynch, data_bytes=NB - 1)
    assert st == lv.ERR_ARG and b"too short" in msg
    for name in ("vert_correction", "rot_correction", "dist_correction", "vert_offset_correction", "horiz_offset_correction"):
        for v in (float("nan"), float("inf"), -float("inf")):
            cal = lv.velodyne_calibration()
            getattr(cal, name)[15] = v
            st, msg = dcall(asynch=asynch, cal=cal)
            assert st == lv.ERR_ARG and b"not finite" in msg, (name, v)
    for j, size in enumerate((12, 8, 4, 4, 4)):
        for start in (BASE + NB - 1, BASE - size * NS + 1, BASE):
            outs = [BASE + (1 << 30) + i * (1 << 24) for i in range(5)]
            outs[j] = start
            st, msg = dcall(asynch=asynch, outs=outs)
            assert st == lv.ERR_ARG and b"overlaps" in msg, (j, start)
        for start in (BASE + NB, BASE - size * NS):                     # adjacent ranges are fine
            outs = [BASE + (1 << 30) + i * (1 << 24) for i in range(5)]
            outs[j] = start
            assert dcall(asynch=asynch, outs=outs) == handle, (j, start)
