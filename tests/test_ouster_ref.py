"""The Ouster packet front end without a GPU.

lv_ouster_to_points (the host build of lv_wire.h's decoder) then the decimator on the rank and lv_time_sort_indices equal the NumPy
restatement of tests/ouster_cases.py bit for bit, for every H and W, n = 0 and 12.163 mm, every rate 1-8 and several min_dist values.
The library's column table, read back through the host decoder, is float64 cos / sin rounded, entry for entry.  An independent
geometric check places points in the LiDAR frame, encodes them by the definitions of range, beam altitude, beam azimuth and beam
origin, and decodes them back; the same frame written as an os_cloud_node PointCloud2 and read by the Ouster PointCloud2 path gives
the same points.  The IMU packet decode, the metadata JSON reader in both firmware layouts, bag parsing of a packet-only bag at every
alignment, and every argument refusal of lv_process_ouster_device(_async) before any device call (the device pointers below are
never dereferenced)."""
import ctypes as C
import json
import math
import struct

import numpy as np
import pytest

import bagwriter as W
import frontend_ref as F
import ouster_cases as OC
from test_bag_reader import OUSTER, BagMessage, CloudLayout

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
    """lv_ouster_to_points -> the decimator on the rank (frontend_ref.temporal) -> lv_time_sort_indices"""
    xyz, t, inten, rg, idx = lv.ouster_to_points(pk.tobytes(), cal)
    keep = F.temporal(xyz, rate, md)
    order = keep[lv.time_sort_indices(t[keep])] if len(keep) else keep
    return xyz[order], t[order], inten[order], rg[order], idx[order]


# ---- the host decoder against the restatement ------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", OC.HS)
def test_ouster_to_points_equals_the_restatement(lv, H):
    rng = np.random.default_rng(20 + H)
    seen = 0
    for Wc in OC.WS:
        for n in (0.0, OC.ORIGIN_MM):
            cal = OC.calibration(lv, Wc, H, n, rng)
            pk = OC.packets(rng, 6, Wc, H, m0=Wc - 40)                 # across the frame wrap
            ref = OC.to_points(pk, cal)
            same(lv.ouster_to_points(pk.tobytes(), cal), ref, (Wc, n))
            seen += len(ref[0])
            for rate in range(1, 9):
                for md in (0.0, 0.9, 3.0):
                    same(host_chain(lv, pk, cal, rate, md), OC.process(pk, cal, rate, md), (Wc, n, rate, md))
    assert seen > 6 * 16 * H * 6 * 0.8


def test_msg2points_rule(lv):
    rng = np.random.default_rng(21)
    cal = OC.calibration(lv, 1024, 32)
    pk = OC.packets(rng, 8, 1024, 32, invalid=0.2, bad_m=0.2, zero=0.3)
    col = pk.reshape(-1)
    idx = lv.ouster_to_points(pk.tobytes(), cal)[4]
    word = col["px"]["range"].reshape(-1)
    g = np.arange(len(word)) // 32
    want = ((col["status"][g] & 1) == 1) & (col["m"][g] < 1024) & ((word & 0xFFFFF) != 0)
    assert set(idx.tolist()) == set(np.nonzero(want)[0].tolist())
    assert (col["status"] == 0).any() and (col["status"] == 0xFFFFFFFE).any() and (col["m"] >= 1024).any()
    assert ((word & 0xFFFFF) == 0).any() and ((word >> 20) != 0).any()                # no return, and garbage in the upper bits
    col["status"] = 1                                                  # only bit 0 is read
    col["m"] = col["m"] % 1024
    word &= 0xFFFFF
    assert len(lv.ouster_to_points(pk.tobytes(), cal)[0]) == int((word != 0).sum())


def test_ouster_time_rule(lv):
    rng = np.random.default_rng(22)
    cal = OC.calibration(lv, 512, 16)
    for ts0 in (1_700_000_000 * 10**9 + 999_990_000, 0, 2**64 - 16 * 5 * OC.column_ns(512) - 1):
        pk = OC.packets(rng, 5, 512, 16, ts0=ts0, invalid=0, bad_m=0, zero=0)
        _, t, _, _, idx = lv.ouster_to_points(pk.tobytes(), cal)
        ts = [ts0 + (i // 16) * OC.column_ns(512) for i in idx.tolist()]
        assert t.tolist() == [float(np.float64(v // 10**9) + np.float64(v % 10**9) * 1e-9) for v in ts], ts0
        assert (np.diff(t) >= 0).all()


# ---- the column table ----------------------------------------------------------------------------------------------------------------
def test_column_table_is_float64_rounded(lv):
    assert f32(1000) * f32(0.001) == 1                                 # d of table_packets
    pk = OC.table_packets()
    xyz, _, _, _, idx = lv.ouster_to_points(pk.tobytes(), OC.table_calibration(lv))
    c, s = OC.tables_from_points(xyz, idx)
    want_c = np.array([f32(math.cos(2.0 * math.pi * q / 2048.0)) for q in range(2048)], f32)
    want_s = np.array([f32(math.sin(2.0 * math.pi * q / 2048.0)) for q in range(2048)], f32)
    assert bits(c) == bits(want_c) and bits(s) == bits(want_s)
    assert c[0] == 1 and s[0] == 0 and s[512] == 1 and c[1024] == -1


# ---- an independent geometric check ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Wc,H,n", [(1024, 64, 0.0), (1024, 64, OC.ORIGIN_MM), (2048, 128, OC.ORIGIN_MM), (512, 16, 27.116)])
def test_decoded_positions_and_times_match_the_geometry(lv, Wc, H, n):
    """points placed in the LiDAR frame (x forward, y left, z up): pixel p of column m sees along the beam that leaves the beam origin
    n (cos a, -sin a, 0), a = 2 pi m / W, at the altitude alt_p and the angle a + az_p clockwise from +x seen from above; the sensor
    reports the distance along the beam plus n, in mm"""
    rng = np.random.default_rng(23)
    alt, az = OC.beam_angles(H, rng)
    cal = lv.ouster_calibration(Wc, alt, az, n)
    pk = OC.packets(rng, 4, Wc, H, m0=int(rng.integers(0, Wc)), invalid=0, bad_m=0, zero=0)
    slot = np.arange(16 * H * 4)
    col = pk.reshape(-1)
    g, p = slot // H, slot % H
    a = 2 * np.pi * col["m"][g].astype(np.float64) / Wc
    el, th = np.radians(np.array(alt))[p], a + np.radians(np.array(az))[p]
    origin = (n / 1000.0) * np.stack([np.cos(a), -np.sin(a), np.zeros_like(a)], 1)
    s = rng.uniform(0.5, 110.0, len(slot))
    pts = origin + s[:, None] * np.stack([np.cos(el) * np.cos(th), -np.cos(el) * np.sin(th), np.sin(el)], 1)
    # encode each point from its position: the distance from the beam origin, its elevation and its clockwise angle
    v = pts - origin
    dist = np.linalg.norm(v, axis=1)
    assert np.allclose(np.arcsin(v[:, 2] / dist), el, atol=1e-12)
    assert np.allclose(np.mod(np.arctan2(-v[:, 1], v[:, 0]) - th + np.pi, 2 * np.pi) - np.pi, 0, atol=1e-9)
    col["px"]["range"] = np.round((dist * 1000.0 + n)).astype(np.uint32).reshape(-1, H)
    xyz, t, inten, rg, idx = lv.ouster_to_points(pk.tobytes(), cal)
    assert (idx == slot).all()
    tol = 0.0006 + 64 * 2.0**-24 * np.linalg.norm(pts, axis=1)         # half a mm step + the fp32 chain
    err = np.linalg.norm(xyz.astype(np.float64) - pts, axis=1)
    assert (err <= tol).all() and err.max() < 0.002, err.max()
    assert (rg == col["px"]["range"].reshape(-1)).all()
    stamp = col["ts"][g]
    assert (t == stamp // 10**9 + (stamp % 10**9) * 1e-9).all()
    if n == 0 and Wc == 1024:                                           # a quarter turn is to the right (-y)
        z = lv.ouster_calibration(Wc, [0.0] * H, [0.0] * H, 0.0)
        quarter = OC.packets(rng, 1, Wc, H, m0=Wc // 4, invalid=0, bad_m=0, zero=0, garbage=False)
        q = lv.ouster_to_points(quarter.tobytes(), z)[0]
        first = quarter.reshape(-1)["px"]["range"][0] * 1e-3
        assert np.allclose(q[:H], np.stack([np.zeros(H), -first, np.zeros(H)], 1), atol=1e-5)


# ---- the Ouster PointCloud2 path gives the same points --------------------------------------------------------------------------------
def test_same_points_as_the_pointcloud2_path(lv):
    """the decoded frame written as os_cloud_node's cloud (the 48-byte layout: stamp = the first point's column time, t = ts - stamp)
    and read by lv_pointcloud2_to_points_checked(LV_LIDAR_OUSTER, stamp_beginning=1, offset_beginning=1)"""
    rng = np.random.default_rng(24)
    cal = OC.calibration(lv, 1024, 64, OC.ORIGIN_MM, rng)
    pk = OC.frame(rng, 1024, 64, ts0=1_712_345_678 * 10**9 + 123_000)
    col = pk.reshape(-1)
    col["status"][0] = OC.VALID
    col["m"][0] = 0
    xyz, t, inten, rg, idx = lv.ouster_to_points(pk.tobytes(), cal)
    ts = col["ts"][idx // 64]
    assert idx[0] < 64 and ts[0] % 1000 == 0
    stamp_us = int(ts[0]) // 1000
    cloud = np.zeros(len(t), OUSTER)
    cloud["x"], cloud["y"], cloud["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    cloud["t"] = (ts - np.uint64(stamp_us * 1000)).astype(np.uint32)
    cloud["reflectivity"] = col["px"]["refl"].reshape(-1)[idx]
    cloud["ring"] = idx % 64
    cloud["range"] = col["px"]["range"].reshape(-1)[idx] & 0xFFFFF
    L = lv.lib()
    L.lv_pointcloud2_to_points_checked.argtypes = [C.c_int, C.POINTER(CloudLayout), C.POINTER(C.c_uint8), C.c_int64, C.c_int64, C.c_uint64,
                                                   C.c_int, C.c_int, C.c_double, C.POINTER(C.c_float), C.POINTER(C.c_double),
                                                   C.POINTER(C.c_float), C.POINTER(C.c_float)]
    lay = lv.cloud_layout("ouster", OUSTER)
    lay = CloudLayout(*(getattr(lay, f) for f, _ in CloudLayout._fields_))
    n = len(cloud)
    got = (np.zeros((n, 3), f32), np.zeros(n), np.zeros(n, f32), np.zeros(n, f32))
    fp, dp = C.POINTER(C.c_float), C.POINTER(C.c_double)
    assert L.lv_pointcloud2_to_points_checked(lv.LIDAR_TYPES["ouster"], C.byref(lay), cloud.ctypes.data_as(C.POINTER(C.c_uint8)),
                                              cloud.nbytes, n, stamp_us, 1, 1, 0.1, got[0].ctypes.data_as(fp),
                                              got[1].ctypes.data_as(dp), got[2].ctypes.data_as(fp), got[3].ctypes.data_as(fp)) == lv.OK
    assert bits(got[0]) == bits(xyz) and bits(got[2]) == bits(inten) and bits(got[3]) == bits(rg)
    assert np.abs(got[1] - t).max() <= 1e-6
    assert n > 50_000


# ---- IMU packets ---------------------------------------------------------------------------------------------------------------------
def test_imu_packet_decode(lv):
    acc, gyr = (0.01, -0.02, 1.003), (0.5, -12.25, 90.0)
    gyro_ts = 1_712_345_678_987_654_321
    pkt = OC.imu_packet(gyro_ts, acc, gyr, sys_ts=5, accel_ts=gyro_ts - 10**6)
    assert len(pkt) == 48
    s = lv.ouster_imu_packet(pkt)
    assert (s.stamp_sec, s.stamp_nsec) == (1_712_345_678, 987_654_321)      # the gyro ts, not sys or accel
    assert list(s.linear_acceleration) == [float(np.float64(f32(v)) * 9.80665) for v in acc]
    assert list(s.angular_velocity) == [float((np.float64(f32(v)) * math.pi) / 180.0) for v in gyr]
    assert list(s.orientation) == [0.0] * 4
    assert abs(s.linear_acceleration[2] - 1.003 * 9.80665) < 1e-6 and abs(s.angular_velocity[2] - math.pi / 2) < 1e-7
    L = lv.lib()
    out = lv.ImuSample()
    last = OC.imu_packet((2**32 - 1) * 10**9 + 999_999_999, acc, gyr)
    assert L.lv_ouster_imu_packet(last, 48, C.byref(out)) == lv.OK and out.stamp_sec == 2**32 - 1
    over = OC.imu_packet(2**32 * 10**9, acc, gyr)                       # seconds above 2^32 - 1
    assert L.lv_ouster_imu_packet(over, 48, C.byref(out)) == lv.ERR_ARG
    for k in (0, 47, 49):
        buf = (pkt + b"\0")[:k]
        assert L.lv_ouster_imu_packet(buf, k, C.byref(out)) == lv.ERR_ARG, k
    assert L.lv_ouster_imu_packet(None, 48, C.byref(out)) == lv.ERR_ARG
    assert L.lv_ouster_imu_packet(pkt, 48, None) == lv.ERR_ARG
    buf = np.zeros(56, np.uint8)                                        # any alignment
    for shift in range(4):
        buf[shift:shift + 48] = np.frombuffer(pkt, np.uint8)
        assert L.lv_ouster_imu_packet(buf.ctypes.data + shift, 48, C.byref(out)) == lv.OK
        assert list(out.angular_velocity) == list(s.angular_velocity) and out.stamp_nsec == 987_654_321


# ---- the metadata JSON reader --------------------------------------------------------------------------------------------------------
def cal_fields(cal):
    H = cal.pixels_per_column
    return (cal.columns_per_frame, H, list(cal.beam_altitude_angles[:H]), list(cal.beam_azimuth_angles[:H]),
            cal.lidar_origin_to_beam_origin_mm, list(cal.beam_altitude_angles[H:]))


@pytest.mark.parametrize("layout", ["v1", "v2"])
def test_metadata_json_layouts(lv, layout):
    rng = np.random.default_rng(25)
    for Wc in OC.WS:
        for H in OC.HS:
            alt, az = OC.beam_angles(H, rng)
            text = OC.metadata_v1(Wc, alt, az) if layout == "v1" else OC.metadata_v2(Wc, alt, az)
            cal = lv.ouster_calibration_from_json(text)
            n = 0.0 if layout == "v1" else OC.ORIGIN_MM
            assert cal_fields(cal) == (Wc, H, alt, az, n, [0.0] * (128 - H)), (Wc, H)
    alt, az = OC.beam_angles(64)
    assert lv.ouster_calibration_from_json(OC.metadata_v1(1024, alt, az, origin_mm=15.806)).lidar_origin_to_beam_origin_mm == 15.806
    compact = json.dumps(json.loads(OC.metadata_v2(2048, alt, az)), separators=(",", ":"))
    assert cal_fields(lv.ouster_calibration_from_json(compact))[:5] == (2048, 64, alt, az, OC.ORIGIN_MM)
    # a key inside a string value is not a key; the first occurrence of a key counts
    tricky = '{"note": "\\"lidar_mode\\": \\"512x10\\"", "lidar_mode": "1024x20", "beam_altitude_angles": %s, ' \
             '"beam_azimuth_angles": %s, "nested": {"lidar_mode": "2048x10"}}' % (json.dumps(alt), json.dumps(az))
    assert lv.ouster_calibration_from_json(tricky).columns_per_frame == 1024


def test_metadata_json_refusals(lv):
    L = lv.lib()
    alt, az = OC.beam_angles(64)
    good = json.loads(OC.metadata_v2(1024, alt, az))

    def v2(edit):
        d = json.loads(json.dumps(good))
        edit(d)
        return json.dumps(d)

    def refused(text):
        raw = text.encode() if isinstance(text, str) else text
        cal = lv.OusterCalibration()
        cal.columns_per_frame = 99
        st = L.lv_ouster_calibration_from_json(raw, len(raw), C.byref(cal))
        return st == lv.ERR_ARG and cal.columns_per_frame == 0

    assert lv.ouster_calibration_from_json(json.dumps(good)).pixels_per_column == 64
    cases = {
        "no altitudes": v2(lambda d: d["beam_intrinsics"].pop("beam_altitude_angles")),
        "no azimuths": v2(lambda d: d["beam_intrinsics"].pop("beam_azimuth_angles")),
        "no mode": v2(lambda d: d["config_params"].pop("lidar_mode")),
        "lengths differ": v2(lambda d: d["beam_intrinsics"]["beam_azimuth_angles"].pop()),
        "H = 20": OC.metadata_v2(1024, alt[:20], az[:20]),
        "H = 0": v2(lambda d: d["beam_intrinsics"].update(beam_altitude_angles=[], beam_azimuth_angles=[])),
        "W = 1000": v2(lambda d: d["config_params"].update(lidar_mode="1000x10")),
        "W = 4096": v2(lambda d: d["config_params"].update(lidar_mode="4096x5")),
        "mode without rate": v2(lambda d: d["config_params"].update(lidar_mode="1024")),
        "mode without W": v2(lambda d: d["config_params"].update(lidar_mode="x10")),
        "mode with letters": v2(lambda d: d["config_params"].update(lidar_mode="1024x10a")),
        "mode not a string": v2(lambda d: d["config_params"].update(lidar_mode=1024)),
        "pixels_per_column": v2(lambda d: d["lidar_data_format"].update(pixels_per_column=32)),
        "columns_per_packet": v2(lambda d: d["lidar_data_format"].update(columns_per_packet=8)),
        "profile": v2(lambda d: d["config_params"].update(udp_profile_lidar="RNG19_RFL8_SIG16_NIR16")),
        "dual profile": v2(lambda d: d["config_params"].update(udp_profile_lidar="RNG19_RFL8_SIG16_NIR16_DUAL")),
        "origin not a number": v2(lambda d: d["beam_intrinsics"].update(lidar_origin_to_beam_origin_mm="12.163")),
        "string in an array": v2(lambda d: d["beam_intrinsics"]["beam_altitude_angles"].__setitem__(3, "x")),
        "null in an array": v2(lambda d: d["beam_intrinsics"]["beam_azimuth_angles"].__setitem__(3, None)),
        "not an array": v2(lambda d: d["beam_intrinsics"].update(beam_altitude_angles=1.0)),
    }
    for name, text in cases.items():
        assert refused(text), name
    text = json.dumps(good)
    cut = text.index("beam_azimuth_angles") + 60                        # truncated inside an array
    assert refused(text[:cut])
    huge = text.replace(json.dumps(alt[0]), "1e999", 1)                 # not finite
    assert "1e999" in huge and refused(huge)
    assert L.lv_ouster_calibration_from_json(None, 10, C.byref(lv.OusterCalibration())) == lv.ERR_ARG
    assert L.lv_ouster_calibration_from_json(text.encode(), -1, C.byref(lv.OusterCalibration())) == lv.ERR_ARG
    assert L.lv_ouster_calibration_from_json(text.encode(), len(text), None) == lv.ERR_ARG
    raw = text.encode()                                                 # len bounds the text: a prefix is not the whole
    assert L.lv_ouster_calibration_from_json(raw, raw.index(b"beam_intrinsics"), C.byref(lv.OusterCalibration())) == lv.ERR_ARG


# ---- the bag reader ---------------------------------------------------------------------------------------------------------------
def read_bag(lv, path):
    """(topic, type, payload bytes, view status, packet bytes, packet address mod 4) of every message"""
    L = lv.lib()
    L.lv_bag_next.argtypes = [C.c_void_p, C.POINTER(BagMessage)]
    L.lv_bag_close.argtypes = [C.c_void_p]
    bag = C.c_void_p()
    assert L.lv_bag_open(path.encode(), C.byref(bag)) == lv.OK
    out, m = [], BagMessage()
    while L.lv_bag_next(bag, C.byref(m)) == 1:
        v = lv.OusterPacketView()
        st = L.lv_bag_parse_ouster_packet(C.cast(m.data, C.c_void_p), m.size, C.byref(v)) if m.type == b"ouster_ros/PacketMsg" else None
        pkt = C.string_at(v.data, v.bytes) if st == lv.OK else None
        out.append((m.topic.decode(), m.type.decode(), C.string_at(m.data, m.size), st, pkt, (v.data or 0) % 4))
    L.lv_bag_close(bag)
    return out


def packet_bag(rng, cal_json, H=64, Wc=1024, n_packets=6, imu_every=2):
    conns = {0: ("/os_node/metadata", "std_msgs/String"), 1: ("/os_node/lidar_packets", "ouster_ros/PacketMsg"),
             2: ("/os_node/imu_packets", "ouster_ros/PacketMsg")}
    pk = OC.packets(rng, n_packets, Wc, H)
    msgs = [(0, 100, 0, OC.string_msg(cal_json))]
    imus = []
    for k in range(n_packets):
        msgs.append((1, 100, 1000 + k, OC.packet_msg(pk[k].tobytes())))
        if k % imu_every == 0:
            ts = int(pk.reshape(-1)["ts"][16 * k])
            imus.append(OC.imu_packet(ts, rng.normal(0, 0.1, 3), rng.normal(0, 5, 3)))
            msgs.append((2, 100, 1000 + k, OC.packet_msg(imus[-1])))
    return conns, msgs, pk, imus


def test_bag_parse_packet_only_bag(lv, tmp_path):
    rng = np.random.default_rng(26)
    alt, az = OC.beam_angles(64, rng)
    text = OC.metadata_v2(1024, alt, az)
    conns, msgs, pk, imus = packet_bag(rng, text)
    path = str(tmp_path / "ouster.bag")
    W.write_bag(path, conns, msgs)
    got = read_bag(lv, path)
    assert [g[0] for g in got] == [conns[c][0] for c, *_ in msgs]
    meta = got[0][2]
    assert got[0][1] == "std_msgs/String" and struct.unpack_from("<I", meta)[0] == len(meta) - 4
    cal = lv.ouster_calibration_from_json(meta[4:])
    assert cal_fields(cal)[:5] == (1024, 64, alt, az, OC.ORIGIN_MM)
    lidar = [g[4] for g in got if g[0] == "/os_node/lidar_packets"]
    imu = [g[4] for g in got if g[0] == "/os_node/imu_packets"]
    assert all(g[3] == lv.OK for g in got[1:])
    assert lidar == [pk[k].tobytes() for k in range(len(pk))] and imu == imus
    batch = b"".join(lidar)                                             # one frame's packets batched
    same(lv.ouster_to_points(batch, cal), OC.to_points(pk, cal), "bag")
    for raw, want in zip(imu, imus):
        s = lv.ouster_imu_packet(raw)
        gyro_ts = struct.unpack_from("<Q", want, 16)[0]
        assert (s.stamp_sec, s.stamp_nsec) == divmod(gyro_ts, 10**9)
    assert lv.bag_parse_ouster_packet(msgs[1][3]) == pk[0].tobytes()
    seen = set()
    for k in range(4):                                                  # metadata lengths mod 4: the packets at every address mod 4
        path = str(tmp_path / ("align%d.bag" % k))
        W.write_bag(path, {0: conns[0], 1: conns[1]}, [(0, 100, 0, OC.string_msg(text + " " * k)), msgs[1]])
        (_, _, meta, _, _, _), (_, _, _, st, pkt, mod4) = read_bag(lv, path)
        assert st == lv.OK and pkt == pk[0].tobytes()
        assert cal_fields(lv.ouster_calibration_from_json(meta[4:])) == cal_fields(cal)
        seen.add(mod4)
    assert seen == {0, 1, 2, 3}
    ref = OC.to_points(pk, cal)                                         # the decoder reads packets at any address
    nb, n = pk.nbytes, 16 * 64 * len(pk)
    for shift in range(4):
        buf = np.zeros(nb + 8, np.uint8)
        buf[shift:shift + nb] = np.frombuffer(pk.tobytes(), np.uint8)
        out = (np.empty((n, 3), f32), np.empty(n), np.empty(n, f32), np.empty(n, f32), np.empty(n, np.int32))
        m = C.c_int64(0)
        assert lv.lib().lv_ouster_to_points(buf.ctypes.data + shift, nb, len(pk), C.byref(cal), *(a.ctypes.data for a in out),
                                            C.byref(m)) == lv.OK
        same(tuple(a[:m.value] for a in out), ref, shift)


def test_bag_parse_packet_refusals(lv):
    L = lv.lib()
    good = OC.packet_msg(OC.packets(np.random.default_rng(27), 1, 1024, 16).tobytes())
    v = lv.OusterPacketView()
    assert L.lv_bag_parse_ouster_packet(good, len(good), C.byref(v)) == lv.OK and v.bytes == OC.packet_bytes(16)
    for cut in (1, 3, 4, 100, len(good) - 1):                          # truncated anywhere
        assert L.lv_bag_parse_ouster_packet(good, len(good) - cut, C.byref(v)) == lv.ERR_ARG, cut
    assert L.lv_bag_parse_ouster_packet(good + b"\x00", len(good) + 1, C.byref(v)) == lv.ERR_ARG
    empty = OC.packet_msg(b"")
    assert L.lv_bag_parse_ouster_packet(empty, len(empty), C.byref(v)) == lv.OK and v.bytes == 0
    huge = (0xFFFFFFFF).to_bytes(4, "little") + good[4:]
    assert L.lv_bag_parse_ouster_packet(huge, len(huge), C.byref(v)) == lv.ERR_ARG
    assert L.lv_bag_parse_ouster_packet(None, len(good), C.byref(v)) == lv.ERR_ARG
    assert L.lv_bag_parse_ouster_packet(good, len(good), None) == lv.ERR_ARG
    assert L.lv_bag_parse_ouster_packet(good, -1, C.byref(v)) == lv.ERR_ARG


# ---- the host decoder's refusals ------------------------------------------------------------------------------------------------
def test_ouster_to_points_refusals(lv):
    L = lv.lib()
    cal = OC.calibration(lv, 1024, 32)
    pk = OC.packets(np.random.default_rng(28), 3, 1024, 32)
    raw = np.frombuffer(pk.tobytes(), np.uint8)
    n = 16 * 32 * 3
    out = [np.empty(3 * n, np.float32), np.empty(n), np.empty(n, np.float32), np.empty(n, np.float32), np.empty(n, np.int32)]
    ptr = [a.ctypes.data_as(C.c_void_p) for a in out]
    m = C.c_int64(7)

    def call(data=raw.ctypes.data_as(C.c_void_p), nb=len(raw), k=3, c=cal, outs=ptr, n_out=True):
        m.value = 7
        st = L.lv_ouster_to_points(data, nb, k, C.byref(c) if c is not None else None, *outs, C.byref(m) if n_out else None)
        return st, m.value
    good = len(OC.to_points(pk, cal)[0])
    assert call() == (lv.OK, good)
    assert call(outs=ptr[:2] + [None] * 3) == (lv.OK, good)             # intensity, range and idx are optional
    assert call(k=0, nb=0) == (lv.OK, 0)
    assert call(nb=len(raw) + 5) == (lv.OK, good)
    for kw in (dict(data=None), dict(nb=len(raw) - 1), dict(k=-1), dict(k=OC.max_packets(32) + 1, nb=1 << 40), dict(c=None),
               dict(outs=[None] + ptr[1:]), dict(outs=ptr[:1] + [None] + ptr[2:]), dict(nb=-1)):
        assert call(**kw) == (lv.ERR_ARG, 0), kw
    assert call(n_out=False)[0] == lv.ERR_ARG
    for bad in bad_calibrations(lv):
        assert call(c=bad) == (lv.ERR_ARG, 0)
    unused = OC.calibration(lv, 1024, 32)
    unused.beam_altitude_angles[32] = float("nan")                      # beyond H: not read
    unused.beam_azimuth_angles[127] = float("inf")
    assert call(c=unused) == (lv.OK, good)


def bad_calibrations(lv):
    out = []
    for Wc, H in ((1000, 32), (0, 32), (4096, 32), (1024, 0), (1024, 24), (1024, 256), (1024, -16)):
        c = OC.calibration(lv, 1024, 32)
        c.columns_per_frame, c.pixels_per_column = Wc, H
        out.append(c)
    for name, p in (("beam_altitude_angles", 0), ("beam_altitude_angles", 31), ("beam_azimuth_angles", 5)):
        for v in (float("nan"), float("inf"), -float("inf")):
            c = OC.calibration(lv, 1024, 32)
            getattr(c, name)[p] = v
            out.append(c)
    for v in (float("nan"), float("inf")):
        c = OC.calibration(lv, 1024, 32)
        c.lidar_origin_to_beam_origin_mm = v
        out.append(c)
    return out


# ---- the device calls' argument checks (before any device work) --------------------------------------------------------------------
NP = 10
HH = 64
NB = OC.packet_bytes(HH) * NP
NS = 16 * HH * NP


@pytest.fixture
def dcall(lv):
    L = lv.lib()
    good = OC.calibration(lv, 1024, HH)

    def run(h=None, data=BASE, data_bytes=NB, k=NP, cal=good, outs=None, n_out=True, asynch=False):
        outs = outs if outs is not None else [BASE + (1 << 30) + j * (1 << 24) for j in range(5)]
        c = C.byref(cal) if cal is not None else None
        if asynch:
            st = L.lv_process_ouster_device_async(h, data, data_bytes, k, c, 4, 3.0, *outs, BASE + (1 << 35) if n_out else None)
        else:
            m = C.c_int64(7)
            st = L.lv_process_ouster_device(h, data, data_bytes, k, c, 4, 3.0, *outs, C.byref(m) if n_out else None)
            if n_out:
                assert m.value == 0
        return st, L.lv_last_error()
    return run


@pytest.mark.parametrize("asynch", [False, True])
def test_process_ouster_refusals_before_device_work(lv, dcall, asynch):
    handle = (lv.ERR_ARG, b"process ouster: null handle")
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
    for k in (-1, OC.max_packets(HH) + 1, 1 << 62):
        st, msg = dcall(asynch=asynch, k=k, data_bytes=1 << 45)
        assert st == lv.ERR_ARG and (b"n_packets" in msg or b"negative" in msg), k
    assert dcall(asynch=asynch, k=0, data_bytes=0) == handle
    st, msg = dcall(asynch=asynch, data_bytes=NB - 1)
    assert st == lv.ERR_ARG and b"too short" in msg
    for bad in bad_calibrations(lv):
        st, msg = dcall(asynch=asynch, cal=bad)
        assert st == lv.ERR_ARG and (b"not finite" in msg or b"columns_per_frame" in msg or b"pixels_per_column" in msg), msg
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
