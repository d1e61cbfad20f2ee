"""Ouster packets for the tests: serialisers of ouster_ros/PacketMsg and std_msgs/String (ROS 1, little endian), a LEGACY lidar packet
generator for any W / H, an IMU packet encoder, metadata JSON writers in the firmware 1.x (flat) and 2.x (nested) layouts, and a
NumPy restatement of the Ouster front end's semantics (include/limovelo_b200.h, "Ouster packets"):

    slots        i -> column g = i // H (packet g // 16, column g % 16), pixel p = i % H
    msg2points   status bit 0 set, measurement_id m < W, range r = word & 0xFFFFF != 0
    tables       C[q], S[q] = float64 cos / sin of 2 pi q / 2048 rounded to float32; column m reads q = m (2048 / W)
    xyz          float32: e = r 0.001 - nf; ch = C ca - S sa; sh = S ca + C sa; ee = e ce; x = ee ch + nf C; y = -(ee sh + nf S); z = e se
    time         the column's uint64 ns timestamp, then seconds as for Livox
    decimate     temporal_keep on the RANK among the msg2points points (frontend_ref.temporal on the point list)
    sort         stable by time

Every NumPy float32 operation below is one IEEE rounding; nothing is fused."""
import json
import math
import struct

import numpy as np

import frontend_ref as F

f32 = np.float32
PIXEL = np.dtype([("range", "<u4"), ("refl", "<u2"), ("signal", "<u2"), ("noise", "<u2"), ("pad", "<u2")])
assert PIXEL.itemsize == 12
COLUMNS = 16
TABLE = 2048
RANGE_MASK = 0xFFFFF
VALID = 0xFFFFFFFF
WS = (512, 1024, 2048)
HS = (16, 32, 64, 128)
ORIGIN_MM = 12.163                                     # OS1 firmware 2.x: lidar_origin_to_beam_origin_mm


def column_dtype(H):
    return np.dtype([("ts", "<u8"), ("m", "<u2"), ("frame_id", "<u2"), ("encoder", "<u4"), ("px", PIXEL, (H,)), ("status", "<u4")])


def packet_dtype(H):
    d = np.dtype((column_dtype(H), (COLUMNS,)))
    assert d.itemsize == COLUMNS * (20 + 12 * H)
    return d


def packet_bytes(H):
    return COLUMNS * (20 + 12 * H)


def max_packets(H):
    return (2**31 - 1) // (COLUMNS * H)


# ---- messages -----------------------------------------------------------------------------------------------------------------------
def packet_msg(pkt):
    """one packet's bytes -> serialised ouster_ros/PacketMsg (uint8[] buf)"""
    b = bytes(memoryview(pkt))
    return struct.pack("<I", len(b)) + b


def string_msg(text):
    """serialised std_msgs/String"""
    b = text.encode()
    return struct.pack("<I", len(b)) + b


def imu_packet(gyro_ts, acc_g, gyro_dps, sys_ts=None, accel_ts=None):
    """the 48 bytes of an IMU packet: sys / accel / gyro timestamps (ns), accelerations in g and angular rates in deg/s (float32)"""
    sys_ts = gyro_ts + 1234 if sys_ts is None else sys_ts
    accel_ts = gyro_ts - 777 if accel_ts is None else accel_ts
    return struct.pack("<QQQ3f3f", sys_ts, accel_ts, gyro_ts, *[float(f32(v)) for v in acc_g], *[float(f32(v)) for v in gyro_dps])


# ---- calibrations and metadata ------------------------------------------------------------------------------------------------------
def beam_angles(H, rng=None):
    """OS1-like beam intrinsics: altitudes from +16.6 to -16.6 deg, azimuth offsets in a repeating 4-beam pattern (degrees)"""
    alt = np.linspace(16.6, -16.6, H)
    az = np.tile([4.23, 1.41, -1.41, -4.23], H // 4)
    if rng is not None:
        alt = alt + rng.normal(0, 0.05, H)
        az = az + rng.normal(0, 0.02, H)
    return [float(a) for a in alt], [float(a) for a in az]


def calibration(lv, W=1024, H=64, origin_mm=0.0, rng=None):
    alt, az = beam_angles(H, rng)
    return lv.ouster_calibration(W, alt, az, origin_mm)


def _mode(W, hz=10):
    return "%dx%d" % (W, hz)


def metadata_v1(W, alt, az, origin_mm=None, **extra):
    """firmware 1.x metadata: every key at the top level"""
    d = {"hostname": "os1-991900123456.local", "prod_line": "OS-1-%d" % len(alt), "prod_sn": "991900123456",
         "build_rev": "v1.13.0", "lidar_mode": _mode(W), "beam_altitude_angles": list(alt), "beam_azimuth_angles": list(az),
         "imu_to_sensor_transform": [1, 0, 0, 6.253, 0, 1, 0, -11.775, 0, 0, 1, 7.645, 0, 0, 0, 1],
         "lidar_to_sensor_transform": [-1, 0, 0, 0, 0, -1, 0, 0, 0, 0, 1, 36.18, 0, 0, 0, 1]}
    if origin_mm is not None:
        d["lidar_origin_to_beam_origin_mm"] = origin_mm
    d.update(extra)
    return json.dumps(d, indent=2)


def metadata_v2(W, alt, az, origin_mm=ORIGIN_MM, profile="LEGACY", H=None, columns_per_packet=16):
    """firmware 2.x metadata: the keys nested under beam_intrinsics, config_params and lidar_data_format"""
    H = len(alt) if H is None else H
    d = {"beam_intrinsics": {"beam_altitude_angles": list(alt), "beam_azimuth_angles": list(az),
                             "lidar_origin_to_beam_origin_mm": origin_mm},
         "calibration_status": {"reflectivity": {"valid": True}},
         "config_params": {"azimuth_window": [0, 360000], "lidar_mode": _mode(W), "udp_profile_lidar": profile,
                           "udp_profile_imu": "LEGACY"},
         "lidar_data_format": {"column_window": [0, W - 1], "columns_per_frame": W, "columns_per_packet": columns_per_packet,
                               "pixel_shift_by_row": [12, 4, -4, -12] * (H // 4), "pixels_per_column": H},
         "sensor_info": {"build_rev": "v2.3.0", "prod_line": "OS-1-%d" % H, "prod_sn": "122201000998", "status": "RUNNING"}}
    return json.dumps(d)


# ---- LEGACY packets -----------------------------------------------------------------------------------------------------------------
def column_ns(W, hz=10):
    return 10**9 // (hz * W)


def packets(rng, n, W=1024, H=64, m0=0, frame_id=7, ts0=1_700_000_000 * 10**9, invalid=0.02, bad_m=0.01, zero=0.1,
            garbage=True, max_mm=120_000):
    """n LEGACY packets of one sensor: measurement ids m0, m0 + 1, ... wrapping at W (the frame id counts the wraps), column stamps
    column_ns(W) apart from ts0, random ranges (a fraction `zero` without return) and reflectivities.  A fraction `invalid` of the
    columns has a status without bit 0 (0 or 0xFFFFFFFE), a fraction `bad_m` an id >= W; `garbage` fills the upper 12 bits of the
    range words"""
    pk = np.zeros(n, packet_dtype(H))
    col = pk.reshape(-1) if n else np.zeros(0, column_dtype(H))
    g = np.arange(16 * n)
    m = (m0 + g) % W
    col["m"] = m
    col["frame_id"] = (frame_id + (m0 + g) // W) % 65536
    col["ts"] = np.uint64(ts0) + g.astype(np.uint64) * np.uint64(column_ns(W))
    col["encoder"] = rng.integers(0, 90112, 16 * n)
    col["status"] = VALID
    bad = rng.random(16 * n) < invalid
    col["status"][bad] = rng.choice(np.array([0, 0xFFFFFFFE], np.uint32), int(bad.sum()))
    wrong = rng.random(16 * n) < bad_m
    col["m"][wrong] = rng.choice(np.array([W, W + 1, 2047, 4095, 65535], np.uint32), int(wrong.sum()))
    r = rng.integers(1, max_mm, (16 * n, H)).astype(np.uint32)
    r[rng.random((16 * n, H)) < zero] = 0
    if garbage:
        r |= (rng.integers(0, 4096, (16 * n, H)).astype(np.uint32) << 20)
    px = col["px"]
    px["range"] = r
    px["refl"] = rng.integers(0, 65536, (16 * n, H))
    px["signal"] = rng.integers(0, 65536, (16 * n, H))
    px["noise"] = rng.integers(0, 65536, (16 * n, H))
    return pk


def frame(rng, W, H, cols_missing=0.1, **kw):
    """the W / 16 packets of one full frame starting at measurement id 0, a fraction `cols_missing` of the pixels without a return"""
    return packets(rng, W // 16, W, H, m0=0, zero=cols_missing, **kw)


# ---- the column table read back through the decoder ---------------------------------------------------------------------------------
def table_packets():
    """128 packets (W = 2048, H = 16): column m = q, every status valid, every range 1000 mm (1000 x 0.001f rounds to exactly 1).
    With zero angles and n = 0 (ce = ca = 1, se = sa = 0) pixel 0 of column q decodes to exactly (x, y, z) = (C[q], -S[q], 0)"""
    pk = np.zeros(128, packet_dtype(16))
    col = pk.reshape(-1)
    col["m"] = np.arange(2048)
    col["status"] = VALID
    col["px"]["range"] = 1000
    return pk


def table_calibration(lv):
    return lv.ouster_calibration(2048, [0.0] * 16, [0.0] * 16, 0.0)


def tables_from_points(xyz, idx):
    """(C, S) from the decoded points of table_packets (slot order or not): the points of pixel 0"""
    sel = idx % 16 == 0
    q = idx[sel] // 16
    C, S = np.empty(TABLE, f32), np.empty(TABLE, f32)
    C[q], S[q] = xyz[sel, 0], -xyz[sel, 1]
    assert np.array_equal(np.sort(q), np.arange(TABLE)) and (xyz[sel, 2] == 0).all()
    return C, S


_TABLE = None


def table():
    """C[q], S[q]: float64 cos / sin of 2 pi q / 2048 (evaluated left to right), rounded to float32"""
    global _TABLE
    if _TABLE is None:
        a = [2.0 * math.pi * q / 2048.0 for q in range(TABLE)]
        _TABLE = (np.array([math.cos(x) for x in a], f32), np.array([math.sin(x) for x in a], f32))
    return _TABLE


def _beams32(cal):
    H = cal.pixels_per_column
    alt = [cal.beam_altitude_angles[p] * math.pi / 180.0 for p in range(H)]
    az = [cal.beam_azimuth_angles[p] * math.pi / 180.0 for p in range(H)]
    c32 = lambda fn, v: np.array([f32(fn(a)) for a in v], f32)
    return c32(math.cos, alt), c32(math.sin, alt), c32(math.cos, az), c32(math.sin, az), f32(cal.lidar_origin_to_beam_origin_mm * 0.001)


# ---- the restatement ------------------------------------------------------------------------------------------------------------------
def to_points(pk, cal):
    """msg2points: (xyz, time, intensity, range, slot) of the points, in slot order"""
    W, H = cal.columns_per_frame, cal.pixels_per_column
    col = np.ascontiguousarray(pk).reshape(-1).view(column_dtype(H)) if len(pk) else np.zeros(0, column_dtype(H))
    n = H * len(col)
    i = np.arange(n)
    g, p = i // H, i % H
    r = col["px"]["range"].reshape(-1) & RANGE_MASK
    valid = ((col["status"][g] & 1) == 1) & (col["m"][g].astype(np.int64) < W) & (r != 0)
    g, p, r, i = g[valid], p[valid], r[valid], i[valid]
    ce, se, ca, sa, nf = _beams32(cal)
    C, S = table()
    q = col["m"][g].astype(np.int64) * (TABLE // W)
    c, s = C[q], S[q]
    e = r.astype(f32) * f32(0.001) - nf
    ch = c * ca[p] - s * sa[p]
    sh = s * ca[p] + c * sa[p]
    ee = e * ce[p]
    x = ee * ch + nf * c
    y = -(ee * sh + nf * s)
    z = e * se[p]
    xyz = np.stack([x, y, z], 1).astype(f32).reshape(-1, 3)
    assert x.dtype == f32 and z.dtype == f32
    ts = col["ts"][g]
    t = (ts // np.uint64(10**9)).astype(np.int64).astype(np.float64) + (ts % np.uint64(10**9)).astype(np.float64) * 1e-9   # unfused
    inten = col["px"]["refl"].reshape(-1)[i].astype(f32)
    return xyz, t, inten, r.astype(f32), i.astype(np.int32)


def process(pk, cal, rate, min_dist):
    """Accumulator::process on Ouster packets: msg2points -> decimation on the rank -> stable time sort"""
    xyz, t, inten, rg, idx = to_points(pk, cal)
    keep = F.temporal(xyz, rate, min_dist)
    order = keep[np.argsort(t[keep], kind="stable")]
    return xyz[order], t[order], inten[order], rg[order], idx[order]
