"""VelodyneScan for the tests: a serialiser of velodyne_msgs/VelodyneScan (ROS 1, little endian), a VLP-16 packet generator, and a
NumPy restatement of the Velodyne front end's semantics (include/limovelo_b200.h, "Velodyne packets"):

    slots        i -> packet k = i // 384, r = i % 384, block b = r // 32, firing f = (r % 32) // 16, laser l = r % 16
    msg2points   mode != 0x39, blocks 0 .. b flagged 0xEEFF, distance != 0
    azimuth      a = A_b + D_b (l 2.304 + f 55.296) / 110.592 in float32, q = round half away from zero, mod 36000
    xyz          float32, every product and sum one rounding, tables from float64 cos / sin rounded to float32
    time         sec 1e9 + nsec + (2b + f) 55296 + l 2304 in uint64 ns, then seconds as for Livox
    decimate     temporal_keep on the RANK among the msg2points points (frontend_ref.temporal on the point list)
    sort         stable by time

Every NumPy float32 operation below is one IEEE rounding; nothing is fused."""
import math
import struct

import numpy as np

import frontend_ref as F

f32 = np.float32
CHANNEL = np.dtype([("dist", "<u2"), ("refl", "u1")])
BLOCK = np.dtype([("flag", "<u2"), ("azimuth", "<u2"), ("ch", CHANNEL, (32,))])
DATA = np.dtype([("blocks", BLOCK, (12,)), ("stamp_us", "<u4"), ("mode", "u1"), ("product", "u1")])
PACKET = np.dtype([("sec", "<u4"), ("nsec", "<u4"), ("data", DATA)])
assert CHANNEL.itemsize == 3 and BLOCK.itemsize == 100 and DATA.itemsize == 1206 and PACKET.itemsize == 1214
SLOTS = 384
FLAG = 0xEEFF
STRONGEST, LAST, DUAL = 0x37, 0x38, 0x39
PACKET_NS = 24 * 55296                       # one packet: 12 blocks x 2 firing sequences
VLP16_DEG = [-15, 1, -13, 3, -11, 5, -9, 7, -7, 9, -5, 11, -3, 13, -1, 15]
HIRES_DEG = [-10, 0.67, -8.67, 2, -7.33, 3.33, -6, 4.67, -4.67, 6, -3.33, 7.33, -2, 8.67, -0.67, 10]
MAX_PACKETS = (2**31 - 1) // SLOTS


def _string(s):
    s = s.encode()
    return struct.pack("<I", len(s)) + s


def scan_msg(packets, sec=0, nsec=0, frame="velodyne", seq=0):
    """packets (PACKET array) -> serialised velodyne_msgs/VelodyneScan"""
    pk = np.ascontiguousarray(packets, PACKET)
    return struct.pack("<III", seq, sec, nsec) + _string(frame) + struct.pack("<I", len(pk)) + pk.tobytes()


def packets(rng, n, az0=None, step=20, sec=1_700_000_000, nsec=0, zero=0.1, mode=STRONGEST, max_range=120.0):
    """n single-return VLP-16 packets of one sweep: block azimuths rising by `step` (0.01 deg) and wrapping at 36000, random
    distances (a fraction `zero` without return) and reflectivities, packet stamps PACKET_NS apart from (sec, nsec)"""
    pk = np.zeros(n, PACKET)
    az0 = int(rng.integers(0, 36000)) if az0 is None else az0
    blocks = pk["data"]["blocks"]
    blocks["flag"] = FLAG
    blocks["azimuth"] = (az0 + step * np.arange(12 * n).reshape(n, 12)) % 36000
    dist = rng.integers(1, int(max_range / 0.002), (n, 12, 32))
    dist[rng.random((n, 12, 32)) < zero] = 0
    blocks["ch"]["dist"] = dist
    blocks["ch"]["refl"] = rng.integers(0, 256, (n, 12, 32))
    pk["data"]["stamp_us"] = rng.integers(0, 3_600_000_000, n)
    pk["data"]["mode"] = mode
    pk["data"]["product"] = 0x22
    total = sec * 10**9 + nsec + PACKET_NS * np.arange(n, dtype=np.int64).astype(object)
    pk["sec"] = [t // 10**9 for t in total]
    pk["nsec"] = [t % 10**9 for t in total]
    return pk


def edge_packets(rng):
    """named packet sets at the edges of the semantics"""
    out = {}
    out["empty"] = packets(rng, 0)
    out["one"] = packets(rng, 1)
    p = packets(rng, 6, az0=35_900)                                    # the azimuth wraps inside a packet
    out["wrap"] = p
    p = packets(rng, 5)
    p["data"]["blocks"]["flag"][1, 7] = 0xDDFF                         # upper-block flag: blocks 7 .. 11 of packet 1 are no points
    p["data"]["blocks"]["flag"][3, 0] = 0                              # the whole packet 3
    p["data"]["blocks"]["flag"][4, 11] = 0x1234                        # the last block only
    out["bad_flags"] = p
    p = packets(rng, 4)
    p["data"]["mode"][2] = LAST
    out["last_return"] = p
    p = packets(rng, 4, zero=0.9)
    p["data"]["blocks"]["ch"]["dist"][0] = 0                          # a packet without a return
    out["sparse"] = p
    p = packets(rng, 8, sec=1_600_000_000, nsec=999_990_000)           # the ns -> s carry between packets
    out["ns_carry"] = p
    out["epoch_max"] = packets(rng, 3, sec=2**32 - 1, nsec=999_999_999 - 2 * PACKET_NS)
    out["sec_zero"] = packets(rng, 3, sec=0, nsec=0)
    p = packets(rng, 4)
    p["data"]["blocks"]["azimuth"][1, 5] = 65535                       # raw azimuths outside [0, 36000)
    p["data"]["blocks"]["azimuth"][2, 11] = 40000
    out["raw_azimuth"] = p
    p = packets(rng, 3, max_range=1.0)                                 # inside min_dist
    out["near"] = p
    p = packets(rng, 4)
    p["sec"], p["nsec"] = p["sec"][0], p["nsec"][0]                    # equal stamps: equal times keep slot order
    out["equal_stamps"] = p
    return out


def dual_packets(rng):
    """packets with one dual-return packet among them (no points, a deferred error on the device)"""
    p = packets(rng, 5)
    p["data"]["mode"][2] = DUAL
    return p


def bad_stamp_packets(rng):
    """packets with one stamp whose nsec is 10^9 (cannot be converted)"""
    p = packets(rng, 4)
    p["nsec"][1] = 1_000_000_000
    return p


# ---- calibrations -------------------------------------------------------------------------------------------------------------------
def calibration(lv, model="vlp16"):
    return lv.velodyne_calibration(model)


def random_calibration(lv, rng):
    """a factory-like calibration: the VLP-16 angles plus small corrections and offsets of every kind"""
    cal = lv.velodyne_calibration("vlp16")
    for l in range(16):
        cal.vert_correction[l] += float(rng.normal(0, 0.002))
        cal.rot_correction[l] = float(rng.normal(0, 0.02))
        cal.dist_correction[l] = float(rng.normal(0, 0.03))
        cal.vert_offset_correction[l] = float(rng.normal(0, 0.01))
        cal.horiz_offset_correction[l] = float(rng.normal(0, 0.01))
    return cal


def _calib32(cal):
    g = lambda name: np.array(getattr(cal, name)[:], np.float64)
    vert, rot = g("vert_correction"), g("rot_correction")
    c32 = lambda fn, v: np.array([f32(fn(float(a))) for a in v], f32)
    return dict(cv=c32(math.cos, vert), sv=c32(math.sin, vert), cr=c32(math.cos, rot), sr=c32(math.sin, rot),
                dist=g("dist_correction").astype(f32), vo=g("vert_offset_correction").astype(f32),
                ho=g("horiz_offset_correction").astype(f32))


_TABLES = None


def tables():
    """C[q], S[q]: float64 cos / sin of q 0.01 pi / 180 (evaluated left to right), rounded to float32"""
    global _TABLES
    if _TABLES is None:
        a = [q * 0.01 * math.pi / 180.0 for q in range(36000)]
        _TABLES = (np.array([math.cos(x) for x in a], f32), np.array([math.sin(x) for x in a], f32))
    return _TABLES


# ---- the rotation tables read back through the decoder ------------------------------------------------------------------------------
def table_packets():
    """3000 packets whose block b of packet k has azimuth q = 12 k + b and every distance 500 (d = 500 x 0.002f rounds to exactly 1):
    with the all-zero calibration (cv = cr = 1, sv = sr = 0) slot r = 32 b (firing 0, laser 0, a = A_b) decodes to exactly
    (x, y, z) = (C[q], -S[q], 0)"""
    pk = np.zeros(3000, PACKET)
    blocks = pk["data"]["blocks"]
    blocks["flag"] = FLAG
    blocks["azimuth"] = np.arange(36000).reshape(3000, 12)
    blocks["ch"]["dist"] = 500
    pk["data"]["mode"] = STRONGEST
    return pk


def tables_from_points(xyz, idx):
    """(C, S) from the decoded points of table_packets (slot order or not): the points of the slots r = 32 b"""
    sel = idx % 32 == 0
    q = (idx[sel] // 384) * 12 + (idx[sel] % 384) // 32
    C, S = np.empty(36000, f32), np.empty(36000, f32)
    C[q], S[q] = xyz[sel, 0], -xyz[sel, 1]
    assert np.array_equal(np.sort(q), np.arange(36000)) and (xyz[sel, 2] == 0).all()
    return C, S


# ---- the restatement ------------------------------------------------------------------------------------------------------------------
def to_points(pk, cal):
    """msg2points: (xyz, time, intensity, range, slot) of the points, in slot order"""
    pk = np.ascontiguousarray(pk, PACKET)
    n = SLOTS * len(pk)
    i = np.arange(n)
    k, r = i // SLOTS, i % SLOTS
    b, f, l = r // 32, (r % 32) // 16, r % 16
    blocks = pk["data"]["blocks"]
    flagged = np.logical_and.accumulate(blocks["flag"] == FLAG, axis=1) if len(pk) else np.zeros((0, 12), bool)
    raw = blocks["ch"]["dist"].reshape(len(pk), SLOTS)[k, r]
    valid = (pk["data"]["mode"][k] != DUAL) & flagged[k, b] & (raw != 0)
    k, r, b, f, l, raw = k[valid], r[valid], b[valid], f[valid], l[valid], raw[valid]
    A = blocks["azimuth"].astype(np.int64)
    delta = np.zeros_like(A)
    delta[:, :11] = (A[:, 1:] + 36000 - A[:, :11]) % 36000
    delta[:, 11] = delta[:, 10]
    a = A[k, b].astype(f32) + (delta[k, b].astype(f32) * (l.astype(f32) * f32(2.304) + f.astype(f32) * f32(55.296))) / f32(110.592)
    assert a.dtype == f32
    q = np.floor(a.astype(np.float64) + 0.5).astype(np.int64) % 36000      # a >= 0: half away from zero
    C, S = tables()
    c = _calib32(cal)
    d = raw.astype(f32) * f32(0.002) + c["dist"][l]
    cosr = C[q] * c["cr"][l] + S[q] * c["sr"][l]
    sinr = S[q] * c["cr"][l] - C[q] * c["sr"][l]
    xy = d * c["cv"][l] - c["vo"][l] * c["sv"][l]
    X = xy * sinr - c["ho"][l] * cosr
    Y = xy * cosr + c["ho"][l] * sinr
    Z = d * c["sv"][l] + c["vo"][l] * c["cv"][l]
    xyz = np.stack([Y, -X, Z], 1).astype(f32).reshape(-1, 3)
    assert xyz.dtype == f32 and Z.dtype == f32
    total = (pk["sec"][k].astype(np.uint64) * np.uint64(10**9) + pk["nsec"][k].astype(np.uint64) +
             (2 * b + f).astype(np.uint64) * np.uint64(55296) + l.astype(np.uint64) * np.uint64(2304))
    qs, rem = total // np.uint64(10**9), total % np.uint64(10**9)
    t = qs.astype(np.int64).astype(np.float64) + rem.astype(np.float64) * 1e-9          # two ufuncs: unfused
    inten = blocks["ch"]["refl"].reshape(len(pk), SLOTS)[k, r].astype(f32)
    x, y, z = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    rng_ = np.sqrt((x * x + y * y) + z * z)
    return xyz, t, inten, rng_.astype(f32), (SLOTS * k + r).astype(np.int32)


def process(pk, cal, rate, min_dist):
    """Accumulator::process on a VelodyneScan: msg2points -> decimation on the rank -> stable time sort"""
    xyz, t, inten, rg, idx = to_points(pk, cal)
    keep = F.temporal(xyz, rate, min_dist)
    order = keep[np.argsort(t[keep], kind="stable")]
    return xyz[order], t[order], inten[order], rg[order], idx[order]
