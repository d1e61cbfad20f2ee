"""Livox CustomMsg for the tests: a serialiser of livox_ros_driver/CustomMsg (ROS 1, little endian), random and edge record sets, and
a NumPy restatement of the Livox front end's semantics (include/limovelo_b200.h, "Livox messages"):

    msg2points   keep a record iff (tag & mask) == 0; xyz as stored; time = (double)(int64)(total // 1e9) + (double)(total % 1e9) * 1e-9
                 with total = timebase + offset_time in uint64; intensity = reflectivity; range = the fp32 norm; idx = message index
    decimate     temporal_keep on the RANK among the tag-kept points (frontend_ref.temporal on the kept list)
    sort         stable by time"""
import struct

import numpy as np

import frontend_ref as F

f32 = np.float32
RECORD = np.dtype({"names": ["offset_time", "x", "y", "z", "reflectivity", "tag", "line"],
                   "formats": ["<u4", "<f4", "<f4", "<f4", "u1", "u1", "u1"], "offsets": [0, 4, 8, 12, 16, 17, 18], "itemsize": 19})
TIMEBASE_MAX = (1 << 64) - (1 << 32)
MASKS = [0, 0x20, 0x0F, 0xFF]


def _string(s):
    s = s.encode()
    return struct.pack("<I", len(s)) + s


def custom_msg(records, timebase, sec=0, nsec=0, frame="livox_frame", seq=0, lidar_id=0, point_num=None):
    """records (RECORD array) -> serialised livox_ros_driver/CustomMsg"""
    recs = np.ascontiguousarray(records, RECORD)
    out = struct.pack("<III", seq, sec, nsec) + _string(frame)
    out += struct.pack("<QIB", timebase, len(recs) if point_num is None else point_num, lidar_id) + b"\x00\x00\x00"
    return out + struct.pack("<I", len(recs)) + recs.tobytes()


def records(rng, n, scale=40.0, t_span=100_000_000):
    """n records: coordinates in a +-scale box, times spread over t_span ns (not sorted), every tag bit and line in use"""
    r = np.zeros(n, RECORD)
    for k in "xyz":
        r[k] = rng.uniform(-scale, scale, n).astype(f32)
    r["offset_time"] = rng.integers(0, t_span, n, dtype=np.uint32)
    r["reflectivity"] = rng.integers(0, 256, n)
    r["tag"] = rng.integers(0, 256, n)
    r["line"] = rng.integers(0, 6, n)
    return r


def to_points(recs, timebase, mask):
    """msg2points: (xyz, time, intensity, range, idx) of the tag-kept records, in message order"""
    recs = np.ascontiguousarray(recs, RECORD)
    idx = np.nonzero((recs["tag"] & mask) == 0)[0].astype(np.int32)
    r = recs[idx]
    xyz = np.stack([r["x"], r["y"], r["z"]], 1).astype(f32).reshape(-1, 3)
    total = np.uint64(timebase) + r["offset_time"].astype(np.uint64)
    q, rem = total // np.uint64(1_000_000_000), total % np.uint64(1_000_000_000)
    t = q.astype(np.int64).astype(np.float64) + rem.astype(np.float64) * 1e-9      # two ufuncs: unfused
    x, y, z = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    rng_ = np.sqrt((x * x + y * y) + z * z)
    return xyz, t, r["reflectivity"].astype(f32), rng_.astype(f32), idx


def process(recs, timebase, mask, rate, min_dist):
    """Accumulator::process on a Livox message: msg2points -> decimation on the rank -> stable time sort"""
    xyz, t, inten, rg, idx = to_points(recs, timebase, mask)
    keep = F.temporal(xyz, rate, min_dist)
    order = keep[np.argsort(t[keep], kind="stable")]
    return xyz[order], t[order], inten[order], rg[order], idx[order]


def edge_records(rng):
    """named record sets at the edges of the semantics, each with its time base"""
    out = {}
    out["empty"] = (np.zeros(0, RECORD), 1_700_000_000 * 10**9)
    out["one"] = (records(rng, 1), 1_700_000_000 * 10**9)
    r = records(rng, 600)
    r["offset_time"] = rng.integers(0, 5, 600)                        # heavy ties: equal times keep message order
    out["ties"] = (r, 1_700_000_000 * 10**9 + 123)
    r = records(rng, 800)                                             # total % 1e9 near 0 and 999 999 999
    r["offset_time"] = (np.where(rng.random(800) < 0.5, 999_999_990, 1_000_000_000) + rng.integers(0, 20, 800)).astype(np.uint32)
    out["ns_boundary"] = (r, 1_700_000_000 * 10**9)
    r = records(rng, 500)
    r["offset_time"][:4] = [0, 0xFFFFFFFF, 1, 0xFFFFFFFE]
    out["timebase_at_limit"] = (r, TIMEBASE_MAX)
    out["timebase_zero"] = (records(rng, 300), 0)
    r = records(rng, 900)
    near = rng.choice(900, 300, replace=False)
    for k in "xyz":
        r[k][near] *= f32(0.01)                                       # inside min_dist
    for k in "xyz":
        r[k][rng.choice(900, 40, replace=False)] = np.nan              # dropped by min_dist < |p|
    out["near_and_nan"] = (r, 1_600_000_000 * 10**9 + 999_999_999)
    r = records(rng, 256)
    r["tag"] = np.arange(256)                                         # every tag value once
    out["every_tag"] = (r, 1_650_000_000 * 10**9)
    return out
