"""Ouster packets of the lidar UDP profiles of firmware 2.2+ for the tests (include/limovelo_b200.h, "Ouster packets"): an encoder
that re-encodes LEGACY packets of tests/ouster_cases.py in RNG19_RFL8_SIG16_NIR16, its dual-return form or the low-data
RNG15_RFL8_NIR8, a metadata writer with any udp_profile_lidar, and a NumPy restatement of the header's profile table:

    packet       32-byte header | 16 columns of uint64 ts | uint16 m | uint16 status | H pixels of s bytes | 32-byte footer
    msg2points   status bit 0 set, measurement_id m < W, range r != 0, r = (u<width> @0 & mask) << shift
    outputs      the LEGACY geometry and time of ouster_cases on r; intensity = u8 @refl

Every NumPy float32 operation below is one IEEE rounding; nothing is fused."""
import json

import numpy as np

import frontend_ref as F
from ouster_cases import (COLUMNS, ORIGIN_MM, RANGE_MASK, TABLE, _beams32, metadata_v1, metadata_v2, packet_bytes, packets, table,
                          to_points)

f32 = np.float32

# lv_ouster_profile values and the metadata's udp_profile_lidar strings
LEGACY, RNG19, DUAL, LOW = 0, 1, 2, 3
PROFILE_NAMES = ("LEGACY", "RNG19_RFL8_SIG16_NIR16", "RNG19_RFL8_SIG16_NIR16_DUAL", "RNG15_RFL8_NIR8")
NEW_PROFILES = (RNG19, DUAL, LOW)
# the header's table: pixel bytes s; range = (u<width> @0 & mask) << shift; reflectivity = u8 @refl.  Packet: 32-byte header | 16
# columns of uint64 ts | uint16 m | uint16 status | H pixels of s bytes | 32-byte footer
PROFILE_TABLE = {RNG19: dict(s=12, width=4, mask=0x7FFFF, shift=0, refl=4),
                 DUAL: dict(s=16, width=4, mask=0x7FFFF, shift=0, refl=3),
                 LOW: dict(s=4, width=2, mask=0x7FFF, shift=3, refl=2)}


def profile_packet_bytes(profile, H):
    if profile == LEGACY:
        return packet_bytes(H)
    return 32 + COLUMNS * (12 + PROFILE_TABLE[profile]["s"] * H) + 32


def profile_packet_dtype(profile, H):
    s = PROFILE_TABLE[profile]["s"]
    col = np.dtype([("ts", "<u8"), ("m", "<u2"), ("status", "<u2"), ("px", np.uint8, (H, s))])
    d = np.dtype([("header", np.uint8, 32), ("col", col, (COLUMNS,)), ("footer", np.uint8, 32)])
    assert d.itemsize == profile_packet_bytes(profile, H)
    return d


def _put(px, off, width, v):
    """v (uint32, one per pixel) little endian into bytes [off, off + width) of each pixel"""
    for b in range(width):
        px[..., off + b] = (v >> np.uint32(8 * b)) & np.uint32(0xFF)


def encode_profile(pk, profile, rng, flags=True):
    """the LEGACY packets pk re-encoded in `profile` (LEGACY: returned as they are): the same column stamps, measurement ids, status
    bit 0, ranges and reflectivities.  The range field is r & mask (the low-data field is round(r / 8), so its range is a multiple
    of 8 mm), the reflectivity its low byte.  Random bytes fill the packet header and footer, the other status bits, signal, NIR and
    padding, and with `flags` the bits above each range mask.  The dual profile's second return is a valid return that differs
    from the first one in range and reflectivity, also where the first has none."""
    if profile == LEGACY:
        return pk
    H = pk.dtype.base["px"].shape[0]
    t = PROFILE_TABLE[profile]
    src = pk.reshape(-1)
    out = np.zeros(len(pk), profile_packet_dtype(profile, H))
    out["header"] = rng.integers(0, 256, out["header"].shape)
    out["footer"] = rng.integers(0, 256, out["footer"].shape)
    col = out["col"]                                    # (n, 16): a packet's header and footer sit between its columns and the next
    col["ts"], col["m"] = src["ts"].reshape(-1, COLUMNS), src["m"].reshape(-1, COLUMNS)
    col["status"] = ((rng.integers(0, 65536, len(src)) & ~1) | (src["status"] & 1)).reshape(-1, COLUMNS)
    px = rng.integers(0, 256, (len(src), H, t["s"])).astype(np.uint8)
    r = src["px"]["range"].astype(np.uint64) & RANGE_MASK
    field = np.minimum((r + 4) >> 3, t["mask"]) if profile == LOW else r & t["mask"]
    field = field.astype(np.uint32)
    if flags:
        field |= rng.integers(0, 2**32, field.shape, dtype=np.uint64).astype(np.uint32) & ~np.uint32(t["mask"]) & \
            np.uint32(2**(8 * t["width"]) - 1)
    _put(px, 0, t["width"], field)
    refl = (src["px"]["refl"] & 0xFF).astype(np.uint32)
    _put(px, t["refl"], 1, refl)
    if profile == DUAL:                                 # range2 u32 @4 (19 bits) | reflectivity2 u8 @7
        r2 = ((field & np.uint32(0x7FFFF)) + rng.integers(1, 5000, field.shape).astype(np.uint32)) & np.uint32(0x7FFFF)
        r2[r2 == 0] = 1
        refl2 = (refl + np.uint32(1) + rng.integers(0, 254, refl.shape).astype(np.uint32)) & np.uint32(0xFF)
        _put(px, 4, 4, r2 | refl2 << np.uint32(24))
    col["px"] = px.reshape(col["px"].shape)
    return out


def profile_packets(rng, n, W, H, profile, flags=True, **kw):
    """n packets of `profile` (the columns of packets(rng, n, W, H, **kw), encode_profile)"""
    return encode_profile(packets(rng, n, W, H, **kw), profile, rng, flags)


def _xyz32(cal, m, p, r):
    """the header's xyz of pixel p of columns with ids m and ranges r (mm), float32"""
    ce, se, ca, sa, nf = _beams32(cal)
    C, S = table()
    q = m.astype(np.int64) * (TABLE // cal.columns_per_frame)
    c, s = C[q], S[q]
    e = r.astype(f32) * f32(0.001) - nf
    ch = c * ca[p] - s * sa[p]
    sh = s * ca[p] + c * sa[p]
    ee = e * ce[p]
    return np.stack([ee * ch + nf * c, -(ee * sh + nf * s), e * se[p]], 1).astype(f32).reshape(-1, 3)


def profile_to_points(pk, cal, profile):
    """msg2points of packets of `profile`, read from their bytes by the header's table: (xyz, time, intensity, range, slot) of the
    points, in slot order"""
    if profile == LEGACY:
        return to_points(pk, cal)
    W, H = cal.columns_per_frame, cal.pixels_per_column
    t = PROFILE_TABLE[profile]
    raw = np.frombuffer(bytes(memoryview(np.ascontiguousarray(pk))), np.uint8)
    dt = profile_packet_dtype(profile, H)
    col = raw.view(dt)["col"].reshape(-1) if len(raw) else np.zeros(0, dt["col"].base)
    px = col["px"].reshape(-1, t["s"]).astype(np.uint32)
    word = sum(px[:, b] << np.uint32(8 * b) for b in range(t["width"]))
    r = (word & np.uint32(t["mask"])) << np.uint32(t["shift"])
    n = H * len(col)
    i = np.arange(n)
    g, p = i // H, i % H
    valid = ((col["status"][g] & 1) == 1) & (col["m"][g].astype(np.int64) < W) & (r != 0)
    g, p, r, i = g[valid], p[valid], r[valid], i[valid]
    xyz = _xyz32(cal, col["m"][g], p, r)
    ts = col["ts"][g]
    tm = (ts // np.uint64(10**9)).astype(np.int64).astype(np.float64) + (ts % np.uint64(10**9)).astype(np.float64) * 1e-9
    return xyz, tm, px[i, t["refl"]].astype(f32), r.astype(f32), i.astype(np.int32)


def profile_process(pk, cal, profile, rate, min_dist):
    """Accumulator::process on packets of `profile`: msg2points -> decimation on the rank -> stable time sort"""
    xyz, t, inten, rg, idx = profile_to_points(pk, cal, profile)
    keep = F.temporal(xyz, rate, min_dist)
    order = keep[np.argsort(t[keep], kind="stable")]
    return xyz[order], t[order], inten[order], rg[order], idx[order]


def metadata(layout, W, alt, az, profile=None, origin_mm=ORIGIN_MM):
    """metadata in the firmware 1.x ("v1") or 2.x ("v2") layout with udp_profile_lidar = profile (a name), or without that key"""
    if layout == "v1":
        extra = {} if profile is None else {"udp_profile_lidar": profile}
        return metadata_v1(W, alt, az, origin_mm, **extra)
    d = json.loads(metadata_v2(W, alt, az, origin_mm))
    if profile is None:
        d["config_params"].pop("udp_profile_lidar")
    else:
        d["config_params"]["udp_profile_lidar"] = profile
    return json.dumps(d)
