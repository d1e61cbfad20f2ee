"""The lidar UDP profiles of Ouster firmware 2.2+ (RNG19_RFL8_SIG16_NIR16, its dual-return form and the low-data RNG15_RFL8_NIR8)
without a GPU.

lv_ouster_packets_to_points equals the NumPy restatement of the header's table (tests/ouster_profile_cases.py, profile_to_points) bit for
bit for every profile, H and W, n = 0 and 12.163 mm, with invalid columns, ids >= W, ranges of 0, flag bits above the range masks,
random packet headers and footers, and a second return that differs from the first; then through the decimator and the time sort.
With LEGACY the new entry point equals lv_ouster_to_points.  One frame encoded as LEGACY and as each new profile gives the same
points; the low-data profile's ranges lie on the 8 mm grid within 8 mm of the geometry; the os_cloud_node cloud of each profile's
points reads back through the Ouster PointCloud2 path.  The metadata reader's profiles and refusals, the argument errors of the host
and device calls (before any device work: the device pointers are never dereferenced), and a packet-only RNG19 bag."""
import ctypes as C
import json

import numpy as np
import pytest

import bagwriter as BW
import frontend_ref as F
import ouster_cases as OC
import ouster_profile_cases as OP
from test_bag_reader import OUSTER, CloudLayout
from test_ouster_ref import bad_calibrations, read_bag

BASE = 1 << 40                       # a device address that is never touched
f32 = np.float32
PROFILES = (OP.LEGACY,) + OP.NEW_PROFILES


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64 if a.dtype.itemsize == 8 else np.uint32).tobytes()


def same(got, ref, what):
    assert len(got) == len(ref) == 5, what
    for name, a, b in zip(("xyz", "time", "intensity", "range", "idx"), got, ref):
        assert a.shape == b.shape and bits(a) == bits(b), (what, name, a.shape, b.shape)


def host_chain(lv, pk, cal, profile, rate, md):
    """lv_ouster_packets_to_points -> the decimator on the rank (frontend_ref.temporal) -> lv_time_sort_indices"""
    xyz, t, inten, rg, idx = lv.ouster_to_points(pk.tobytes(), cal, profile)
    keep = F.temporal(xyz, rate, md)
    order = keep[lv.time_sort_indices(t[keep])] if len(keep) else keep
    return xyz[order], t[order], inten[order], rg[order], idx[order]


# ---- the host decoder against the restatement ------------------------------------------------------------------------------------
def test_packet_sizes_follow_the_table(lv):
    assert [OP.profile_packet_bytes(p, 64) for p in OP.NEW_PROFILES] == [12_544, 16_640, 4_352]
    for p in PROFILES:
        for H in OC.HS:
            assert lv.ouster_packet_bytes(H, p) == OP.profile_packet_bytes(p, H)


@pytest.mark.parametrize("profile", OP.NEW_PROFILES)
@pytest.mark.parametrize("H", OC.HS)
def test_profile_decoder_equals_the_restatement(lv, profile, H):
    rng = np.random.default_rng(40 + 4 * H + profile)
    seen = 0
    for Wc in OC.WS:
        for n in (0.0, OC.ORIGIN_MM):
            cal = OC.calibration(lv, Wc, H, n, rng)
            pk = OP.profile_packets(rng, 6, Wc, H, profile, m0=Wc - 40, invalid=0.05, bad_m=0.05)   # across the frame wrap
            ref = OP.profile_to_points(pk, cal, profile)
            same(lv.ouster_to_points(pk.tobytes(), cal, profile), ref, (Wc, n))
            seen += len(ref[0])
            for rate, md in ((1, 0.0), (3, 0.9), (8, 3.0)):
                same(host_chain(lv, pk, cal, profile, rate, md), OP.profile_process(pk, cal, profile, rate, md), (Wc, n, rate, md))
    assert seen > 6 * 16 * H * 6 * 0.7


@pytest.mark.parametrize("profile", OP.NEW_PROFILES)
def test_profile_msg2points_rule(lv, profile):
    """which slots are points, from the bytes: status bit 0 (the other status bits, the flags above the range mask, the header,
    footer and, for dual return, the second return do not matter)"""
    rng = np.random.default_rng(41 + profile)
    t = OP.PROFILE_TABLE[profile]
    cal = OC.calibration(lv, 1024, 32)
    pk = OP.profile_packets(rng, 8, 1024, 32, profile, invalid=0.2, bad_m=0.2, zero=0.3)
    col = pk["col"].reshape(-1)
    idx = lv.ouster_to_points(pk.tobytes(), cal, profile)[4]
    px = col["px"].reshape(-1, t["s"]).astype(np.uint32)
    word = sum(px[:, b] << np.uint32(8 * b) for b in range(t["width"]))
    g = np.arange(len(word)) // 32
    want = ((col["status"][g] & 1) == 1) & (col["m"][g] < 1024) & ((word & t["mask"]) != 0)
    assert set(idx.tolist()) == set(np.nonzero(want)[0].tolist())
    assert ((col["status"] & 1) == 0).any() and ((col["status"] >> 1) != 0).any() and (col["m"] >= 1024).any()
    assert ((word & t["mask"]) == 0).any() and ((word & ~np.uint32(t["mask"])) != 0).any()    # no return; flags above the mask
    if profile == OP.DUAL:
        second = px[:, 4] | px[:, 5] << 8 | (px[:, 6] & 7) << 16
        assert (second[~want] != 0).all()                              # the second return of the slots that are not points
    noise = pk.copy()                                                  # header, footer, flags and the other status bits are not read
    noise["header"], noise["footer"] = 255 - pk["header"], 255 - pk["footer"]
    noise["col"]["status"] ^= 0xFFFE
    flip = (0xFFFFFFFF >> (32 - 8 * t["width"])) & ~t["mask"] & (0x00FFFFFF if profile == OP.DUAL else 0xFFFFFFFF)
    pxn = noise["col"]["px"]
    w = sum(pxn[..., b].astype(np.uint32) << np.uint32(8 * b) for b in range(t["width"])) ^ np.uint32(flip)
    for b in range(t["width"]):
        pxn[..., b] = (w >> np.uint32(8 * b)) & np.uint32(0xFF)
    assert not np.array_equal(noise["col"]["px"], pk["col"]["px"])
    same(lv.ouster_to_points(noise.tobytes(), cal, profile), lv.ouster_to_points(pk.tobytes(), cal, profile), "noise")


def test_second_return_never_leaks(lv):
    """dual return: the first return only, whatever the second holds"""
    rng = np.random.default_rng(42)
    cal = OC.calibration(lv, 1024, 64, OC.ORIGIN_MM, rng)
    pk = OP.profile_packets(rng, 8, 1024, 64, OP.DUAL)
    got = lv.ouster_to_points(pk.tobytes(), cal, OP.DUAL)
    swapped = pk.copy()                                                # another second return
    swapped["col"]["px"][..., 4:8] = rng.integers(0, 256, swapped["col"]["px"][..., 4:8].shape)
    same(lv.ouster_to_points(swapped.tobytes(), cal, OP.DUAL), got, "second return")
    px = pk["col"]["px"].reshape(-1, 16).astype(np.uint32)
    first = (px[:, 0] | px[:, 1] << 8 | px[:, 2] << 16 | px[:, 3] << 24) & 0x7FFFF
    second = (px[:, 4] | px[:, 5] << 8 | px[:, 6] << 16 | px[:, 7] << 24) & 0x7FFFF
    assert (first != second).all() and (px[:, 3] != px[:, 7]).all()
    assert bits(got[3]) == bits(first[got[4]].astype(f32)) and bits(got[2]) == bits(px[got[4], 3].astype(f32))


# ---- LEGACY through the new entry points ---------------------------------------------------------------------------------------------
def test_legacy_entry_point_is_unchanged(lv):
    L = lv.lib()
    rng = np.random.default_rng(43)
    for Wc, H in ((512, 16), (1024, 64), (2048, 128)):
        cal = OC.calibration(lv, Wc, H, OC.ORIGIN_MM, rng)
        pk = OC.packets(rng, 5, Wc, H, m0=Wc - 20, invalid=0.1, bad_m=0.1)
        raw = np.frombuffer(pk.tobytes(), np.uint8)
        n = 16 * H * len(pk)
        outs = []
        for fn, extra in ((L.lv_ouster_to_points, ()), (L.lv_ouster_packets_to_points, (OP.LEGACY,))):
            out = (np.empty((n, 3), f32), np.empty(n), np.empty(n, f32), np.empty(n, f32), np.empty(n, np.int32))
            m = C.c_int64(-1)
            assert fn(raw.ctypes.data, len(raw), len(pk), C.byref(cal), *extra, *(a.ctypes.data for a in out), C.byref(m)) == lv.OK
            outs.append(tuple(a[:m.value] for a in out))
        same(outs[1], outs[0], (Wc, H))
        same(outs[0], OC.to_points(pk, cal), (Wc, H))
        for k, nb in ((5, len(raw) - 1), (-1, len(raw))):               # and the same refusals
            for fn, extra in ((L.lv_ouster_to_points, ()), (L.lv_ouster_packets_to_points, (OP.LEGACY,))):
                m = C.c_int64(7)
                assert fn(raw.ctypes.data, nb, k, C.byref(cal), *extra, *(a.ctypes.data for a in out), C.byref(m)) == lv.ERR_ARG
                assert m.value == 0


# ---- one frame in every profile -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("profile", (OP.RNG19, OP.DUAL))
def test_one_frame_in_legacy_and_rng19_gives_the_same_points(lv, profile):
    rng = np.random.default_rng(44 + profile)
    cal = OC.calibration(lv, 1024, 64, OC.ORIGIN_MM, rng)
    pk = OC.frame(rng, 1024, 64, invalid=0.05, bad_m=0.02)
    refl = pk.reshape(-1)["px"]["refl"]
    small = rng.random(refl.shape) < 0.8
    refl[small] &= 0xFF                                                # most reflectivities fit a byte, some do not
    a = lv.ouster_to_points(pk.tobytes(), cal)
    b = lv.ouster_to_points(OP.encode_profile(pk, profile, rng).tobytes(), cal, profile)
    for k in (0, 1, 3, 4):                                             # xyz, time, range, slot
        assert bits(a[k]) == bits(b[k]), k
    low = a[2] < 256
    assert low.sum() > 0.7 * len(low) and (~low).sum() > 0.1 * len(low)
    assert bits(a[2][low]) == bits(b[2][low]) and (b[2] < 256).all()
    assert len(a[0]) > 50_000


def test_low_data_ranges_lie_on_the_8mm_grid_near_the_geometry(lv):
    """points placed in the LiDAR frame (as test_ouster_ref's geometric check) and encoded in the low-data profile"""
    rng = np.random.default_rng(45)
    Wc, H, n = 1024, 64, OC.ORIGIN_MM
    alt, az = OC.beam_angles(H, rng)
    cal = lv.ouster_calibration(Wc, alt, az, n)
    pk = OC.packets(rng, 4, Wc, H, m0=int(rng.integers(0, Wc)), invalid=0, bad_m=0, zero=0, garbage=False)
    slot = np.arange(16 * H * 4)
    col = pk.reshape(-1)
    g, p = slot // H, slot % H
    a = 2 * np.pi * col["m"][g].astype(np.float64) / Wc
    el, th = np.radians(np.array(alt))[p], a + np.radians(np.array(az))[p]
    origin = (n / 1000.0) * np.stack([np.cos(a), -np.sin(a), np.zeros_like(a)], 1)
    s = rng.uniform(0.5, 110.0, len(slot))
    pts = origin + s[:, None] * np.stack([np.cos(el) * np.cos(th), -np.cos(el) * np.sin(th), np.sin(el)], 1)
    col["px"]["range"] = np.round(s * 1000.0 + n).astype(np.uint32).reshape(-1, H)
    xyz, t, inten, rg, idx = lv.ouster_to_points(OP.encode_profile(pk, OP.LOW, rng).tobytes(), cal, OP.LOW)
    assert (idx == slot).all()
    assert (rg % 8 == 0).all() and (np.abs(rg - col["px"]["range"].reshape(-1)) <= 4).all()
    err = np.linalg.norm(xyz.astype(np.float64) - pts, axis=1)
    assert err.max() < 0.008, err.max()
    stamp = col["ts"][g]
    assert (t == stamp // 10**9 + (stamp % 10**9) * 1e-9).all()


@pytest.mark.parametrize("profile", PROFILES)
def test_same_points_as_the_pointcloud2_path(lv, profile):
    """each profile's decoded frame written as os_cloud_node's cloud (48-byte layout, reflectivity and range as decoded) and read by
    lv_pointcloud2_to_points_checked(LV_LIDAR_OUSTER, stamp_beginning=1, offset_beginning=1)"""
    rng = np.random.default_rng(46 + profile)
    cal = OC.calibration(lv, 1024, 64, OC.ORIGIN_MM, rng)
    legacy = OC.frame(rng, 1024, 64, ts0=1_712_345_678 * 10**9 + 123_000)
    col = legacy.reshape(-1)
    col["status"][0], col["m"][0] = OC.VALID, 0
    col["px"]["range"][0, 0] = 5000
    pk = OP.encode_profile(legacy, profile, rng)
    xyz, t, inten, rg, idx = lv.ouster_to_points(pk.tobytes(), cal, profile)
    ts = col["ts"][idx // 64]
    assert idx[0] == 0 and ts[0] % 1000 == 0
    stamp_us = int(ts[0]) // 1000
    cloud = np.zeros(len(t), OUSTER)
    cloud["x"], cloud["y"], cloud["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    cloud["t"] = (ts - np.uint64(stamp_us * 1000)).astype(np.uint32)
    cloud["reflectivity"] = inten.astype(np.uint16)
    cloud["ring"] = idx % 64
    cloud["range"] = rg.astype(np.uint32)
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


# ---- the metadata JSON reader --------------------------------------------------------------------------------------------------------
def sensor(lv, text):
    """lv_ouster_sensor_from_json: (status, calibration, profile), the outputs preset to garbage"""
    raw = text.encode() if isinstance(text, str) else text
    cal, prof = lv.OusterCalibration(), C.c_int(77)
    cal.columns_per_frame = 99
    st = lv.lib().lv_ouster_sensor_from_json(raw, len(raw), C.byref(cal), C.byref(prof))
    return st, cal, prof.value


@pytest.mark.parametrize("layout", ["v1", "v2"])
def test_metadata_profiles(lv, layout):
    rng = np.random.default_rng(47)
    alt, az = OC.beam_angles(64, rng)
    n = OC.ORIGIN_MM
    for name in (None,) + OP.PROFILE_NAMES:
        text = OP.metadata(layout, 2048, alt, az, name, n)
        cal, profile = lv.ouster_sensor_from_json(text)
        assert profile == (OP.LEGACY if name is None else OP.PROFILE_NAMES.index(name)), name
        assert profile == lv.OUSTER_PROFILES.get(name, lv.OUSTER_LEGACY)
        assert (cal.columns_per_frame, cal.pixels_per_column, list(cal.beam_altitude_angles[:64]),
                list(cal.beam_azimuth_angles[:64]), cal.lidar_origin_to_beam_origin_mm) == (2048, 64, alt, az, n), name
        st = lv.lib().lv_ouster_calibration_from_json(text.encode(), len(text), C.byref(lv.OusterCalibration()))
        assert st == (lv.OK if profile == OP.LEGACY else lv.ERR_ARG), name            # the LEGACY reader is unchanged
    compact = json.dumps(json.loads(OP.metadata("v2", 512, alt[:16], az[:16], "RNG15_RFL8_NIR8")), separators=(",", ":"))
    assert lv.ouster_sensor_from_json(compact)[1] == OP.LOW


def test_metadata_refusals(lv):
    alt, az = OC.beam_angles(64)
    good = json.loads(OP.metadata("v2", 1024, alt, az, "RNG19_RFL8_SIG16_NIR16"))

    def v2(edit):
        d = json.loads(json.dumps(good))
        edit(d)
        return json.dumps(d)

    def refused(text):
        st, cal, prof = sensor(lv, text)
        return st == lv.ERR_ARG and cal.columns_per_frame == 0 and prof == OP.LEGACY

    assert sensor(lv, json.dumps(good))[0] == lv.OK and sensor(lv, json.dumps(good))[2] == OP.RNG19
    bad_profiles = ("FUSA_RNG15_RFL8_NIR8_DUAL", "FUSA_RNG15_RFL8_NIR8", "RNG19_RFL8_SIG16_NIR16_dual", "rng19_rfl8_sig16_nir16",
                    "RNG19_RFL8_SIG16", "LEGACY ", "", "RNG15_RFL8_NIR8_DUAL")
    cases = {"profile %r" % p: v2(lambda d, p=p: d["config_params"].update(udp_profile_lidar=p)) for p in bad_profiles}
    cases.update({
        "profile not a string": v2(lambda d: d["config_params"].update(udp_profile_lidar=1)),
        "profile null": v2(lambda d: d["config_params"].update(udp_profile_lidar=None)),
        "v1 FUSA": OP.metadata("v1", 1024, alt, az, "FUSA_RNG15_RFL8_NIR8_DUAL"),
        # every refusal of the LEGACY reader other than the profile, with a new profile
        "no altitudes": v2(lambda d: d["beam_intrinsics"].pop("beam_altitude_angles")),
        "no azimuths": v2(lambda d: d["beam_intrinsics"].pop("beam_azimuth_angles")),
        "no mode": v2(lambda d: d["config_params"].pop("lidar_mode")),
        "lengths differ": v2(lambda d: d["beam_intrinsics"]["beam_azimuth_angles"].pop()),
        "H = 20": OC.metadata_v2(1024, alt[:20], az[:20], profile="RNG19_RFL8_SIG16_NIR16"),
        "H = 0": v2(lambda d: d["beam_intrinsics"].update(beam_altitude_angles=[], beam_azimuth_angles=[])),
        "W = 1000": v2(lambda d: d["config_params"].update(lidar_mode="1000x10")),
        "W = 4096": v2(lambda d: d["config_params"].update(lidar_mode="4096x5")),
        "mode without rate": v2(lambda d: d["config_params"].update(lidar_mode="1024")),
        "mode without W": v2(lambda d: d["config_params"].update(lidar_mode="x10")),
        "mode with letters": v2(lambda d: d["config_params"].update(lidar_mode="1024x10a")),
        "mode not a string": v2(lambda d: d["config_params"].update(lidar_mode=1024)),
        "pixels_per_column": v2(lambda d: d["lidar_data_format"].update(pixels_per_column=32)),
        "columns_per_packet": v2(lambda d: d["lidar_data_format"].update(columns_per_packet=8)),
        "origin not a number": v2(lambda d: d["beam_intrinsics"].update(lidar_origin_to_beam_origin_mm="12.163")),
        "string in an array": v2(lambda d: d["beam_intrinsics"]["beam_altitude_angles"].__setitem__(3, "x")),
        "null in an array": v2(lambda d: d["beam_intrinsics"]["beam_azimuth_angles"].__setitem__(3, None)),
        "not an array": v2(lambda d: d["beam_intrinsics"].update(beam_altitude_angles=1.0)),
    })
    for name, text in cases.items():
        assert refused(text), name
    text = json.dumps(good)
    assert refused(text[:text.index("beam_azimuth_angles") + 60])      # truncated inside an array
    assert refused(text.replace(json.dumps(alt[0]), "1e999", 1))       # not finite
    L = lv.lib()
    cal, prof = lv.OusterCalibration(), C.c_int(5)
    assert L.lv_ouster_sensor_from_json(None, 10, C.byref(cal), C.byref(prof)) == lv.ERR_ARG
    assert L.lv_ouster_sensor_from_json(text.encode(), -1, C.byref(cal), C.byref(prof)) == lv.ERR_ARG
    assert L.lv_ouster_sensor_from_json(text.encode(), len(text), None, C.byref(prof)) == lv.ERR_ARG
    assert L.lv_ouster_sensor_from_json(text.encode(), len(text), C.byref(cal), None) == lv.ERR_ARG
    raw = text.encode()                                                 # len bounds the text: the profile's string is cut
    assert refused(raw[:raw.index(b'"RNG19_RFL8') + 8])


# ---- argument errors ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("profile", PROFILES)
def test_host_decoder_refusals(lv, profile):
    L = lv.lib()
    H = 32
    cal = OC.calibration(lv, 1024, H)
    pk = OP.profile_packets(np.random.default_rng(48), 3, 1024, H, profile)
    raw = np.frombuffer(pk.tobytes(), np.uint8)
    assert len(raw) == 3 * OP.profile_packet_bytes(profile, H)
    n = 16 * H * 3
    out = [np.empty(3 * n, f32), np.empty(n), np.empty(n, f32), np.empty(n, f32), np.empty(n, np.int32)]
    ptr = [a.ctypes.data_as(C.c_void_p) for a in out]
    m = C.c_int64(7)

    def call(data=raw.ctypes.data_as(C.c_void_p), nb=len(raw), k=3, c=cal, prof=profile, outs=ptr, n_out=True):
        m.value = 7
        st = L.lv_ouster_packets_to_points(data, nb, k, C.byref(c) if c is not None else None, prof, *outs, C.byref(m) if n_out else None)
        return st, m.value
    good = len(OP.profile_to_points(pk, cal, profile)[0])
    assert call() == (lv.OK, good)
    assert call(outs=ptr[:2] + [None] * 3) == (lv.OK, good)
    assert call(k=0, nb=0) == (lv.OK, 0)
    assert call(nb=len(raw) + 5) == (lv.OK, good)
    for kw in (dict(nb=len(raw) - 1), dict(k=2, nb=2 * OP.profile_packet_bytes(profile, H) - 1), dict(k=1, nb=0), dict(data=None),
               dict(k=-1), dict(k=OC.max_packets(H) + 1, nb=1 << 40), dict(c=None), dict(outs=[None] + ptr[1:]),
               dict(outs=ptr[:1] + [None] + ptr[2:]), dict(nb=-1), dict(prof=-1), dict(prof=4), dict(prof=99)):
        assert call(**kw) == (lv.ERR_ARG, 0), kw
    assert call(n_out=False)[0] == lv.ERR_ARG
    for bad in bad_calibrations(lv):
        assert call(c=bad) == (lv.ERR_ARG, 0)


@pytest.mark.parametrize("asynch", [False, True])
@pytest.mark.parametrize("profile", PROFILES)
def test_device_refusals_before_device_work(lv, profile, asynch):
    L = lv.lib()
    H, k = 64, 10
    cal = OC.calibration(lv, 1024, H)
    nb, ns = OP.profile_packet_bytes(profile, H) * k, 16 * H * k

    def call(data=BASE, data_bytes=nb, n_packets=k, c=cal, prof=profile, outs=None, n_out=True):
        outs = outs if outs is not None else [BASE + (1 << 30) + j * (1 << 24) for j in range(5)]
        cp = C.byref(c) if c is not None else None
        if asynch:
            st = L.lv_process_ouster_packets_device_async(None, data, data_bytes, n_packets, cp, prof, 4, 3.0, *outs,
                                                          BASE + (1 << 35) if n_out else None)
        else:
            m = C.c_int64(7)
            st = L.lv_process_ouster_packets_device(None, data, data_bytes, n_packets, cp, prof, 4, 3.0, *outs,
                                                    C.byref(m) if n_out else None)
            if n_out:
                assert m.value == 0
        return st, L.lv_last_error()
    handle = (lv.ERR_ARG, b"process ouster: null handle")
    assert call() == handle                                            # every argument good: only the handle is missing
    assert call(n_packets=0, data_bytes=0) == handle
    for kw in (dict(data=None), dict(n_out=False), dict(c=None)):
        st, msg = call(**kw)
        assert st == lv.ERR_ARG and b"null packets" in msg, kw
    st, msg = call(data_bytes=nb - 1)
    assert st == lv.ERR_ARG and b"too short" in msg
    for prof in (-1, 4, 1 << 20):
        st, msg = call(prof=prof)
        assert st == lv.ERR_ARG and b"profile" in msg, prof
    for n_packets in (-1, OC.max_packets(H) + 1):
        st, msg = call(n_packets=n_packets, data_bytes=1 << 45)
        assert st == lv.ERR_ARG and (b"n_packets" in msg or b"negative" in msg), n_packets
    for bad in bad_calibrations(lv):
        st, msg = call(c=bad)
        assert st == lv.ERR_ARG and (b"not finite" in msg or b"columns_per_frame" in msg or b"pixels_per_column" in msg), msg
    for j, size in enumerate((12, 8, 4, 4, 4)):
        outs = [BASE + (1 << 30) + i * (1 << 24) for i in range(5)]
        outs[j] = BASE + nb - 1
        st, msg = call(outs=outs)
        assert st == lv.ERR_ARG and b"overlaps" in msg, j
        outs[j] = BASE - size * ns                                     # adjacent is fine
        assert call(outs=outs) == handle, j


# ---- a packet-only RNG19 bag ---------------------------------------------------------------------------------------------------------
def test_rng19_packet_only_bag(lv, tmp_path):
    rng = np.random.default_rng(49)
    alt, az = OC.beam_angles(64, rng)
    text = OP.metadata("v2", 1024, alt, az, "RNG19_RFL8_SIG16_NIR16")
    pk = OP.profile_packets(rng, 6, 1024, 64, OP.RNG19)
    conns = {0: ("/ouster/metadata", "std_msgs/String"), 1: ("/ouster/lidar_packets", "ouster_sensor_msgs/PacketMsg"),
             2: ("/ouster/imu_packets", "ouster_sensor_msgs/PacketMsg")}
    msgs = [(0, 100, 0, OC.string_msg(text))]
    imus = []
    for k in range(len(pk)):
        msgs.append((1, 100, 1000 + k, OC.packet_msg(pk[k].tobytes())))
        imus.append(OC.imu_packet(int(pk[k]["col"][0]["ts"]), rng.normal(0, 0.1, 3), rng.normal(0, 5, 3)))
        msgs.append((2, 100, 1000 + k, OC.packet_msg(imus[-1])))
    path = str(tmp_path / "rng19.bag")
    BW.write_bag(path, conns, msgs)
    L = lv.lib()
    got = read_bag(lv, path)                                           # parses only ouster_ros/PacketMsg: do it here for the new type
    assert [g[1] for g in got] == [conns[c][1] for c, *_ in msgs]
    cal, profile = lv.ouster_sensor_from_json(got[0][2][4:])
    assert profile == OP.RNG19 and cal.pixels_per_column == 64 and cal.columns_per_frame == 1024
    lidar, imu = [], []
    for topic, _, payload, _, _, _ in got[1:]:
        v = lv.OusterPacketView()
        assert L.lv_bag_parse_ouster_packet(payload, len(payload), C.byref(v)) == lv.OK
        (lidar if topic.endswith("lidar_packets") else imu).append(C.string_at(v.data, v.bytes))
    assert lidar == [pk[k].tobytes() for k in range(len(pk))] and imu == imus
    assert all(len(b) == lv.ouster_packet_bytes(64, profile) == 12_544 for b in lidar)
    same(lv.ouster_to_points(b"".join(lidar), cal, profile), OP.profile_to_points(pk, cal, OP.RNG19), "bag")
    assert lv.ouster_imu_packet(imu[0]).stamp_nsec == int(pk[0]["col"][0]["ts"]) % 10**9
